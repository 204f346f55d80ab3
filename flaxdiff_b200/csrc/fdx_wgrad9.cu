// fdx_wgrad9.cu -- 3x3 convolution weight gradient with all nine taps in one CTA.
//
//   dW[ky][kx][ci][co] = sum_{n,y,x} X[n, y+ky-1, x+kx-1, ci] * dY[n, y, x, co]
// (the weight half of jax.value_and_grad through flax nn.Conv, flaxdiff/models/common.py:166-172 via
//  trainer/general_diffusion_trainer.py:321-322).
//
// The generic split-K engine (fdx_tc.cu, TC_MNMN) re-reads X and dY from L2 once per (tap, row block,
// column block).  Here one CTA owns a 64(ci) x 64(co) block of ALL nine taps for its slice of the pixels, and
// the SHIFTS ARE SPLIT between the operands:  dW[ky][kx][ci][co] = sum_px X[y+ky-1, x'][ci] * dY[y, x'-kx+1][co]
//   * A (M) = the ky views of ONE X box (TH+2 rows, no x halo): rows of TW pixels are TW*128 B apart
//             (1024-aligned), so each ky is a 64-channel MN-major operand at a plain byte offset;
//   * B (N) = THREE dY boxes shifted by kx-1 pixels (TMA zero-fills outside the image), contiguous in shared
//             memory: N = 3 kx x 64 co = 192 (descriptor leading-dimension offset 8192).
// Consumer warpgroup ky issues one m64 n192 k16 wgmma per 16 pixels; its accumulator row is (ky, ci) and its
// columns (kx, co) are contiguous in HWIO, so the split-K partial sums leave the registers as 8-byte
// red.global.add.v2.f32.  36 KB of TMA per 64-pixel block.
// Tiles = (ci block, co block, pixel split).
#include "fdx_common.cuh"
#include "../../include/fdx.h"

namespace {

constexpr int kStages = 5;
constexpr int kThreads = 3 * 128 + 32;   // three consumer warpgroups (ky) + the producer warp

struct W9Dev {
  int TW, TH;              // pixel patch (TW*TH == 64)
  int nxb, nyb, nimg;
  int Cin, Cout, cib, cob;
  int splits, ntiles;
  float* dw;               // [9][Cin][Cout] f32, accumulated
};

__global__ void __launch_bounds__(kThreads, 1)
fdx_wgrad9_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapY,
                  const W9Dev p) {
  constexpr int S = kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int row_bytes = p.TW * 128;                      // one pixel row of the box: TW pixels x 64 channels
  const int xbuf_bytes = (p.TH + 2) * row_bytes;         // multiple of 1024
  const int ybuf_bytes = 64 * 128;
  const int stage_bytes = xbuf_bytes + 3 * ybuf_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 12 && lane == 0) {
    tma_prefetch_desc(&mapX);
    tma_prefetch_desc(&mapY);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 3); }
    fence_barrier_init();
  }
  __syncthreads();
  const long long kblocks = (long long)p.nxb * p.nyb * p.nimg;

  if (warp == 12) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        int r = tile;
        const int cb = r % p.cib; r /= p.cib;
        const int ob = r % p.cob; r /= p.cob;
        const int sp = r;
        const int pb0 = (int)((kblocks * sp) / p.splits), pb1 = (int)((kblocks * (sp + 1)) / p.splits);
        for (int pb = pb0; pb < pb1; ++pb) {
          const int xb = pb % p.nxb, yb = (pb / p.nxb) % p.nyb, nb = pb / (p.nxb * p.nyb);
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sx = smem + stage * stage_bytes;
          uint8_t* sy = sx + xbuf_bytes;
          mbar_arrive_expect_tx(&full[stage], stage_bytes);
          tma_load_4d(sx, &mapX, &full[stage], cb * 64, xb * p.TW, yb * p.TH - 1, nb);
#pragma unroll
          for (int kx = 0; kx < 3; ++kx)     // dY[y, x' - kx + 1]
            tma_load_4d(sy + kx * ybuf_bytes, &mapY, &full[stage], ob * 64, xb * p.TW + 1 - kx, yb * p.TH, nb);
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    const int ky = warp >> 2;                            // this warpgroup's row of taps
    const int w = warp & 3;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float acc[96];
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      int r = tile;
      const int cb = r % p.cib; r /= p.cib;
      const int ob = r % p.cob; r /= p.cob;
      const int sp = r;
      const int nk = (int)((kblocks * (sp + 1)) / p.splits) - (int)((kblocks * sp) / p.splits);
#pragma unroll
      for (int i = 0; i < 96; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int i = 0; i < nk; ++i) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t sx = smem_u32(smem + stage * stage_bytes);
        const uint32_t sy = sx + xbuf_bytes;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = gmma_desc_sw128(sx + ky * row_bytes + k * 2048, 1024, 1024);   // 64 ci x 16 px
          const uint64_t db = gmma_desc_sw128(sy + k * 2048, 8192, 1024);                    // 3 kx x 64 co
          wgmma_bf16<192, 1, 1>(acc, da, db);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
      if (nk > 0) {
        // fragment: rows ci = 16 w + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1) = (kx, co)
        const int ci = cb * 64 + w * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 24; ++j) {
          const int kx = j >> 3, co = ob * 64 + (j & 7) * 8 + 2 * (lane & 3);
          if (co >= p.Cout) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (ci + 8 * h >= p.Cin) continue;
            float* out = p.dw + ((long long)(ky * 3 + kx) * p.Cin + ci + 8 * h) * p.Cout + co;
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(out), "f"(acc[4 * j + 2 * h]),
                         "f"(acc[4 * j + 2 * h + 1])
                         : "memory");
          }
        }
      }
    }
  }
}

}  // namespace

// Returns FDX_ERR_UNSUPPORTED (without setting an error) when the shape does not fit this kernel;
// the caller then uses the generic engine.
int fdx_wgrad9_launch(const fdx_act* x, const fdx_act* dy, float* dw, cudaStream_t stream) {
  const int W = dy->w, H = dy->h;
  if (W < 8 || (W & (W - 1)) != 0 || (H & (H - 1)) != 0) return FDX_ERR_UNSUPPORTED;
  if (x->w != W || x->h != H) return FDX_ERR_UNSUPPORTED;
  W9Dev d{};
  d.TW = W >= 16 ? 16 : 8;
  d.TH = 64 / d.TW;
  if (H < d.TH) return FDX_ERR_UNSUPPORTED;
  d.nxb = W / d.TW; d.nyb = H / d.TH; d.nimg = dy->n;
  d.Cin = x->c; d.Cout = dy->c;
  d.cib = (x->c + 63) / 64; d.cob = (dy->c + 63) / 64;
  d.dw = dw;
  const long long kblocks = (long long)d.nxb * d.nyb * d.nimg;
  const long long bt = (long long)d.cib * d.cob;
  const int sms = fdx_num_sms();
  if (sms <= 0) return FDX_ERR_NO_DEVICE;
  double best = -1.0; int splits = 1;
  for (int w = 1; w <= 4; ++w) {
    long long sp = ((long long)sms * w) / bt;
    if (sp < 1) sp = 1;
    if (sp > kblocks) sp = kblocks;
    const long long tiles = bt * sp, waves = (tiles + sms - 1) / sms;
    const double eff = (double)tiles / (double)(waves * sms);
    if (eff > best + 0.03) { best = eff; splits = (int)sp; }
  }
  d.splits = splits;
  d.ntiles = (int)(bt * splits);

  CUtensorMap mX, mY;
  {
    uint64_t dims[4] = {(uint64_t)x->c, (uint64_t)x->w, (uint64_t)x->h, (uint64_t)x->n};
    uint64_t str[3] = {(uint64_t)x->pix_stride * 2, (uint64_t)x->pix_stride * x->w * 2,
                       (uint64_t)x->pix_stride * x->w * x->h * 2};
    uint32_t box[4] = {64, (uint32_t)d.TW, (uint32_t)(d.TH + 2), 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&mX, x->ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  {
    uint64_t dims[4] = {(uint64_t)dy->c, (uint64_t)dy->w, (uint64_t)dy->h, (uint64_t)dy->n};
    uint64_t str[3] = {(uint64_t)dy->pix_stride * 2, (uint64_t)dy->pix_stride * dy->w * 2,
                       (uint64_t)dy->pix_stride * dy->w * dy->h * 2};
    uint32_t box[4] = {64, (uint32_t)d.TW, (uint32_t)d.TH, 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&mY, dy->ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  // Cout must be even for the 8-byte reductions (it is a multiple of 64 on every UNet layer).
  if (d.Cout % 2 != 0) return FDX_ERR_UNSUPPORTED;
  const int stage_bytes = (d.TH + 2) * d.TW * 128 + 3 * 64 * 128;
  const int smem_bytes = kStages * stage_bytes + 1024 + 256;
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(fdx_wgrad9_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  kStages * (6 * 16 * 128 + 3 * 64 * 128) + 1024 + 256));
    attr_set = true;
  }
  const int grid = sms < d.ntiles ? sms : d.ntiles;
  fdx_wgrad9_kernel<<<grid, kThreads, smem_bytes, stream>>>(mX, mY, d);
  fdx_note_kernel(FDX_KERNEL_WGRAD9);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}
