// fdx_tct.cu -- the TRANSPOSED formulation of the 3x3 convolution (forward and data gradient) for
// layers with few output channels (Cout = 64 / 128 forward, Cin = 64 / 128 in the data gradient).
//
// fdx_tc.cu puts the pixels in the M dimension, so a Cout = 64 layer can only issue N = 64 MMAs, whose
// shared-memory operand traffic per FLOP is twice that of N = 128.  Here the roles are swapped,
//     D^T[co, px] = sum_tap sum_ci  W_tap[ci, co]  *  X[px + tap, ci]
// A = the weight tile (M = 64 or 128 output channels x 64 k; MN-major straight from HWIO in the forward,
// K-major from the (Cout, Cin, tap) view in the data gradient), B = 256 pixels (two 16 x 8 TMA boxes of
// 64 channels, K-major).  The accumulator is D^T: row = output channel, column = pixel.  Two consumer
// warpgroups each own 128 of the pixel columns and issue m64 n128 k16 wgmma (two per K step at M = 128).
//
// M = 64 (64 output channels): TWO pixel halves (2 x 256 pixels, 16 wide x 32 tall) share a tile - half 0
// in accumulator rows 0-63, half 1 in rows 64-127 - so a warpgroup again holds a 128-row accumulator.  K
// steps alternate between the halves; the 8 KB weight tile is simply fetched for both.
//
// Warps 8..11 = producer (one thread issues TMA), warps 0..7 = the two consumer warpgroups (main loop, then epilogue on their own
// columns).  Geometry: stride 1, W and H multiples of 16.
#include "fdx_tc.cuh"
#include "fdx_epilogue.cuh"
#include <stdlib.h>

namespace {

constexpr int kEpiWarps = 8;                 // two warpgroups: the tile's pixel columns are split between them
constexpr int kThreads = 32 * kEpiWarps + 128;  // + the producer warpgroup (one thread issues TMA)
constexpr int kLdT = 128 + 4;                // row of the transposed exchange tile [32 px][128 channel rows]
constexpr int kPixBytes = 2 * 128 * 128;     // two boxes of 128 pixels x 64 channels bf16

struct TctDev {
  int nxb, nyb, nimg, W, H;
  int ntaps, tap_dx[kTcMaxTaps], tap_dy[kTcMaxTaps], tap_b[kTcMaxTaps];
  int kchunks, K, Ncols, cblks, ntiles;
  void* out;
  long long os_x, os_y, os_n;
  float alpha;
  const float* bias;
  const float* rowvec;
  const void* res;
  long long rs_x, rs_y, rs_n;
  float* cs_ws;            // fused per-(image, channel) sums or null
  int cs_slots, cs_ld;
  const float* gn_ab;      // GNB kernels: [N][2][Ncols] GroupNorm coefficients a, b of the tensor `res` (= x)
};

// HALO = true (3x3 stride-1 only): with per-tap loads every (tap, K chunk) re-loads its 256 pixels, 40 KB of TMA
// per 2.1 MFLOP at M = 64 = 52 FLOP per byte, so the layers are L2 -> shared-memory bandwidth bound.  ONE tall box of
// 16 x 18 pixels (rows y0-1 .. y0+16) is loaded per (kx, K chunk); the three ky taps are 2048-byte row offsets
// into it (swizzle-aligned views, exactly as in the nine-tap weight gradient), so a stage carries three weight
// tiles + 36 KB of pixels and feeds twelve MMAs: 96 -> 36 KB of pixel traffic per three taps.
// GNB = true (data gradient only): the first pass of the GroupNorm(+SiLU) backward in the epilogue - with x = the
// GroupNorm input (side input `res`) and z = a_c x + b_c the kernel stores dz = dy * silu'(z) instead of dy and
// accumulates S0 = sum dz, S1 = sum dz * x per (image, channel) into the column-sum workspace, exactly as the
// pixels-as-M engine's EPI_GN_BWD (fdx_epilogue.cuh).
template <int MT, bool A_MN, bool HALO, bool GNB>
__global__ void __launch_bounds__(kThreads, 1)
fdx_tct_kernel(const __grid_constant__ CUtensorMap mapW, const __grid_constant__ CUtensorMap mapX,
               const TctDev p) {
  constexpr int kWBytes = MT * 128;                       // MT channels x 64 k
  constexpr int kHaloBytes = 18 * 16 * 128;               // 16 x 18 pixel box
  constexpr int kStageBytes = HALO ? (3 * kWBytes + kHaloBytes) : (kWBytes + kPixBytes);
  constexpr int S = HALO ? ((MT == 128) ? 2 : 3) : ((MT == 128) ? 3 : 4);
  constexpr bool IL = (MT == 64);                         // two interleaved pixel halves per tile
  constexpr int NH = IL ? 2 : 1;
  constexpr int TH = 16 * NH;                             // pixel rows per tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * kStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == kEpiWarps && lane == 0) {
    tma_prefetch_desc(&mapW);
    tma_prefetch_desc(&mapX);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp >= kEpiWarps) producer_regs(); else consumer_regs();
  const int nk = p.ntaps * p.kchunks;

  if (warp >= kEpiWarps) {
    if (warp == kEpiWarps && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const int cb = tile % p.cblks;
        const int mt = tile / p.cblks;
        const int xb = mt % p.nxb, yb = (mt / p.nxb) % p.nyb, nb = mt / (p.nxb * p.nyb);
        const int x0 = xb * 16;
        if constexpr (HALO) {
          // stages: (kx, K chunk, half); taps t = ky * 3 + kx (fdx_conv3x3_fwd / dgrad fill order)
          for (int qq = 0; qq < 3 * p.kchunks * NH; ++qq) {
            const int q = qq / NH, y0 = yb * TH + 16 * (qq % NH);
            const int kx = q / p.kchunks, kc = q % p.kchunks;
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sw = smem + stage * kStageBytes;
            uint8_t* sx = sw + 3 * kWBytes;
            mbar_arrive_expect_tx(&full[stage], kStageBytes);
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
              const int t = ky * 3 + kx;
              if constexpr (A_MN) {
#pragma unroll
                for (int j = 0; j < MT / 64; ++j)
                  tma_load_4d(sw + ky * kWBytes + j * 8192, &mapW, &full[stage], cb * MT + j * 64,
                              p.tap_b[t] + kc * 64, 0, 0);
              } else {
                tma_load_4d(sw + ky * kWBytes, &mapW, &full[stage], kc * 64, cb * MT, p.tap_b[t], 0);
              }
            }
            tma_load_4d(sx, &mapX, &full[stage], kc * 64, x0 + kx - 1, y0 - 1, nb);
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        } else
        for (int qq = 0; qq < nk * NH; ++qq) {
          const int q = qq / NH, y0 = yb * TH + 16 * (qq % NH);
          const int t = q / p.kchunks, kc = q % p.kchunks;
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sw = smem + stage * kStageBytes;
          uint8_t* sx = sw + kWBytes;
          mbar_arrive_expect_tx(&full[stage], kStageBytes);
          if constexpr (A_MN) {
            // HWIO rows = (tap, ci), co contiguous: MT/64 boxes of (64 co, 64 k rows)
#pragma unroll
            for (int j = 0; j < MT / 64; ++j)
              tma_load_4d(sw + j * 8192, &mapW, &full[stage], cb * MT + j * 64, p.tap_b[t] + kc * 64, 0, 0);
          } else {
            // (k = Cout contiguous, rows = Cin, z1 = tap): one box (64 k, MT rows)
            tma_load_4d(sw, &mapW, &full[stage], kc * 64, cb * MT, p.tap_b[t], 0);
          }
          tma_load_4d(sx, &mapX, &full[stage], kc * 64, x0 + p.tap_dx[t], y0 + p.tap_dy[t], nb);
          tma_load_4d(sx + 16384, &mapX, &full[stage], kc * 64, x0 + p.tap_dx[t], y0 + 8 + p.tap_dy[t], nb);
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============ consumers: main loop, then epilogue ====================================================
    // The f32 values of a 32-pixel chunk are transposed through the warpgroup's shared-memory tile
    // [32 px][128 channel rows] and leave as 16-byte channel pieces: lane -> (pixel l / PPX + k * (32 / PPX),
    // piece l % PPX).  A lane always owns the same 8 channels, so bias, timestep row and the fused GroupNorm
    // sums are per-lane registers, reduced once per tile.
    const int q = warp & 3;
    const int wg = warp >> 2;
    const int ew = warp;                                 // 0 .. kEpiWarps-1
    const int c_begin = wg * 128, c_end = c_begin + 128;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const int xbar = 1 + wg;
    constexpr int PPX = 4;                               // 16-byte pieces per staged pixel column
    constexpr int CPW = IL ? 16 : 32;                    // channels owned by one warp
    float* xsT = reinterpret_cast<float*>(smem + S * kStageBytes + 256) + wg * (32 * kLdT);
    const int piece = lane % PPX, prow = lane / PPX;     // read phase: this lane's piece and first pixel
    // accumulator row of this lane's first channel: M = 128: channel; M = 64: half * 64 + channel
    const int srow = IL ? (piece >> 1) * 64 + q * 16 + (piece & 1) * 8 : q * 32 + piece * 8;
    __nv_bfloat16* outp = static_cast<__nv_bfloat16*>(p.out);
    const __nv_bfloat16* resp = static_cast<const __nv_bfloat16*>(p.res);
    WgAcc<128> acc;
    int stage = 0; uint32_t phase = 0;
    // Side input (residual / accumulate source): each epilogue chunk loads its own pieces, which hides an L2
    // hit, not HBM.  So the consumer threads pull the side input of the NEXT tile into L2 while they work on
    // the current one (one line per pixel and 64 channels; <= 64 KB per CTA in flight).
    auto prefetch_res = [&](int t) {
      if (resp == nullptr || t >= p.ntiles) return;
      const int cb_ = t % p.cblks, mt_ = t / p.cblks;
      const int xb_ = mt_ % p.nxb, yb_ = (mt_ / p.nxb) % p.nyb, nb_ = mt_ / (p.nxb * p.nyb);
      const int nch = min(MT, p.Ncols - cb_ * MT);
      const __nv_bfloat16* base = resp + (long long)nb_ * p.rs_n + (long long)(xb_ * 16) * p.rs_x + cb_ * MT;
      for (int pi = ew * 32 + lane; pi < TH * 16; pi += 32 * kEpiWarps) {
        const int y = yb_ * TH + (pi >> 4);
        if (y >= p.H) continue;
        const __nv_bfloat16* a = base + (long long)y * p.rs_y + (long long)(pi & 15) * p.rs_x;
        for (int c = 0; c < nch; c += 64) asm volatile("prefetch.global.L2 [%0];" ::"l"(a + c));
      }
    };
    prefetch_res(blockIdx.x);
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      prefetch_res(tile + gridDim.x);
      const int cb = tile % p.cblks;
      const int mt = tile / p.cblks;
      const int xb = mt % p.nxb, yb = (mt / p.nxb) % p.nyb, nb = mt / (p.nxb * p.nyb);
      const int cw0 = cb * MT + q * CPW;                  // first channel of this warp
      // read phase: piece -> (pixel half, 8-channel group); half 1 lies 16 pixel rows below half 0
      const int yh = yb * TH + (IL ? 16 * (piece >> 1) : 0);
      const long long obase = (long long)nb * p.os_n + (long long)yh * p.os_y + (long long)(xb * 16) * p.os_x;
      const long long rbase = (long long)nb * p.rs_n + (long long)yh * p.rs_y + (long long)(xb * 16) * p.rs_x;
      const int ch = cw0 + (IL ? (piece & 1) : piece) * 8;   // read phase: this lane's first channel
      const bool ch_ok = ch < p.Ncols && yh < p.H;           // (H % 32 == 16: the last tile has no half 1)
      float add[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) add[i] = 0.f;
      if (ch_ok) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (p.bias) add[i] += __ldg(p.bias + ch + i);
          if (p.rowvec) add[i] += __ldg(p.rowvec + (long long)nb * p.Ncols + ch + i);
        }
      }
      float ga[8], gb[8];
      if constexpr (GNB) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { ga[i] = 0.f; gb[i] = 0.f; }
        if (ch_ok) {
          const float4* a4 = reinterpret_cast<const float4*>(p.gn_ab + (long long)nb * 2 * p.Ncols + ch);
          const float4* b4 = reinterpret_cast<const float4*>(p.gn_ab + ((long long)nb * 2 + 1) * p.Ncols + ch);
          const float4 a0 = __ldg(a4), a1 = __ldg(a4 + 1), b0 = __ldg(b4), b1 = __ldg(b4 + 1);
          ga[0] = a0.x; ga[1] = a0.y; ga[2] = a0.z; ga[3] = a0.w; ga[4] = a1.x; ga[5] = a1.y; ga[6] = a1.z; ga[7] = a1.w;
          gb[0] = b0.x; gb[1] = b0.y; gb[2] = b0.z; gb[3] = b0.w; gb[4] = b1.x; gb[5] = b1.y; gb[6] = b1.z; gb[7] = b1.w;
        }
      }
      auto load_res = [&](int c0, uint4 (&r)[PPX]) {
#pragma unroll
        for (int k = 0; k < PPX; ++k) {
          const int j = prow + k * (32 / PPX);
          r[k] = make_uint4(0, 0, 0, 0);
          if (resp && ch_ok && c0 < c_end)
            r[k] = *reinterpret_cast<const uint4*>(resp + rbase + (long long)(c0 / 16 + (j >> 4)) * p.rs_y +
                                                   (long long)(j & 15) * p.rs_x + ch);
        }
      };
      uint4 rcur[PPX];
      // ---- main loop: this warpgroup's 128 pixel columns ----
      acc.zero();
      int prev = -1;
      auto release = [&]() {
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      };
      // The half index is a compile-time constant (the halves are an unrolled inner loop): with a run-time
      // choice of accumulator, or with the two halves' wgmma on different control paths, ptxas serialises
      // every wgmma of the kernel.  For the same reason a tile without half 1 (H % 32 == 16) still runs it,
      // on the zero rows TMA fills in below the image; the epilogue stores none of it.
      const int nq = HALO ? 3 * p.kchunks : nk;
      for (int kq = 0; kq < nq; ++kq) {
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
          mbar_wait(&full[stage], phase);
          wgmma_fence();
          const uint32_t sw = smem_u32(smem + stage * kStageBytes);
          // HALO: pixel rows 8 wg .. 8 wg + 7 of the box view; per-tap: this warpgroup's 128-pixel box
          const uint32_t sx = sw + (HALO ? 3 : 1) * kWBytes + wg * 16384;
#pragma unroll
          for (int ky = 0; ky < (HALO ? 3 : 1); ++ky) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t aw = A_MN ? sw + ky * kWBytes + k * 2048 : sw + ky * kWBytes + k * 32;
              const uint64_t db = gmma_desc_sw128(sx + ky * 2048 + k * 32, 16, 1024);   // HALO: rows ky .. ky+15
              const uint64_t da = A_MN ? gmma_desc_sw128(aw, 8192, 1024) : gmma_desc_sw128(aw, 16, 1024);
              if constexpr (IL) {
                acc.mma_half<A_MN ? 1 : 0, 0>(hh, da, db);
              } else {
                acc.mma<A_MN ? 1 : 0, 0>(da, A_MN ? gmma_desc_sw128(aw + 8192, 8192, 1024)
                                                  : gmma_desc_sw128(aw + 8192, 16, 1024), db);
              }
            }
          }
          release();
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);

      float s0[8], s1[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { s0[i] = 0.f; s1[i] = 0.f; }
      // Unrolled: the chunk index is a compile-time register index, and the 32 accumulator registers of a
      // chunk die once it is written out, which keeps the epilogue within the consumer register budget.
#pragma unroll
      for (int ci = 0; ci < 4; ++ci) {
        const int c0 = c_begin + 32 * ci;
        // The side input of this chunk is requested before the exchange so its latency overlaps it.  (A
        // register prefetch one chunk ahead would keep 16 more registers live and push the epilogue into spills.)
        load_res(c0, rcur);
        // ---- write phase: accumulator fragments of columns c0 .. c0+31 -> xsT[px][channel row] ----
        named_bar_sync(xbar, 128);                       // the previous chunk's reads are done
        {
          const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int r = h * 64 + w * 16 + (l >> 2), n = jj * 8 + 2 * (l & 3);
              const float* d = &acc.d[h][(ci * 4 + jj) * 4];
              xsT[n * kLdT + r] = d[0];
              xsT[(n + 1) * kLdT + r] = d[1];
              xsT[n * kLdT + r + 8] = d[2];
              xsT[(n + 1) * kLdT + r + 8] = d[3];
            }
        }
        named_bar_sync(xbar, 128);
        // ---- read phase: 16-byte channel pieces; columns c0 .. c0+31 = pixel rows c0/16, c0/16 + 1 ----
#pragma unroll
        for (int k = 0; k < PPX; ++k) {
          const int j = prow + k * (32 / PPX);            // pixel (column) within the chunk
          const int ty = c0 / 16 + (j >> 4), tx = j & 15;
          const float4 a = *reinterpret_cast<const float4*>(xsT + j * kLdT + srow);
          const float4 b = *reinterpret_cast<const float4*>(xsT + j * kLdT + srow + 4);
          float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) f[i] = f[i] * p.alpha + add[i];
          if (ch_ok) {
            float xv[8];
            if (resp) {
              const uint4 r = rcur[k];
              const float2 r0 = unpack_bf16x2(r.x), r1 = unpack_bf16x2(r.y), r2 = unpack_bf16x2(r.z),
                           r3 = unpack_bf16x2(r.w);
              xv[0] = r0.x; xv[1] = r0.y; xv[2] = r1.x; xv[3] = r1.y;
              xv[4] = r2.x; xv[5] = r2.y; xv[6] = r3.x; xv[7] = r3.y;
              if constexpr (GNB) {
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] = epi_silu_grad_times(f[i], fmaf(xv[i], ga[i], gb[i]));
              } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] += xv[i];
              }
            }
            uint4 o;
            o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
            o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
            *reinterpret_cast<uint4*>(outp + obase + (long long)ty * p.os_y + (long long)tx * p.os_x + ch) = o;
            if (p.cs_ws) {
              const float2 h0 = unpack_bf16x2(o.x), h1 = unpack_bf16x2(o.y), h2 = unpack_bf16x2(o.z),
                           h3 = unpack_bf16x2(o.w);
              const float hv[8] = {h0.x, h0.y, h1.x, h1.y, h2.x, h2.y, h3.x, h3.y};
              // second factor: the GroupNorm input x (GNB) or the stored value itself (forward column statistics)
#pragma unroll
              for (int i = 0; i < 8; ++i) { s0[i] += hv[i]; s1[i] = fmaf(hv[i], GNB ? xv[i] : hv[i], s1[i]); }
            }
          }
        }
      }
      if (p.cs_ws) {
        // lanes with the same piece (l % PPX) hold the same 8 channels: combine them
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
          for (int o = (IL ? 2 : PPX); o < 32; o <<= 1) {
            s0[i] += __shfl_xor_sync(0xffffffffu, s0[i], o);
            s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], o);
          }
        }
        if (lane < (IL ? 2 : PPX) && ch < p.Ncols) {
          float* w = p.cs_ws + (((long long)(tile % p.cs_slots) * p.nimg + nb) * 2) * p.cs_ld + ch;
#pragma unroll
          for (int i = 0; i < 8; ++i) { atomicAdd(w + i, s0[i]); atomicAdd(w + p.cs_ld + i, s1[i]); }
        }
      }
    }
  }
}

template <int MT, bool A_MN, bool HALO, bool GNB = false>
int launch_tct(const CUtensorMap& mW, const CUtensorMap& mX, const TctDev& d, cudaStream_t stream) {
  constexpr int S = HALO ? ((MT == 128) ? 2 : 3) : ((MT == 128) ? 3 : 4);
  constexpr int stage = HALO ? (3 * MT * 128 + 18 * 16 * 128) : (MT * 128 + kPixBytes);
  constexpr int smem = S * stage + 1024 + 256 + 2 * 32 * kLdT * 4 /* epilogue transpose tiles */;
  static_assert(smem <= 227 * 1024, "tct: shared memory");
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(fdx_tct_kernel<MT, A_MN, HALO, GNB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  int grid = fdx_num_sms();
  if (grid <= 0) return FDX_ERR_NO_DEVICE;
  if (d.ntiles < grid) grid = d.ntiles;
  fdx_tct_kernel<MT, A_MN, HALO, GNB><<<grid, kThreads, smem, stream>>>(mW, mX, d);
  fdx_note_kernel(FDX_KERNEL_TCT);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // namespace

// FDX_ERR_UNSUPPORTED (no error text) = geometry not covered; the caller uses the generic engine.
int fdx_tct_launch(const TcLaunch& L, cudaStream_t stream) {
  if (L.mode == TC_MNMN || L.gemm_like || L.es != 1 || L.out_f32 || L.out_atomic || L.b_batched)
    return FDX_ERR_UNSUPPORTED;
  // fused GroupNorm-backward first pass: data gradient with x as the side input and the sums workspace
  if (L.gn_ab && (L.mode != TC_KK || !L.res || !L.gn_ws || L.bias || L.rowvec)) return FDX_ERR_UNSUPPORTED;
  // column counts the generic engine would have to cover with N < 256 tiles (64, 128, 192, 320, 384, ...)
  if (L.Ncols % 64 != 0 || L.Ncols % 256 == 0 || L.Ncols > 512) return FDX_ERR_UNSUPPORTED;
  if (L.W % 16 != 0 || L.H % 16 != 0 || L.K % 64 != 0) return FDX_ERR_UNSUPPORTED;
  TctDev d{};
  d.W = L.W; d.H = L.H; d.nimg = L.N;
  const int MT = (L.Ncols % 128 == 0) ? 128 : 64;
  d.nxb = L.W / 16; d.nyb = (MT == 64) ? (L.H + 31) / 32 : L.H / 16;
  d.ntaps = L.ntaps;
  for (int i = 0; i < kTcMaxTaps; ++i) { d.tap_dx[i] = L.tap_dx[i]; d.tap_dy[i] = L.tap_dy[i]; d.tap_b[i] = L.tap_b[i]; }
  d.K = L.K; d.kchunks = L.K / 64; d.Ncols = L.Ncols;
  d.cblks = L.Ncols / MT;
  d.ntiles = d.cblks * d.nxb * d.nyb * d.nimg;
  d.out = L.out; d.os_x = L.os_x; d.os_y = L.os_y; d.os_n = L.os_n;
  d.alpha = L.alpha; d.bias = L.bias; d.rowvec = L.rowvec;
  d.res = L.res; d.rs_x = L.rs_x; d.rs_y = L.rs_y; d.rs_n = L.rs_n;
  d.cs_ws = L.gn_ws; d.cs_slots = L.gn_slots > 0 ? L.gn_slots : 1; d.cs_ld = L.ws_ld > 0 ? L.ws_ld : L.Ncols;
  d.gn_ab = L.gn_ab;

  // halo-sharing variant: standard 3x3 stride-1 tap set in (ky, kx) order.  FDX_TCT_HALO=0 disables it,
  // FDX_TCT_HALO=64 / 128 restricts it to that M tile.
  bool halo = L.ntaps == 9;
  for (int t = 0; t < 9 && halo; ++t) halo = (L.tap_dx[t] == t % 3 - 1) && (L.tap_dy[t] == t / 3 - 1);
  const char* he = getenv("FDX_TCT_HALO");          // read per launch: the A/B tests toggle it in-process
  const int halo_env = (he && *he) ? atoi(he) : -1;
  if (halo_env == 0 || (halo_env > 0 && halo_env != MT)) halo = false;
  CUtensorMap mW, mX;
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.A.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.A.strides[i] * 2;
    uint32_t box[4] = {64, 16, (uint32_t)(halo ? 18 : 8), 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&mX, L.A.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.B.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.B.strides[i] * 2;
    uint32_t box[4] = {64, (uint32_t)(L.mode == TC_KK ? MT : 64), 1, 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&mW, L.B.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
#define FDX_TCT_GO(M_, AMN_)                                                                   \
  (halo ? launch_tct<M_, AMN_, true>(mW, mX, d, stream) : launch_tct<M_, AMN_, false>(mW, mX, d, stream))
  if (L.mode == TC_KMN) return MT == 128 ? FDX_TCT_GO(128, true) : FDX_TCT_GO(64, true);
  if (L.gn_ab) {
#define FDX_TCT_GN(M_) \
  (halo ? launch_tct<M_, false, true, true>(mW, mX, d, stream) : launch_tct<M_, false, false, true>(mW, mX, d, stream))
    return MT == 128 ? FDX_TCT_GN(128) : FDX_TCT_GN(64);
#undef FDX_TCT_GN
  }
  return MT == 128 ? FDX_TCT_GO(128, false) : FDX_TCT_GO(64, false);
#undef FDX_TCT_GO
}
