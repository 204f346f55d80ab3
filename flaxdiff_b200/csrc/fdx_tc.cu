// fdx_tc.cu -- the wgmma / TMA "tap-GEMM" engine for sm_90a.
//
// Replaces what the reference delegates to XLA for every dense contraction on the
// UNet hot path: flax nn.Conv 3x3 / 1x1 (flaxdiff/models/common.py:166-172,
// 237-244, 324-333), nn.DenseGeneral projections (models/attention.py:132-154)
// and the QK^T / PV products of nn.dot_product_attention (attention.py:170-174),
// forward and backward.
//
// Design (one CTA per SM, persistent over 128 x BN output tiles):
//   last WG     TMA producer (one thread): per K-chunk one 128B-swizzled A box (64 channels x
//               128 pixels, shifted by the tap offset; out-of-image = zero fill
//               = SAME padding) and the matching B box, into a ring of stages.
//   warpgroups  consumers (one per 128 output columns): wgmma m64 x {64,128} x 16
//               (bf16 -> f32 registers) over all 128 rows, release each stage once
//               its MMAs retire, then run the epilogue on their own columns: fuse
//               bias + per-image timestep vector + residual, store bf16/f32 (or f32
//               atomics for the split-K weight gradient).
#include "fdx_tc.cuh"
#include "fdx_epilogue.cuh"
#include <stdlib.h>

namespace {

constexpr int kBK = 64;                 // K elements (or K rows) per pipeline stage
constexpr int kABytes = 128 * kBK * 2;  // 16 KB per stage for A in every mode

template <int BN>
struct TcCfg {
  static constexpr int kWG = (BN == 256) ? 2 : 1;   // consumer warpgroups; each owns BN / kWG columns
  static constexpr int kWN = BN / kWG;              // wgmma N
  static constexpr int kThreads = 128 * (kWG + 1);  // + the producer warpgroup (one thread issues TMA)
  // K chunks (64 deep) per pipeline stage: at BN = 64 one chunk is only 8 wgmma (two row halves x 4 K
  // steps), too little work per mbarrier round trip, so two chunks share a stage there.  Not used by the
  // MN-major-A (weight-gradient) mode.
  static constexpr int kSub = (BN == 64) ? 2 : 1;
  static constexpr int kStages = (BN == 128) ? 5 : 3;   // as many as fit in 227 KB
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kSub * (kABytes + kBBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/ +
                                    kWG * (16384 /*epilogue staging: 4 warps x 4 KB*/ + kAccXchgBytes);
  static_assert(kSmemBytes <= 227 * 1024, "tc: shared memory");
};

struct TcDev {
  int mode;
  int TW, TH, TN;        // pixel box of one A tile (128 pixels for K-major A, 64 for MN-major A)
  int nxb, nyb, nnb;     // pixel blocks along x, y, n
  int W, H, N;
  int es;
  int ntaps;
  int tap_dx[kTcMaxTaps], tap_dy[kTcMaxTaps], tap_b[kTcMaxTaps];
  int es_b, tap_bdx[kTcMaxTaps], tap_bdy[kTcMaxTaps];   // TC_MNMN strided / shifted B view
  int kchunks;           // K chunks per tap (TC_KK/TC_KMN)
  int K;
  int M;                 // TC_MNMN valid rows
  int mblks;             // TC_MNMN: row blocks of 128
  int Ncols, nblks;      // column blocks of BN
  int b_batched;
  int mn_batched;        // TC_MNMN: reduce over x blocks only, (y, n) blocks are batch
  int tpp;               // TC_MNMN: taps per tile (2 when M <= 64: two taps share one M=128 MMA)
  int ntp;               // TC_MNMN: number of tap groups = ceil(ntaps / tpp)
  int splits;
  int ntiles;
  // epilogue
  void* out;
  int out_f32, out_atomic;
  long long os_x, os_y, os_n, os_tap, os_m;
  float alpha;
  const float* bias;
  const float* rowvec;
  const void* res;
  long long rs_x, rs_y, rs_n;
  // fused GroupNorm-backward first pass (GN kernels only; see fdx_epilogue.cuh)
  const float* gn_ab;
  float* gn_ws;
  int gn_slots;
  int ws_ld;               // row length of gn_ws (EPI_COLSTATS: channels of the destination buffer)
};

// TC_MNMN tile decode: tile -> (batch block bz, split, nt, mb, tap) and the K range [pb0, pb1)
struct MnTile {
  int bz, sp, nt, mb, t, pb0, pb1;
};
__device__ __forceinline__ MnTile decode_mn(const TcDev& p, int tile) {
  // fastest -> slowest: tap group, column block, row block, batch block, K split.  CTAs that run
  // concurrently therefore work on the same pixel range and share A / B boxes in L2.
  MnTile m;
  int r = tile;
  const int nbz = p.mn_batched ? p.nyb * p.nnb : 1;
  m.t = r % p.ntp;     r /= p.ntp;
  m.nt = r % p.nblks;  r /= p.nblks;
  m.mb = r % p.mblks;  r /= p.mblks;
  m.bz = r % nbz;      r /= nbz;
  m.sp = r;
  const long long kblocks = p.mn_batched ? p.nxb : (long long)p.nxb * p.nyb * p.nnb;
  m.pb0 = (int)((kblocks * m.sp) / p.splits);
  m.pb1 = (int)((kblocks * (m.sp + 1)) / p.splits);
  return m;
}

template <int BN, int MODE, int EPI>
__global__ void __launch_bounds__(TcCfg<BN>::kThreads, 1)
fdx_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
              const TcDev p) {
  using Cfg = TcCfg<BN>;
  constexpr int S = Cfg::kStages;
  constexpr int WN = Cfg::kWN;
  constexpr bool A_MN = (MODE == TC_MNMN);
  constexpr bool B_MN = (MODE != TC_KK);
  constexpr int SUB = A_MN ? 1 : Cfg::kSub;    // K chunks per stage

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * Cfg::kStageBytes);
  uint64_t* full = bars;            // [S]
  uint64_t* empty = bars + S;       // [S]
  uint8_t* epi_stage = smem + S * Cfg::kStageBytes + 256;   // kWG x 16 KB, 128-byte aligned
  float* acc_xchg = reinterpret_cast<float*>(epi_stage + Cfg::kWG * 16384);   // kWG x kAccXchgBytes

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kProducer = 4 * Cfg::kWG;

  if (warp == kProducer && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], Cfg::kWG);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (Cfg::kWG == 2) {
    if (warp >= kProducer) producer_regs(); else consumer_regs();
  }

  // ---- tile decode helpers ------------------------------------------------
  // TC_KK / TC_KMN : tile -> (nt, xb, yb, nb);  nk = ntaps * kchunks
  // TC_MNMN        : tile -> (split, nt, mb, tap); nk = pixel blocks of this split

  if (warp >= kProducer) {
    // =========================== TMA producer ==============================
    if (warp == kProducer && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        if constexpr (!A_MN) {
          const int nt = tile % p.nblks;
          const int mt = tile / p.nblks;
          const int xb = mt % p.nxb;
          const int yb = (mt / p.nxb) % p.nyb;
          const int nb = mt / (p.nxb * p.nyb);
          const int x0 = xb * p.TW * p.es, y0 = yb * p.TH * p.es, n0 = nb * p.TN;
          const int zb1 = p.b_batched ? yb : 0, zb2 = p.b_batched ? nb : 0;
          const int nk = p.ntaps * p.kchunks;
          for (int q = 0; q < nk; q += SUB) {
            const int nsub = (nk - q) < SUB ? (nk - q) : SUB;
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa0 = smem + stage * Cfg::kStageBytes;
            uint8_t* sb0 = sa0 + SUB * kABytes;
            mbar_arrive_expect_tx(&full[stage], nsub * (kABytes + Cfg::kBBytes));
            for (int u = 0; u < nsub; ++u) {
              const int t = (q + u) / p.kchunks, kc = (q + u) % p.kchunks;
              uint8_t* sa = sa0 + u * kABytes;
              uint8_t* sb = sb0 + u * Cfg::kBBytes;
              tma_load_4d(sa, &mapA, &full[stage], kc * kBK, x0 + p.tap_dx[t], y0 + p.tap_dy[t], n0);
              if constexpr (!B_MN) {
                // B K-major: box (64 k, BN rows); tap selects z1 (or batched z1/z2)
                tma_load_4d(sb, &mapB, &full[stage], kc * kBK, nt * BN,
                            p.b_batched ? zb1 : p.tap_b[t], zb2);
              } else {
                // B MN-major: BN/64 boxes of (64 n, 64 k rows)
#pragma unroll
                for (int j = 0; j < BN / 64; ++j)
                  tma_load_4d(sb + j * (kBK * 128), &mapB, &full[stage], nt * BN + j * 64,
                              p.tap_b[t] + kc * kBK, zb1, zb2);
              }
            }
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        } else {
          const MnTile mt_ = decode_mn(p, tile);
          const int nt = mt_.nt, mb = mt_.mb, t = mt_.t;
          for (int pb = mt_.pb0; pb < mt_.pb1; ++pb) {
            int xb, yb, nb;
            if (p.mn_batched) {
              xb = pb; yb = mt_.bz % p.nyb; nb = mt_.bz / p.nyb;
            } else {
              xb = pb % p.nxb; yb = (pb / p.nxb) % p.nyb; nb = pb / (p.nxb * p.nyb);
            }
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * Cfg::kStageBytes;
            uint8_t* sb = sa + kABytes;
            mbar_arrive_expect_tx(&full[stage], kABytes + Cfg::kBBytes);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              // tpp == 1: the two 64-channel halves of row block mb for tap t
              // tpp == 2: channels [0,64) of taps 2t and 2t+1 (a missing tap reads out of range = 0)
              const int tap = (p.tpp == 2) ? (2 * t + j) : t;
              const bool live = tap < p.ntaps;
              const int tt = live ? tap : 0;
              const int ch = (p.tpp == 2) ? (live ? 0 : (int)p.M + 64) : (mb * 128 + j * 64);
              tma_load_4d(sa + j * (kBK * 128), &mapA, &full[stage], ch,
                          xb * p.TW * p.es + p.tap_dx[tt], yb * p.TH * p.es + p.tap_dy[tt], nb * p.TN);
            }
            const int tb = (p.tpp == 2) ? 0 : t;    // per-tap B views only without tap pairing
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_4d(sb + j * (kBK * 128), &mapB, &full[stage], nt * BN + j * 64,
                          xb * p.TW * p.es_b + p.tap_bdx[tb], yb * p.TH * p.es_b + p.tap_bdy[tb], nb * p.TN);
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ========================= consumer warpgroups ==========================
    const int wg = warp >> 2;            // columns [wg * WN, wg * WN + WN) of the tile
    const int q = warp & 3;
    const int row = q * 32 + lane;       // accumulator row this thread stores in the epilogue
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float* xs = acc_xchg + wg * (kAccXchgBytes / 4);
    const int xbar = 1 + wg;             // named barrier of this warpgroup's accumulator exchange
    WgAcc<WN> acc;
    int stage = 0;
    uint32_t phase = 0;
    int gn_par = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      int nt;
      bool valid;
      long long obase, rbase = 0;
      int img = 0;
      bool has_acc = true;
      int nk;
      if constexpr (!A_MN) {
        nt = tile % p.nblks;
        const int mt = tile / p.nblks;
        const int xb = mt % p.nxb;
        const int yb = (mt / p.nxb) % p.nyb;
        const int nb = mt / (p.nxb * p.nyb);
        const int tx = row % p.TW, ty = (row / p.TW) % p.TH, tn = row / (p.TW * p.TH);
        const int x = xb * p.TW + tx, y = yb * p.TH + ty, n = nb * p.TN + tn;
        valid = (x < p.W) && (y < p.H) && (n < p.N);
        img = n;
        obase = (long long)n * p.os_n + (long long)y * p.os_y + (long long)x * p.os_x;
        nk = p.ntaps * p.kchunks;
        if (p.res) {
          rbase = (long long)n * p.rs_n + (long long)y * p.rs_y + (long long)x * p.rs_x;
          // the side input of this row: request all of its lines now (L2 prefetch), before the main loop -
          // the epilogue's own register prefetch runs only one 64-column chunk ahead
          if (valid && !p.out_f32 && !p.out_atomic) {
            const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(p.res) + rbase + nt * BN + wg * WN;
            const int ncol = min(WN, p.Ncols - nt * BN - wg * WN);
            for (int c = 0; c < ncol; c += 64) asm volatile("prefetch.global.L2 [%0];" ::"l"(a + c));
          }
        }
      } else {
        const MnTile mt_ = decode_mn(p, tile);
        nt = mt_.nt;
        int m, tap;
        if (p.tpp == 2) { m = row & 63; tap = 2 * mt_.t + (row >> 6); }
        else            { m = mt_.mb * 128 + row; tap = mt_.t; }
        valid = (m < p.M) && (tap < p.ntaps);
        obase = (long long)p.tap_b[valid ? tap : 0] * p.os_tap + (long long)m * p.os_m;
        if (p.mn_batched)
          obase += (long long)(mt_.bz % p.nyb) * p.os_y + (long long)(mt_.bz / p.nyb) * p.os_n;
        nk = mt_.pb1 - mt_.pb0;
        has_acc = nk > 0;
      }
      // main loop: the MMAs of stage s are retired (and s released to the producer) while those of s+1 run
      auto mainloop = [&]() {
        acc.zero();
        int prev = -1;
        for (int qk = 0; qk < nk; qk += SUB) {
          const int nsub = (nk - qk) < SUB ? (nk - qk) : SUB;
          mbar_wait(&full[stage], phase);
          wgmma_fence();
          const uint32_t sa0 = smem_u32(smem + stage * Cfg::kStageBytes);
          const uint32_t sb0 = sa0 + SUB * kABytes + wg * WN * 128;   // this warpgroup's B columns
          for (int u = 0; u < nsub; ++u) {
            const uint32_t sa = sa0 + u * kABytes;
            const uint32_t sb = sb0 + u * Cfg::kBBytes;
#pragma unroll
            for (int k = 0; k < kBK / 16; ++k) {
              // K-major: advance 16 elements (32 B) inside the 128B swizzle row; SBO = 8 rows.
              // MN-major: advance 16 k-rows (2048 B); LBO = next 64-wide block, SBO = 8 rows.
              // Rows 64..127 of A start 8 KB further in both layouts.
              const uint32_t ao = A_MN ? sa + k * 2048 : sa + k * 32;
              const uint64_t da0 = A_MN ? gmma_desc_sw128(ao, kBK * 128, 1024) : gmma_desc_sw128(ao, 16, 1024);
              const uint64_t da1 = A_MN ? gmma_desc_sw128(ao + 8192, kBK * 128, 1024)
                                        : gmma_desc_sw128(ao + 8192, 16, 1024);
              const uint64_t db = B_MN ? gmma_desc_sw128(sb + k * 2048, kBK * 128, 1024)
                                       : gmma_desc_sw128(sb + k * 32, 16, 1024);
              acc.template mma<A_MN ? 1 : 0, B_MN ? 1 : 0>(da0, da1, db);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
          prev = stage;
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
      };
      if (!A_MN && !p.out_f32 && !p.out_atomic) {
        // bf16 output: stage through shared memory so global stores / side-input loads are coalesced
        EpiArgs ea{p.out, p.bias, p.rowvec, p.res, p.Ncols, p.alpha, p.gn_ab, p.gn_ws, p.N, p.ws_ld};
        epilogue_bf16_coalesced<WN, EPI>(ea, epi_stage + (wg * 4 + q) * 4096, acc, xs, xbar, lane,
                                         nt * BN + wg * WN, valid && has_acc, obase, rbase, img, mainloop,
                                         &gn_par, EPI != EPI_PLAIN ? tile % p.gn_slots : 0);
      } else {
      mainloop();
#pragma unroll 1
      for (int c0 = 0; c0 < WN; c0 += 32) {
        float f[32];
        acc.row32(xs, xbar, c0, f);
        const int col0 = nt * BN + wg * WN + c0;
        if (valid && has_acc && col0 < p.Ncols) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] *= p.alpha;
          if (p.bias) {
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] += __ldg(p.bias + col0 + j);
          }
          if (p.rowvec) {
            const float* rv = p.rowvec + (long long)img * p.Ncols + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] += __ldg(rv + j);
          }
          if (p.res) {
            const uint4* rp =
                reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(p.res) + rbase + col0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint4 u = rp[j];
              float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
                     d = unpack_bf16x2(u.w);
              f[8 * j + 0] += a.x; f[8 * j + 1] += a.y; f[8 * j + 2] += b.x; f[8 * j + 3] += b.y;
              f[8 * j + 4] += c.x; f[8 * j + 5] += c.y; f[8 * j + 6] += d.x; f[8 * j + 7] += d.y;
            }
          }
          if (p.out_atomic) {
            float* op = static_cast<float*>(p.out) + obase + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j) atomicAdd(op + j, f[j]);
          } else if (p.out_f32) {
            float4* op = reinterpret_cast<float4*>(static_cast<float*>(p.out) + obase + col0);
#pragma unroll
            for (int j = 0; j < 8; ++j)
              op[j] = make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
          } else {
            uint4* op =
                reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.out) + obase + col0);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              uint4 u;
              u.x = pack_bf16x2(f[8 * j + 0], f[8 * j + 1]);
              u.y = pack_bf16x2(f[8 * j + 2], f[8 * j + 3]);
              u.z = pack_bf16x2(f[8 * j + 4], f[8 * j + 5]);
              u.w = pack_bf16x2(f[8 * j + 6], f[8 * j + 7]);
              op[j] = u;
            }
          }
        }
      }
      }
    }
  }
}

template <int BN, int MODE, int EPI>
int launch_cfg(const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d, cudaStream_t stream) {
  using Cfg = TcCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(fdx_tc_kernel<BN, MODE, EPI>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  int grid = fdx_num_sms();
  if (grid <= 0) return FDX_ERR_NO_DEVICE;
  if (d.ntiles < grid) grid = d.ntiles;
  fdx_tc_kernel<BN, MODE, EPI><<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mA, mB, d);
  fdx_note_kernel(FDX_KERNEL_TC);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

template <int BN, int MODE>
int launch_gn(const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d, cudaStream_t stream) {
  if constexpr (MODE == TC_KK) {
    if (d.gn_ab) return launch_cfg<BN, MODE, EPI_GN_BWD>(mA, mB, d, stream);
  }
  if constexpr (MODE == TC_KMN) {
    if (d.gn_ws && !d.gn_ab) return launch_cfg<BN, MODE, EPI_COLSTATS>(mA, mB, d, stream);
  }
  return launch_cfg<BN, MODE, EPI_PLAIN>(mA, mB, d, stream);
}

template <int MODE>
int launch_mode(int BN, const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d,
                cudaStream_t stream) {
  switch (BN) {
    case 64: return launch_gn<64, MODE>(mA, mB, d, stream);
    case 128: return launch_gn<128, MODE>(mA, mB, d, stream);
    case 256: return launch_gn<256, MODE>(mA, mB, d, stream);
  }
  fdx_set_error("tc: unsupported BN %d", BN);
  return FDX_ERR_UNSUPPORTED;
}

int pow2_floor(int v) {
  int p = 1;
  while (p * 2 <= v) p *= 2;
  return p;
}

}  // namespace

int fdx_tc_launch(const TcLaunch& L, cudaStream_t stream) {
  FDX_REQUIRE(L.mode >= TC_KK && L.mode <= TC_MNMN, "tc: bad mode %d", L.mode);
  FDX_REQUIRE(L.ntaps >= 1 && L.ntaps <= kTcMaxTaps, "tc: bad ntaps %d", L.ntaps);
  FDX_REQUIRE(L.es == 1 || L.es == 2, "tc: bad element stride %d", L.es);
  FDX_REQUIRE(L.Ncols > 0 && L.Ncols % 32 == 0, "tc: Ncols=%d must be a multiple of 32", L.Ncols);
  FDX_REQUIRE(L.A.strides[0] == 1 && L.B.strides[0] == 1, "tc: innermost strides must be 1");

  // Few output columns (Ncols = 64 / 128): the transposed formulation (fdx_tct.cu) issues M x 256 x 16 MMAs
  // instead of 128 x Ncols x 16 ones; faster on every such layer (profiles/layers_r01_tct.txt).
  if (L.mode != TC_MNMN && !getenv("FDX_NO_TCT")) {
    const int rt = fdx_tct_launch(L, stream);
    if (rt != FDX_ERR_UNSUPPORTED) return rt;
  }
  TcDev d{};
  d.mode = L.mode;
  d.W = L.W; d.H = L.H; d.N = L.N; d.es = L.es; d.ntaps = L.ntaps;
  d.es_b = L.es_b > 1 ? L.es_b : 1;
  FDX_REQUIRE(d.es_b <= 2, "tc: bad B element stride %d", L.es_b);
  bool b_view = d.es_b != 1;
  for (int i = 0; i < kTcMaxTaps; ++i) {
    d.tap_dx[i] = L.tap_dx[i]; d.tap_dy[i] = L.tap_dy[i]; d.tap_b[i] = L.tap_b[i];
    d.tap_bdx[i] = L.tap_bdx[i]; d.tap_bdy[i] = L.tap_bdy[i];
    b_view = b_view || L.tap_bdx[i] != 0 || L.tap_bdy[i] != 0;
  }
  FDX_REQUIRE(!b_view || L.mode == TC_MNMN, "tc: strided / shifted B views exist only in TC_MNMN");
  d.K = L.K; d.M = L.M; d.Ncols = L.Ncols; d.b_batched = L.b_batched; d.mn_batched = L.mn_batched;
  d.out = L.out; d.out_f32 = L.out_f32; d.out_atomic = L.out_atomic;
  d.os_x = L.os_x; d.os_y = L.os_y; d.os_n = L.os_n; d.os_tap = L.os_tap; d.os_m = L.os_m;
  d.alpha = L.alpha; d.bias = L.bias; d.rowvec = L.rowvec; d.res = L.res;
  d.rs_x = L.rs_x; d.rs_y = L.rs_y; d.rs_n = L.rs_n;
  d.gn_ab = L.gn_ab; d.gn_ws = L.gn_ws; d.gn_slots = L.gn_slots > 0 ? L.gn_slots : 1;
  d.ws_ld = L.ws_ld > 0 ? L.ws_ld : L.Ncols;
  if (L.gn_ws && !L.gn_ab) {
    FDX_REQUIRE(L.mode == TC_KMN && !L.gemm_like && !L.out_f32 && !L.out_atomic,
                "tc: output column statistics need a bf16 convolution-forward launch");
  }
  if (L.gn_ab) {
    FDX_REQUIRE(L.mode == TC_KK && !L.gemm_like && L.res && L.gn_ws && !L.out_f32 && !L.out_atomic &&
                    !L.bias && !L.rowvec,
                "tc: GroupNorm-backward fusion needs a plain bf16 data-gradient launch");
  }

  // ---- column tile --------------------------------------------------------
  // cost model per row tile: ntiles * (BN + 64)  (MMA columns incl. padding + A re-read per tile)
  int BN = 64;
  {
    long long best = -1;
    const int cands[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
      const int bn = cands[i];
      const long long nt = (L.Ncols + bn - 1) / bn;
      const long long cost = nt * (bn + 64);
      if (best < 0 || cost < best) { best = cost; BN = bn; }
    }
  }
  const int rows_per_tile = (L.mode == TC_MNMN) ? 64 : 128;
  // ---- pixel box ----------------------------------------------------------
  int TW, TH, TN;
  if (!L.gemm_like) {
    // conv: a 16 x 8 (or 16 x 4) pixel patch; small images pack several per tile
    TW = pow2_floor(L.W < 16 ? L.W : 16);
    int rem = rows_per_tile / TW;
    TH = pow2_floor(L.H < rem ? L.H : rem);
    TN = rem / TH;
  } else {
    // GEMM: rows along x only; (y, n) are batch coordinates. A box taller than the
    // matrix is fine: TMA zero-fills and the epilogue predicates on x < W.
    TW = rows_per_tile;
    TH = 1;
    TN = 1;
  }
  d.TW = TW; d.TH = TH; d.TN = TN;
  if (L.gn_ws && TN != 1) {
    fdx_set_error("tc: fused per-image column sums need at least 128 pixels per image (got %dx%d)", L.W, L.H);
    return FDX_ERR_UNSUPPORTED;
  }
  d.nxb = (L.W + TW - 1) / TW;
  d.nyb = (L.H + TH - 1) / TH;
  d.nnb = (L.N + TN - 1) / TN;
  const long long pix_blocks = (long long)d.nxb * d.nyb * d.nnb;

  if (L.mode != TC_MNMN) {
    // Round 1 narrowed the column tile until the launch had two waves of tiles; narrower tiles re-read the A
    // operand once per column block and add rounds.  FDX_TC_BN_V1=1 restores the old rule.
    static const bool bn_v1 = getenv("FDX_TC_BN_V1") != nullptr;
    while (bn_v1 && BN > 64 && pix_blocks * ((L.Ncols + BN - 1) / BN) < 2LL * fdx_num_sms())
      BN /= 2;
    d.nblks = (L.Ncols + BN - 1) / BN;
    d.kchunks = (L.K + kBK - 1) / kBK;
    d.ntiles = (int)(pix_blocks * d.nblks);
    d.splits = 1;
    d.mblks = 1;
    d.tpp = 1;
    d.ntp = L.ntaps;
    FDX_REQUIRE(!L.res || !L.out_atomic, "tc: residual with atomic output unsupported");
  } else {
    d.nblks = (L.Ncols + BN - 1) / BN;
    d.tpp = (L.M <= 64 && L.ntaps > 1 && !b_view) ? 2 : 1;
    d.ntp = (L.ntaps + d.tpp - 1) / d.tpp;
    d.mblks = (L.M + 127) / 128;
    d.kchunks = 0;
    long long base_tiles = (long long)d.ntp * d.mblks * d.nblks;
    const long long kblocks = L.mn_batched ? d.nxb : pix_blocks;
    const long long nbz = L.mn_batched ? (long long)d.nyb * d.nnb : 1;
    int splits = L.splits;
    if (splits <= 0) {
      // wave-aware split-K: pick the split count whose tile total fills w waves of the machine
      // best (w = 1..4); more waves only when they raise the fill by > 3 %.
      const int sms = fdx_num_sms();
      const long long bt = base_tiles * nbz;
      double best_eff = -1.0;
      splits = 1;
      for (int w = 1; w <= 4; ++w) {
        long long sp = ((long long)sms * w) / bt;
        if (sp < 1) sp = 1;
        if (sp > kblocks) sp = kblocks;
        const long long tiles = bt * sp;
        const long long waves = (tiles + sms - 1) / sms;
        const double eff = (double)tiles / (double)(waves * sms);
        if (eff > best_eff + 0.03) { best_eff = eff; splits = (int)sp; }
      }
    }
    if (splits > kblocks) splits = (int)kblocks;
    FDX_REQUIRE(splits == 1 || L.out_atomic, "tc: split-K needs atomic output");
    d.splits = splits;
    d.ntiles = (int)(base_tiles * splits * nbz);
  }

  // ---- tensor maps ----------------------------------------------------------
  CUtensorMap mA, mB;
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.A.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.A.strides[i] * 2;
    uint32_t box[4] = {64, (uint32_t)(TW * L.es), (uint32_t)(TH * L.es), (uint32_t)TN};
    uint32_t est[4] = {1, (uint32_t)L.es, (uint32_t)L.es, 1};
    int s = fdx_make_tmap_bf16(&mA, L.A.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.B.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.B.strides[i] * 2;
    uint32_t box[4];
    uint32_t est[4] = {1, 1, 1, 1};
    if (L.mode == TC_KK) {
      box[0] = 64; box[1] = (uint32_t)BN; box[2] = 1; box[3] = 1;
    } else if (L.mode == TC_KMN) {
      box[0] = 64; box[1] = 64; box[2] = 1; box[3] = 1;
    } else {
      box[0] = 64; box[1] = (uint32_t)(TW * d.es_b); box[2] = (uint32_t)(TH * d.es_b); box[3] = (uint32_t)TN;
      est[1] = est[2] = (uint32_t)d.es_b;
    }
    int s = fdx_make_tmap_bf16(&mB, L.B.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }

  switch (L.mode) {
    case TC_KK: return launch_mode<TC_KK>(BN, mA, mB, d, stream);
    case TC_KMN: return launch_mode<TC_KMN>(BN, mA, mB, d, stream);
    default: return launch_mode<TC_MNMN>(BN, mA, mB, d, stream);
  }
}
