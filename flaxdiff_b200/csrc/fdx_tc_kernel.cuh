// fdx_tc_kernel.cuh -- the tap-GEMM kernel of fdx_tc.cu (design notes there).  fdx_tc.cu launches its one-source
// instantiations; fdx_tc_cat.cu instantiates the two-source A (fdx_gemm_cat) in a translation unit of its own.
#pragma once
#include "fdx_tc.cuh"
#include "fdx_epilogue.cuh"

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
  int cat_kc;              // two-source A (fdx_tc_cat.cu): k chunks [0, cat_kc) from mapA, the rest from the second map
};

// The two-source launch (fdx_tc_cat.cu): TC_KK / TC_KMN, column tile BN, second A map mA1.
int fdx_tc_cat_launch(int BN, int mode, const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mA1,
                      const TcDev& d, cudaStream_t stream);

namespace {

constexpr int kBK = 64;                 // K elements (or K rows) per pipeline stage
constexpr int kABytes = 128 * kBK * 2;  // 16 KB per stage for A in every mode

template <int BN>
struct TcCfg {
  static constexpr int kWG = (BN == 256) ? 2 : 1;   // consumer warpgroups; each owns BN / kWG columns
  static constexpr int kWN = BN / kWG;              // wgmma N
  static constexpr int kThreads = 128 * (kWG + 1);  // + the producer warpgroup (one thread issues TMA)
  // K chunks (64 deep) per pipeline stage: at BN = 64 one chunk is only 8 wgmma (two row halves x 4 K
  // steps), too little work per mbarrier round trip, so two chunks share a stage there.  The consumers always
  // issue the MMAs of kSub chunks: the missing tail chunk of an odd chunk count reads a zeroed shared-memory
  // block instead, so the MMA loop has one control path.  Not used by the MN-major-A (weight-gradient) mode.
  static constexpr int kSub = (BN == 64) ? 2 : 1;
  static constexpr int kStages = (BN == 128) ? 5 : 3;   // as many as fit in 227 KB
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kSub * (kABytes + kBBytes);
  static constexpr int kZeroBytes = (kSub > 1) ? kABytes : 0;   // zero operand block of the tail chunk
  static constexpr int kSmemBytes = kStages * kStageBytes + kZeroBytes + 1024 /*align*/ + 256 /*barriers*/ +
                                    kWG * (16384 /*epilogue staging: 4 warps x 4 KB*/ + kAccXchgBytes);
  static_assert(kSmemBytes <= 227 * 1024, "tc: shared memory");
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

// A1 = <> (every launch of fdx_tc.cu) or <CUtensorMap> (fdx_tc_cat.cu): with the second tensor map the A operand of
// TC_KK / TC_KMN has two sources.  k chunk kc < p.cat_kc is read from mapA at k = kc * 64, a later one from the second
// map at k = (kc - cat_kc) * 64.  Only the producer's choice of map differs; the MMAs, their order and the epilogue
// are the one-source kernel's, so the sum over K is the same f32 accumulation as over the concatenated matrix.  The
// empty pack leaves the one-source kernels' parameter list, and with it their code, as it was.
template <int BN, int MODE, int EPI, typename... A1>
__global__ void __launch_bounds__(TcCfg<BN>::kThreads, 1)
fdx_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
              const TcDev p, const __grid_constant__ A1... mapA1_) {
  constexpr bool CAT = sizeof...(A1) == 1;
  static_assert(!CAT || MODE != TC_MNMN, "tc: a two-source A exists only in TC_KK / TC_KMN");
  const CUtensorMap* mapA1 = nullptr;
  if constexpr (CAT) mapA1 = &(mapA1_, ...);
  using Cfg = TcCfg<BN>;
  constexpr int S = Cfg::kStages;
  constexpr int WN = Cfg::kWN;
  constexpr bool A_MN = (MODE == TC_MNMN);
  constexpr bool B_MN = (MODE != TC_KK);
  constexpr int SUB = A_MN ? 1 : Cfg::kSub;    // K chunks per stage

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* zero_blk = smem + S * Cfg::kStageBytes;                   // kZeroBytes, 1024-byte aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(zero_blk + Cfg::kZeroBytes);
  uint64_t* full = bars;            // [S]
  uint64_t* empty = bars + S;       // [S]
  uint8_t* epi_stage = zero_blk + Cfg::kZeroBytes + 256;   // kWG x 16 KB, 128-byte aligned
  float* acc_xchg = reinterpret_cast<float*>(epi_stage + Cfg::kWG * 16384);   // kWG x kAccXchgBytes

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kProducer = 4 * Cfg::kWG;

  if (warp == kProducer && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    if constexpr (CAT) tma_prefetch_desc(mapA1);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], Cfg::kWG);
    }
    fence_barrier_init();
  }
  if constexpr (Cfg::kZeroBytes > 0) {
    for (int i = threadIdx.x; i < Cfg::kZeroBytes / 16; i += blockDim.x)
      reinterpret_cast<uint4*>(zero_blk)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();       // the zeros are read by wgmma (async proxy)
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
              if constexpr (CAT) {
                const bool second = kc >= p.cat_kc;
                tma_load_4d(sa, second ? mapA1 : &mapA, &full[stage], (second ? kc - p.cat_kc : kc) * kBK,
                            x0 + p.tap_dx[t], y0 + p.tap_dy[t], n0);
              } else {
                tma_load_4d(sa, &mapA, &full[stage], kc * kBK, x0 + p.tap_dx[t], y0 + p.tap_dy[t], n0);
              }
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
          // the side input of this row: request all of its lines now (L2 prefetch), before the main loop, so
          // that the epilogue's per-chunk loads of it hit L2
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
          mbar_wait(&full[stage], phase);
          wgmma_fence();
          const uint32_t sa0 = smem_u32(smem + stage * Cfg::kStageBytes);
          const uint32_t sb0 = sa0 + SUB * kABytes + wg * WN * 128;   // this warpgroup's B columns
#pragma unroll
          for (int u = 0; u < SUB; ++u) {
            // an odd chunk count's missing tail chunk: both operands read the zero block, adding exact zeros
            const bool live = qk + u < nk;
            const uint32_t sa = live ? sa0 + u * kABytes : smem_u32(zero_blk);
            const uint32_t sb = live ? sb0 + u * Cfg::kBBytes : smem_u32(zero_blk);
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
      // Unrolled for the same reason as epilogue_bf16_coalesced: row32 then reads fixed accumulator registers.
#pragma unroll
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
            for (int j = 0; j < 8; ++j)
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(op + 4 * j), "f"(f[4 * j]),
                           "f"(f[4 * j + 1]), "f"(f[4 * j + 2]), "f"(f[4 * j + 3])
                           : "memory");
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

}  // namespace
