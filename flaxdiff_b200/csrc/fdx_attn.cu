// fdx_attn.cu -- fused scaled-dot-product attention for sm_90a: nn.dot_product_attention as used by
// NormalAttention (flaxdiff/models/attention.py:156-177, softmax(q k^T / sqrt(d)) v, self- and cross-attention
// to the 77 x 768 text context) and its backward (jax.value_and_grad, trainer/general_diffusion_trainer.py:321).
//
// As separate QK^T, softmax and PV launches, the f32 logits S and the bf16 probabilities P would round-trip HBM
// ((B, h, L, Lk): 2.1 GB + 1 GB per block at 256x256).  Here S and P never leave the SM:
//
//   forward  (one CTA per 128 queries x head x image; flash-style loop over 128-key blocks)
//     warp 4      TMA: Q tile once, K_j / V_j tiles through an mbarrier ring (128B-swizzled boxes of
//                 64 channels; a head narrower than 64 is addressed by a byte offset inside the swizzle row)
//     warps 0..3  one warpgroup: wgmma S_j = Q K_j^T into registers, then softmax with one query row per
//                 thread (WgAcc::row32), running max / sum in the log2 domain, P_j written as bf16 straight
//                 into the K-major swizzled shared-memory tile that is the A operand of the wgmma
//                 O_j = P_j V_j (fence.proxy.async), O accumulated per row with the usual exp2(m_old - m_new)
//                 correction, final O / l and the log-sum-exp row for the backward.
//   backward = two kernels with the same skeleton, S and dP recomputed on chip (FlashAttention-2 recipe,
//     7 small GEMMs instead of 5, no atomics, deterministic):
//       fdx_attn_bwd_dq   per 128-query tile, loop over key blocks:  dS = P o (dP - D) ;  dQ += dS K
//       fdx_attn_bwd_dkv  per 128-key block, loop over query tiles (transposed tiles, tile row = key):
//                         dV += P^T dO ;  dK += dS^T Q
//     with P = exp2(s * scale*log2e - lse*log2e), D = rowsum(dO o O), dS including the 1/sqrt(d) factor.
// Tensors are bf16 [B][L][heads * dh] (row stride and batch stride given), dh in {32, 64, 128, 256}; keys beyond
// Lk and query rows beyond L are handled by TMA zero fill + masking, so 77-key cross-attention needs no padded
// copies.  dh = 128 has kernels of its own (fdx_attn_fwd128_kernel, fdx_attn_bwd128_kernel: two consumer
// warpgroups of 64 rows that keep every product in its wgmma fragment, 64-row backward tiles), and so has dh = 256
// (fdx_attn_fwd256_kernel, fdx_attn_bwd256_kernel: the same design on 64-key blocks), described above them.
#include "fdx_common.cuh"
#include "../../include/fdx.h"
#include <math.h>
#include <type_traits>

namespace {

constexpr int kThreads = 160;           // forward: one consumer warpgroup + the producer warp
constexpr int kTile = 128 * 128;          // bytes of one [128 rows][64 ch] bf16 swizzled tile
constexpr int kKV = 3;                    // K/V ring stages (forward, dQ kernel)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct AttnDev {
  int B, heads, L, Lk, dh;
  float scale_log2;        // softmax scale * log2(e)
  float scale;             // softmax scale
  __nv_bfloat16* o; long long o_ld, o_bs;
  float* lse;              // [B][heads][L]
  // backward
  const __nv_bfloat16* d_o; long long do_ld, do_bs;
  const __nv_bfloat16* o_in; long long oin_ld, oin_bs;
  float* dvec;             // [B][heads][L] rowsum(dO o O)
  __nv_bfloat16* dq; long long dq_ld, dq_bs;
  __nv_bfloat16* dk; long long dk_ld, dk_bs;
  __nv_bfloat16* dv; long long dv_ld, dv_bs;
  // masked forward (fdx_attention_fwd_masked)
  const int32_t* key_mask;  // [B][Lk] 0 / 1, or NULL
  int causal;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// byte offset of the 16-byte piece (row r, piece p) inside a [rows][128 B] 128B-swizzled tile
__device__ __forceinline__ uint32_t swz(int r, int p) { return (uint32_t)(r * 128 + ((p ^ (r & 7)) << 4)); }

// store 32 consecutive bf16 (columns c0 .. c0+31 of row r) of a [128][128-key] K-major tile pair
// (two 64-key chunks of 16 KB each)
__device__ __forceinline__ void store_p_chunk(uint32_t sP, int r, int c0, const uint32_t (&w)[16]) {
  const uint32_t base = sP + (uint32_t)(c0 >> 6) * kTile;
  const int p0 = (c0 & 63) >> 3;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(base + swz(r, p0 + i)), "r"(w[4 * i]),
                 "r"(w[4 * i + 1]), "r"(w[4 * i + 2]), "r"(w[4 * i + 3])
                 : "memory");
}

// bit i set: query `qrow` may attend key key0 + i (inside the tensor, key_mask[b][key] set, and key <= qrow when
// causal).  One coalesced key-mask load per lane, then a ballot: every lane of the warp gets the whole word.
__device__ __forceinline__ uint32_t allowed_bits(const AttnDev& p, int b, int key0, int qrow, int lane) {
  const int key = key0 + lane;
  bool ok = key < p.Lk;
  if (ok && p.key_mask) ok = p.key_mask[(long long)b * p.Lk + key] != 0;
  uint32_t w = __ballot_sync(0xffffffffu, ok);
  if (p.causal) {
    const int lim = qrow - key0;                   // highest allowed bit
    w &= lim >= 31 ? 0xffffffffu : (lim < 0 ? 0u : (2u << lim) - 1u);
  }
  return w;
}

// ======================================================================================================
// forward
// ======================================================================================================
// SHORT = the keys fit one 128-key block (77 text tokens): a single K/V stage.  Otherwise a ring of NKV stages
// keeps the next key blocks in flight while the warpgroup works through the serial chain
// S_j -> softmax_j -> PV_j.
// MASKED = fdx_attention_fwd_masked: the bounds test on the last key block becomes the per-row allowed-key word of
// allowed_bits on every block; a row with no allowed key so far keeps m = -inf with corr = 1 and ends with l = 0,
// which writes zeros.
template <int DH, bool SHORT, bool MASKED = false>
__global__ void __launch_bounds__(kThreads, 1)
fdx_attn_fwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                    const __grid_constant__ CUtensorMap mapV, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  constexpr int NKV = SHORT ? 1 : kKV;               // K/V ring stages
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + kTile;                       // NKV x (K tile, V tile)
  uint8_t* sP = sKV + NKV * 2 * kTile;               // two 64-key chunks
  float* xs = reinterpret_cast<float*>(sP + 2 * kTile);   // accumulator exchange tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(xs) + kAccXchgBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;          // [NKV]
  uint64_t* kv_empty = bars + 1 + kKV;   // [NKV]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * 128;
  int nblk = (p.Lk + 127) / 128;
  if constexpr (MASKED) {
    if (p.causal && nblk > qt + 1) nblk = qt + 1;           // later key blocks lie wholly after the tile's queries
  }
  const int c0 = (head * DH) / 64 * 64;                     // first channel of the 64-wide TMA box
  const uint32_t koff = (uint32_t)((head * DH) % 64) * 2;   // byte offset of this head inside the swizzle row

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&mapQ); tma_prefetch_desc(&mapK); tma_prefetch_desc(&mapV);
    mbar_init(q_full, 1);
    for (int i = 0; i < NKV; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 1); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kTile);
      tma_load_4d(sQ, &mapQ, q_full, c0, q0, b, 0);
      for (int j = 0; j < nblk; ++j) {
        const int s = j % NKV;
        mbar_wait(&kv_empty[s], ((j / NKV) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * kTile);
        tma_load_4d(sKV + s * 2 * kTile, &mapK, &kv_full[s], c0, j * 128, b, 0);
        tma_load_4d(sKV + s * 2 * kTile + kTile, &mapV, &kv_full[s], c0, j * 128, b, 0);
      }
    }
  } else {
    const int row = warp * 32 + lane;
    const uint32_t aQ = smem_u32(sQ) + koff;
    const uint32_t sPa = smem_u32(sP);
    float m = -INFINITY, l = 0.f;
    float acc[DH];
#pragma unroll
    for (int i = 0; i < DH; ++i) acc[i] = 0.f;
    mbar_wait(q_full, 0);

    for (int j = 0; j < nblk; ++j) {
      const int s = j % NKV;
      mbar_wait(&kv_full[s], (j / NKV) & 1);
      const uint32_t aK = smem_u32(sKV + s * 2 * kTile) + koff;
      const uint32_t aV = aK + kTile;
      WgAcc<128> S;
      S.zero();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k)
        S.mma<0, 0>(gmma_desc_sw128(aQ + k * 32, 16, 1024), gmma_desc_sw128(aQ + 8192 + k * 32, 16, 1024),
                    gmma_desc_sw128(aK + k * 32, 16, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      const int kbase = j * 128;
      // pass A: row maximum over the valid keys (only the last key block can be partial)
      const bool partial = kbase + 128 > p.Lk;
      float mx = -INFINITY;
#pragma unroll 1
      for (int c = 0; c < 128; c += 32) {
        float v[32];
        S.row32(xs, 1, c, v);
        if constexpr (MASKED) {
          const uint32_t ok = allowed_bits(p, b, kbase + c, q0 + row, lane);
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if ((ok >> i) & 1u) mx = fmaxf(mx, v[i]);
        } else if (partial) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (kbase + c + i < p.Lk) mx = fmaxf(mx, v[i]);
        } else {
          float m4[4] = {mx, -INFINITY, -INFINITY, -INFINITY};        // four independent chains
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
#pragma unroll
            for (int u = 0; u < 4; ++u) m4[u] = fmaxf(m4[u], v[i + u]);
          }
          mx = fmaxf(fmaxf(m4[0], m4[1]), fmaxf(m4[2], m4[3]));
        }
      }
      const float m_new = fmaxf(m, mx * p.scale_log2);
      float corr = ex2(m - m_new);                 // first block: exp2(-inf) = 0
      if constexpr (MASKED) {
        if (m_new == -INFINITY) corr = 1.f;        // no allowed key yet: acc and l stay 0
      }
      // pass B: probabilities -> bf16 -> the swizzled A tile of the PV MMA
      float rs = 0.f;
#pragma unroll 1
      for (int c = 0; c < 128; c += 32) {
        float v[32];
        uint32_t w[16];
        S.row32(xs, 1, c, v);
        uint32_t ok = 0;
        if constexpr (MASKED) ok = allowed_bits(p, b, kbase + c, q0 + row, lane);
        float rs4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          float pe[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            pe[u] = ex2(fmaf(v[i + u], p.scale_log2, -m_new));
            if constexpr (MASKED) {
              if (!((ok >> (i + u)) & 1u)) pe[u] = 0.f;
            } else if (partial && !(kbase + c + i + u < p.Lk)) {
              pe[u] = 0.f;
            }
            rs4[u] += pe[u];
          }
          w[i >> 1] = pack_bf16x2(pe[0], pe[1]);
          w[(i >> 1) + 1] = pack_bf16x2(pe[2], pe[3]);
        }
        rs += (rs4[0] + rs4[1]) + (rs4[2] + rs4[3]);
        store_p_chunk(sPa, row, c, w);
      }
      l = fmaf(l, corr, rs);
      m = m_new;
      fence_proxy_async_smem();
      named_bar_sync(1, 128);                      // every row of P_j is in shared memory
      WgAcc<DH> O;
      O.zero();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t ap = sPa + (k >> 2) * kTile + (k & 3) * 32;
        O.mma<0, 1>(gmma_desc_sw128(ap, 16, 1024), gmma_desc_sw128(ap + 8192, 16, 1024),
                    gmma_desc_sw128(aV + k * 2048, 8192, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (threadIdx.x == 0) mbar_arrive(&kv_empty[s]);
#pragma unroll
      for (int c = 0; c < DH; c += 32) {           // acc = acc * corr + O_j
        float v[32];
        O.row32(xs, 1, c, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[c + i] = fmaf(acc[c + i], corr, v[i]);
      }
    }
    if (q0 + row < p.L) {
      float inv = 1.f / l;
      if constexpr (MASKED) {
        if (l == 0.f) inv = 0.f;                   // no allowed key: zeros
      }
      __nv_bfloat16* op = p.o + (long long)b * p.o_bs + (long long)(q0 + row) * p.o_ld + head * DH;
#pragma unroll
      for (int c = 0; c < DH; c += 8) {
        uint4 u;
        u.x = pack_bf16x2(acc[c] * inv, acc[c + 1] * inv);
        u.y = pack_bf16x2(acc[c + 2] * inv, acc[c + 3] * inv);
        u.z = pack_bf16x2(acc[c + 4] * inv, acc[c + 5] * inv);
        u.w = pack_bf16x2(acc[c + 6] * inv, acc[c + 7] * inv);
        *reinterpret_cast<uint4*>(op + c) = u;
      }
      if (p.lse) p.lse[((long long)b * p.heads + head) * p.L + q0 + row] = m * kLn2 + logf(l);
    }
  }
}

// ======================================================================================================
// backward, part 0: D[b][h][row] = sum_c dO[row][c] * O[row][c]
// ======================================================================================================
__global__ void attn_dvec_kernel(const AttnDev p) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // (b, row, head)
  const long long total = (long long)p.B * p.L * p.heads;
  if (idx >= total) return;
  const int head = (int)(idx % p.heads);
  const long long r = idx / p.heads;
  const int row = (int)(r % p.L), b = (int)(r / p.L);
  const __nv_bfloat16* a = p.d_o + (long long)b * p.do_bs + (long long)row * p.do_ld + head * p.dh;
  const __nv_bfloat16* o = p.o_in + (long long)b * p.oin_bs + (long long)row * p.oin_ld + head * p.dh;
  float s = 0.f;
  for (int c = 0; c < p.dh; c += 8) {
    const uint4 ua = *reinterpret_cast<const uint4*>(a + c), uo = *reinterpret_cast<const uint4*>(o + c);
    const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wo[4] = {uo.x, uo.y, uo.z, uo.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fa = unpack_bf16x2(wa[i]), fo = unpack_bf16x2(wo[i]);
      s = fmaf(fa.x, fo.x, s);
      s = fmaf(fa.y, fo.y, s);
    }
  }
  p.dvec[((long long)b * p.heads + head) * p.L + row] = s;
}

// ======================================================================================================
// backward, shared skeleton.  ROWS_ARE_KEYS = false: the dQ kernel (tile rows = queries, loop over key blocks);
// true: the dK / dV kernel (tile rows = keys, loop over query tiles).  Per loop step two 128 x 128 products are
// computed by two warpgroups, each owning 64 of the columns: S (or S^T) and dP (or dP^T) in registers.  Each
// warpgroup turns its columns into the bf16 tiles E1 = P (only needed for dV) and E2 = dS in shared memory, and
// once both halves are published the accumulating products run on the whole tiles:
//   dQ  += dS  . K_j                (warpgroup 0)                          [ROWS_ARE_KEYS = false]
//   dV  += P^T . dO_i  (warpgroup 0),  dK += dS^T . Q_i  (warpgroup 1)     [ROWS_ARE_KEYS = true]
// with the accumulators in registers across the whole loop (no rescaling: P is recomputed from the saved
// log-sum-exp).  Shared memory: R1, R2 = the two row-side operands (Q, dO | K, V), ring of (C1, C2) = the
// column-side pair (K_j, V_j | Q_i, dO_i), E1 / E2 tiles of 2 x 16 KB each.
// ======================================================================================================
constexpr int kBwdThreads = 3 * 128;   // two consumer warpgroups + the producer warpgroup (one thread issues TMA)

template <int DH, bool ROWS_ARE_KEYS>
__global__ void __launch_bounds__(kBwdThreads, 1)
fdx_attn_bwd_kernel(const __grid_constant__ CUtensorMap mapR1, const __grid_constant__ CUtensorMap mapR2,
                    const __grid_constant__ CUtensorMap mapC1, const __grid_constant__ CUtensorMap mapC2,
                    const AttnDev p) {
  constexpr int RING = 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sR1 = smem;
  uint8_t* sR2 = smem + kTile;
  uint8_t* sC = smem + 2 * kTile;                      // RING x (C1, C2)
  uint8_t* sE1 = sC + RING * 2 * kTile;                // 2 chunks
  uint8_t* sE2 = sE1 + 2 * kTile;                      // 2 chunks
  float* sStat = reinterpret_cast<float*>(sE2 + 2 * kTile);     // RING x (lse[128], dvec[128]) of the column side
  float* sX = sStat + RING * 256;                      // 2 x accumulator exchange tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sX) + 2 * kAccXchgBytes);
  uint64_t* r_full = bars;
  uint64_t* c_full = bars + 1;            // [RING]
  uint64_t* c_empty = c_full + RING;      // [RING]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int r0 = rt * 128;
  const int nrows = ROWS_ARE_KEYS ? p.Lk : p.L;        // extent of the row side
  const int ncols = ROWS_ARE_KEYS ? p.L : p.Lk;        // extent of the looped (column) side
  const int nstep = (ncols + 127) / 128;
  const int c0 = (head * DH) / 64 * 64;
  const uint32_t koff = (uint32_t)((head * DH) % 64) * 2;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapR1); tma_prefetch_desc(&mapR2); tma_prefetch_desc(&mapC1); tma_prefetch_desc(&mapC2);
    mbar_init(r_full, 1);
    for (int i = 0; i < RING; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  if (warp >= 8) producer_regs(); else consumer_regs();

  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(r_full, 2 * kTile);
      tma_load_4d(sR1, &mapR1, r_full, c0, r0, b, 0);
      tma_load_4d(sR2, &mapR2, r_full, c0, r0, b, 0);
      for (int j = 0; j < nstep; ++j) {
        const int s = j % RING;
        mbar_wait(&c_empty[s], ((j / RING) & 1) ^ 1);
        mbar_arrive_expect_tx(&c_full[s], 2 * kTile);
        tma_load_4d(sC + s * 2 * kTile, &mapC1, &c_full[s], c0, j * 128, b, 0);
        tma_load_4d(sC + s * 2 * kTile + kTile, &mapC2, &c_full[s], c0, j * 128, b, 0);
      }
    }
  } else {
    const int wg = warp >> 2;                          // columns [64 wg, 64 wg + 64) of S / dP
    constexpr int CW = 64;
    const int row = (warp & 3) * 32 + lane;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float* xs = sX + wg * (kAccXchgBytes / 4);
    const int xbar = 2 + wg;
    const long long stat_base = ((long long)b * p.heads + head) * p.L;
    // dQ kernel: this thread's query row statistics; dK/dV kernel: they belong to the COLUMNS (queries)
    float lse_r = 0.f, d_r = 0.f;
    if constexpr (!ROWS_ARE_KEYS) {
      if (r0 + row < p.L) {
        lse_r = p.lse[stat_base + r0 + row] * kLog2e;
        d_r = p.dvec[stat_base + r0 + row] * p.scale;
      }
    }
    const uint32_t aR1 = smem_u32(sR1) + koff, aR2 = smem_u32(sR2) + koff;
    const uint32_t sE1a = smem_u32(sE1), sE2a = smem_u32(sE2);
    WgAcc<DH> A;                                       // dQ | dV (warpgroup 0) or dK (warpgroup 1)
    A.zero();
    mbar_wait(r_full, 0);
    for (int j = 0; j < nstep; ++j) {
      const int s = j % RING;
      const int cbase = j * 128;
      if constexpr (ROWS_ARE_KEYS) {
        // stage the query-side statistics of this step (parity buffer j & 1), 128 threads = 128 columns
        if (wg == 0) {
          float* st = sStat + (j & 1) * 256;
          const bool ok = cbase + row < p.L;
          st[row] = ok ? p.lse[stat_base + cbase + row] * kLog2e : 0.f;
          st[128 + row] = ok ? p.dvec[stat_base + cbase + row] * p.scale : 0.f;
        }
      }
      mbar_wait(&c_full[s], (j / RING) & 1);
      const uint32_t aC1 = smem_u32(sC + s * 2 * kTile) + koff, aC2 = aC1 + kTile;
      // S (or S^T) = R1 . C1^T ;  dP (or dP^T) = R2 . C2^T  - this warpgroup's 64 columns
      WgAcc<64> Sa, Pa;
      Sa.zero();
      Pa.zero();
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < DH / 16; ++k) {
        Sa.mma<0, 0>(gmma_desc_sw128(aR1 + k * 32, 16, 1024), gmma_desc_sw128(aR1 + 8192 + k * 32, 16, 1024),
                     gmma_desc_sw128(aC1 + wg * 8192 + k * 32, 16, 1024));
        Pa.mma<0, 0>(gmma_desc_sw128(aR2 + k * 32, 16, 1024), gmma_desc_sw128(aR2 + 8192 + k * 32, 16, 1024),
                     gmma_desc_sw128(aC2 + wg * 8192 + k * 32, 16, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();
      // the statistics are staged and the previous step's accumulation has consumed E1 / E2
      named_bar_sync(1, 256);
      const float* st = sStat + (j & 1) * 256;
      const bool row_in = ROWS_ARE_KEYS ? (r0 + row < p.Lk) : (r0 + row < p.L);
      const int col_lim = (ROWS_ARE_KEYS ? p.L : p.Lk) - cbase;      // columns of this step inside the tensor
      // P = exp2(s * scale*log2e - lse*log2e);  dS = P * (dP * scale - D * scale)  (D * scale staged / hoisted).
      // Only the last step / the last row tile needs the bounds masks: MASK = false is the 5-instruction path.
      auto ewise = [&](auto mask_tag) {
        constexpr bool MASK = decltype(mask_tag)::value;
#pragma unroll 1
        for (int cl = 0; cl < CW; cl += 32) {
          const int c = wg * CW + cl;
          float vs[32], vp[32];
          uint32_t w1[16], w2[16];
          Sa.row32(xs, xbar, cl, vs);
          Pa.row32(xs, xbar, cl, vp);
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            float lq[4] = {lse_r, lse_r, lse_r, lse_r}, dq4[4] = {d_r, d_r, d_r, d_r};
            if constexpr (ROWS_ARE_KEYS) {
              const float4 a4 = *reinterpret_cast<const float4*>(st + c + i);
              const float4 b4 = *reinterpret_cast<const float4*>(st + 128 + c + i);
              lq[0] = a4.x; lq[1] = a4.y; lq[2] = a4.z; lq[3] = a4.w;
              dq4[0] = b4.x; dq4[1] = b4.y; dq4[2] = b4.z; dq4[3] = b4.w;
            }
            float pr[4], ds[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              float pv = ex2(fmaf(vs[i + u], p.scale_log2, -lq[u]));
              if (MASK && !(row_in && (c + i + u < col_lim))) pv = 0.f;
              pr[u] = pv;
              ds[u] = pv * fmaf(vp[i + u], p.scale, -dq4[u]);
            }
            w1[i >> 1] = pack_bf16x2(pr[0], pr[1]);
            w1[(i >> 1) + 1] = pack_bf16x2(pr[2], pr[3]);
            w2[i >> 1] = pack_bf16x2(ds[0], ds[1]);
            w2[(i >> 1) + 1] = pack_bf16x2(ds[2], ds[3]);
          }
          if constexpr (ROWS_ARE_KEYS) store_p_chunk(sE1a, row, c, w1);
          store_p_chunk(sE2a, row, c, w2);
        }
      };
      // warpgroup-uniform choice (row32 synchronises the warpgroup)
      const bool need_mask = r0 + 128 > nrows || col_lim < 128;
      if (need_mask) ewise(std::true_type{}); else ewise(std::false_type{});
      fence_proxy_async_smem();
      named_bar_sync(1, 256);                          // both halves of E1 / E2 are published
      if (ROWS_ARE_KEYS || wg == 0) {
        // dV += P^T . dO_i (B = C2, MN-major) | dK += dS^T . Q_i (B = C1) | dQ += dS . K_j (B = C1)
        const uint32_t aE = (ROWS_ARE_KEYS && wg == 0) ? sE1a : sE2a;
        const uint32_t aB = (ROWS_ARE_KEYS && wg == 0) ? aC2 : aC1;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t eo = aE + (uint32_t)((k >> 2) * kTile + (k & 3) * 32);
          A.mma<0, 1>(gmma_desc_sw128(eo, 16, 1024), gmma_desc_sw128(eo + 8192, 16, 1024),
                      gmma_desc_sw128(aB + k * 2048, 8192, 1024));
        }
        wgmma_commit();
        wgmma_wait<0>();
      }
      if (wg_leader) mbar_arrive(&c_empty[s]);
    }
    // epilogue: accumulator rows -> bf16
    if (ROWS_ARE_KEYS || wg == 0) {
      const bool row_ok = r0 + row < nrows;
      __nv_bfloat16* base;
      if constexpr (ROWS_ARE_KEYS)
        base = wg == 0 ? p.dv + (long long)b * p.dv_bs + (long long)(r0 + row) * p.dv_ld
                       : p.dk + (long long)b * p.dk_bs + (long long)(r0 + row) * p.dk_ld;
      else
        base = p.dq + (long long)b * p.dq_bs + (long long)(r0 + row) * p.dq_ld;
      base += head * DH;
#pragma unroll
      for (int c = 0; c < DH; c += 32) {
        float v[32];
        A.row32(xs, xbar, c, v);
        if (row_ok) {
#pragma unroll
          for (int i = 0; i < 32; i += 8) {
            uint4 u;
            u.x = pack_bf16x2(v[i], v[i + 1]);
            u.y = pack_bf16x2(v[i + 2], v[i + 3]);
            u.z = pack_bf16x2(v[i + 4], v[i + 5]);
            u.w = pack_bf16x2(v[i + 6], v[i + 7]);
            *reinterpret_cast<uint4*>(base + c + i) = u;
          }
        }
      }
    }
  }
}

// ======================================================================================================
// head width 128.  The kernels above hold 128-row products per warpgroup and hand their rows out through the
// exchange tile; at 128 channels those products no longer fit the register file next to the accumulators.
// These kernels keep every product in its wgmma fragment: thread l of warp w of a warpgroup owns rows
// 16 w + l/4 (h = 0) and 16 w + l/4 + 8 (h = 1) of the 64-row fragment and, for g = 0 .. N/8 - 1, columns
// 8 g + 2 (l % 4) + e (e = 0, 1) in element 4 g + 2 h + e.  Row reductions run over the four lanes of a quad.
// A 128-channel tile is two 64-channel chunks (two TMA boxes); 128 channels start on a chunk boundary, so the
// in-row byte offset of the narrower kernels is always 0 here.
// ======================================================================================================
constexpr int kWTile = 2 * kTile;                // [128 rows][128 ch] bf16: two [128][64] chunks
constexpr int kFwd128Threads = 2 * 128 + 32;     // two consumer warpgroups + the producer warp

// one bf16 pair (row r, columns col, col + 1) into a [rows][64 col] K-major 128B-swizzled chunk; a quad's four
// lanes fill one 16-byte piece and the eight quads of a warp hit eight different pieces: no bank conflicts
__device__ __forceinline__ void st_frag_pair(uint32_t chunk, int r, int col, uint32_t w) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(chunk + swz(r, col >> 3) + (col & 7) * 2), "r"(w) : "memory");
}

// forward, 128 queries per CTA: warpgroup wg owns query rows [64 wg, 64 wg + 64).  Per key block S = Q K_j^T
// is one m64n128 fragment (64 registers), O one more; P_j goes through the warpgroup's own [64][128] bf16 tile.
// Shared memory: Q 32 KB, NKV x (K, V) 64 KB, P 2 x 16 KB.
template <bool SHORT>
__global__ void __launch_bounds__(kFwd128Threads, 1)
fdx_attn_fwd128_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                       const __grid_constant__ CUtensorMap mapV, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  constexpr int NKV = SHORT ? 1 : 2;
  uint8_t* sQ = smem;                                 // [2 chunks][128 queries][64 ch]
  uint8_t* sKV = smem + kWTile;                       // NKV x (K, V), each [2 chunks][128 keys][64 ch]
  uint8_t* sP = sKV + NKV * 2 * kWTile;               // per warpgroup [2 chunks][64 queries][64 keys]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + kWTile);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;          // [NKV]
  uint64_t* kv_empty = bars + 3;         // [NKV]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * 128;
  const int nblk = (p.Lk + 127) / 128;
  const int c0 = head * 128;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapQ); tma_prefetch_desc(&mapK); tma_prefetch_desc(&mapV);
    mbar_init(q_full, 1);
    for (int i = 0; i < NKV; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kWTile);
      tma_load_4d(sQ, &mapQ, q_full, c0, q0, b, 0);
      tma_load_4d(sQ + kTile, &mapQ, q_full, c0 + 64, q0, b, 0);
      for (int j = 0; j < nblk; ++j) {
        const int s = j % NKV;
        uint8_t* kv = sKV + s * 2 * kWTile;
        mbar_wait(&kv_empty[s], ((j / NKV) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * kWTile);
        tma_load_4d(kv, &mapK, &kv_full[s], c0, j * 128, b, 0);
        tma_load_4d(kv + kTile, &mapK, &kv_full[s], c0 + 64, j * 128, b, 0);
        tma_load_4d(kv + kWTile, &mapV, &kv_full[s], c0, j * 128, b, 0);
        tma_load_4d(kv + kWTile + kTile, &mapV, &kv_full[s], c0 + 64, j * 128, b, 0);
      }
    }
  } else {
    const int wg = warp >> 2;
    const int rq = (warp & 3) * 16 + (lane >> 2);      // fragment rows rq, rq + 8 of this warpgroup's 64
    const int cq = 2 * (lane & 3);                     // fragment column offset inside each 8-column group
    const uint32_t aQ = smem_u32(sQ) + wg * 8192;
    const uint32_t aP = smem_u32(sP) + wg * kTile;
    float m[2] = {-INFINITY, -INFINITY};               // running row maxima (log2 domain, scaled)
    float l[2] = {0.f, 0.f};                           // running row sums over this thread's columns
    float O[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) O[i] = 0.f;
    mbar_wait(q_full, 0);

    for (int j = 0; j < nblk; ++j) {
      const int s = j % NKV;
      mbar_wait(&kv_full[s], (j / NKV) & 1);
      const uint32_t aK = smem_u32(sKV + s * 2 * kWTile), aV = aK + kWTile;
      float S[64];                                     // the first K step overwrites it (scale_d = 0)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t ko = (uint32_t)((k >> 2) * kTile + (k & 3) * 32);
        wgmma_m64n128k16<0, 0>(S, gmma_desc_sw128(aQ + ko, 16, 1024), gmma_desc_sw128(aK + ko, 16, 1024), k > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // keys beyond Lk (TMA zero fill; only the last block can be partial) drop out as -inf logits
      const int kvalid = p.Lk - j * 128;
      if (kvalid < 128) {
#pragma unroll
        for (int g = 0; g < 16; ++g)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * g + cq + e >= kvalid) S[4 * g + e] = S[4 * g + 2 + e] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int g = 0; g < 16; ++g)
#pragma unroll
        for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], fmaxf(S[4 * g + 2 * h], S[4 * g + 2 * h + 1]));
      float corr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float m_new = fmaxf(m[h], mx[h] * p.scale_log2);
        corr[h] = ex2(m[h] - m_new);                   // first block: exp2(-inf) = 0
        m[h] = m_new;
      }
      // probabilities -> bf16 -> the K-major swizzled A tile of the PV MMA
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        float pe[4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            pe[2 * h + e] = ex2(fmaf(S[4 * g + 2 * h + e], p.scale_log2, -m[h]));
            rs[h] += pe[2 * h + e];
          }
        const uint32_t chunk = aP + (uint32_t)(g >> 3) * 8192;
        st_frag_pair(chunk, rq, (g & 7) * 8 + cq, pack_bf16x2(pe[0], pe[1]));
        st_frag_pair(chunk, rq + 8, (g & 7) * 8 + cq, pack_bf16x2(pe[2], pe[3]));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l[h] = fmaf(l[h], corr[h], rs[h]);
#pragma unroll
      for (int g = 0; g < 16; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) O[4 * g + i] *= corr[i >> 1];
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);                     // every row of this warpgroup's P_j is in shared memory
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k)                      // B = V_j, MN-major: 64-channel chunks kTile apart
        wgmma_m64n128k16<0, 1>(O, gmma_desc_sw128(aP + (k >> 2) * 8192 + (k & 3) * 32, 16, 1024),
                               gmma_desc_sw128(aV + k * 2048, kTile, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[s]);
    }
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      inv[h] = 1.f / l[h];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = q0 + wg * 64 + rq + 8 * h;
      if (row < p.L) {
        __nv_bfloat16* op = p.o + (long long)b * p.o_bs + (long long)row * p.o_ld + c0 + cq;
#pragma unroll
        for (int g = 0; g < 16; ++g)
          *reinterpret_cast<uint32_t*>(op + 8 * g) = pack_bf16x2(O[4 * g + 2 * h] * inv[h], O[4 * g + 2 * h + 1] * inv[h]);
        if (p.lse && (lane & 3) == 0) p.lse[((long long)b * p.heads + head) * p.L + row] = m[h] * kLn2 + logf(l[h]);
      }
    }
  }
}

// backward at head width 128: the skeleton of fdx_attn_bwd_kernel on 64-row tiles.  Per loop step each
// warpgroup computes 64 of the 128 columns of S and dP (m64n64, 32 + 32 registers) and writes its half of
// E1 = P and E2 = dS; then
//   dQ[:, 64 wg .. +64] += dS . K_j[:, 64 wg .. +64]   (m64n64 per warpgroup)         [ROWS_ARE_KEYS = false]
//   dV += P^T . dO_i (warpgroup 0),  dK += dS^T . Q_i (warpgroup 1)   (m64n128)        [ROWS_ARE_KEYS = true]
// Shared memory: R1, R2 2 x 16 KB, a ring of 2 x (C1, C2) 2 x 64 KB, E1, E2 2 x 16 KB.
template <bool ROWS_ARE_KEYS>
__global__ void __launch_bounds__(kBwdThreads, 1)
fdx_attn_bwd128_kernel(const __grid_constant__ CUtensorMap mapR1, const __grid_constant__ CUtensorMap mapR2,
                       const __grid_constant__ CUtensorMap mapC1, const __grid_constant__ CUtensorMap mapC2,
                       const AttnDev p) {
  constexpr int RING = 2;
  constexpr int AN = ROWS_ARE_KEYS ? 128 : 64;         // accumulator columns per warpgroup
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sR1 = smem;                                 // [2 chunks][64 rows][64 ch]
  uint8_t* sR2 = smem + kTile;
  uint8_t* sC = smem + 2 * kTile;                      // RING x (C1, C2), each [2 chunks][128 rows][64 ch]
  uint8_t* sE1 = sC + RING * 2 * kWTile;               // [2 chunks][64 rows][64 columns]
  uint8_t* sE2 = sE1 + kTile;
  float* sStat = reinterpret_cast<float*>(sE2 + kTile);          // RING x (lse[128], dvec[128]) of the columns
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStat + RING * 256);
  uint64_t* r_full = bars;
  uint64_t* c_full = bars + 1;            // [RING]
  uint64_t* c_empty = c_full + RING;      // [RING]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, b = blockIdx.z;
  const int r0 = blockIdx.x * 64;
  const int nrows = ROWS_ARE_KEYS ? p.Lk : p.L;
  const int ncols = ROWS_ARE_KEYS ? p.L : p.Lk;
  const int nstep = (ncols + 127) / 128;
  const int c0 = head * 128;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapR1); tma_prefetch_desc(&mapR2); tma_prefetch_desc(&mapC1); tma_prefetch_desc(&mapC2);
    mbar_init(r_full, 1);
    for (int i = 0; i < RING; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // setmaxnreg sits inside each role's branch: issued before code both roles run, ptxas ignores it (C7507)
  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(r_full, 2 * kTile);
      tma_load_4d(sR1, &mapR1, r_full, c0, r0, b, 0);
      tma_load_4d(sR1 + 8192, &mapR1, r_full, c0 + 64, r0, b, 0);
      tma_load_4d(sR2, &mapR2, r_full, c0, r0, b, 0);
      tma_load_4d(sR2 + 8192, &mapR2, r_full, c0 + 64, r0, b, 0);
      for (int j = 0; j < nstep; ++j) {
        const int s = j % RING;
        uint8_t* c = sC + s * 2 * kWTile;
        mbar_wait(&c_empty[s], ((j / RING) & 1) ^ 1);
        mbar_arrive_expect_tx(&c_full[s], 2 * kWTile);
        tma_load_4d(c, &mapC1, &c_full[s], c0, j * 128, b, 0);
        tma_load_4d(c + kTile, &mapC1, &c_full[s], c0 + 64, j * 128, b, 0);
        tma_load_4d(c + kWTile, &mapC2, &c_full[s], c0, j * 128, b, 0);
        tma_load_4d(c + kWTile + kTile, &mapC2, &c_full[s], c0 + 64, j * 128, b, 0);
      }
    }
  } else {
    consumer_regs();
    const int wg = warp >> 2;                          // columns [64 wg, 64 wg + 64) of S / dP
    const int rq = (warp & 3) * 16 + (lane >> 2);      // fragment rows rq, rq + 8
    const int cq = 2 * (lane & 3);
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const long long stat_base = ((long long)b * p.heads + head) * p.L;
    const bool row_in[2] = {r0 + rq < nrows, r0 + rq + 8 < nrows};
    // dQ kernel: the statistics of this thread's two query rows; dK/dV kernel: they belong to the COLUMNS
    float lse_r[2] = {0.f, 0.f}, d_r[2] = {0.f, 0.f};
    if constexpr (!ROWS_ARE_KEYS) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (row_in[h]) {
          lse_r[h] = p.lse[stat_base + r0 + rq + 8 * h] * kLog2e;
          d_r[h] = p.dvec[stat_base + r0 + rq + 8 * h] * p.scale;
        }
    }
    const uint32_t aR1 = smem_u32(sR1), aR2 = smem_u32(sR2);
    const uint32_t aE1 = smem_u32(sE1), aE2 = smem_u32(sE2);
    float A[AN / 2];                                   // dQ half | dV (warpgroup 0) or dK (warpgroup 1)
#pragma unroll
    for (int i = 0; i < AN / 2; ++i) A[i] = 0.f;
    mbar_wait(r_full, 0);
    for (int j = 0; j < nstep; ++j) {
      const int s = j % RING;
      const int cbase = j * 128;
      if constexpr (ROWS_ARE_KEYS) {
        // stage the query-side statistics of this step (parity buffer j & 1), 128 threads = 128 columns
        if (wg == 0) {
          float* st = sStat + (j & 1) * 256;
          const int t = threadIdx.x;
          const bool ok = cbase + t < p.L;
          st[t] = ok ? p.lse[stat_base + cbase + t] * kLog2e : 0.f;
          st[128 + t] = ok ? p.dvec[stat_base + cbase + t] * p.scale : 0.f;
        }
      }
      mbar_wait(&c_full[s], (j / RING) & 1);
      const uint32_t aC1 = smem_u32(sC + s * 2 * kWTile), aC2 = aC1 + kWTile;
      // S (or S^T) = R1 . C1^T ;  dP (or dP^T) = R2 . C2^T  - this warpgroup's 64 columns
      float Sa[32], Pa[32];                            // the first K step overwrites them (scale_d = 0)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t ro = (uint32_t)((k >> 2) * 8192 + (k & 3) * 32);
        const uint32_t co = (uint32_t)((k >> 2) * kTile + wg * 8192 + (k & 3) * 32);
        wgmma_m64n64k16<0, 0>(Sa, gmma_desc_sw128(aR1 + ro, 16, 1024), gmma_desc_sw128(aC1 + co, 16, 1024), k > 0);
        wgmma_m64n64k16<0, 0>(Pa, gmma_desc_sw128(aR2 + ro, 16, 1024), gmma_desc_sw128(aC2 + co, 16, 1024), k > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // the statistics are staged and the previous step's accumulation has consumed E1 / E2
      named_bar_sync(1, 256);
      const float* st = sStat + (j & 1) * 256;
      // rows / columns outside the tensors (TMA zero fill; only the last row tile or step) drop out as -inf
      // logits: P = 0 and dS = 0 there
      const int col_lim = ncols - cbase - wg * 64;     // columns of this warpgroup inside the tensor
      if (r0 + 64 > nrows || col_lim < 64) {
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (!(row_in[h] && 8 * g + cq + e < col_lim)) Sa[4 * g + 2 * h + e] = -INFINITY;
      }
      // P = exp2(s * scale*log2e - lse*log2e);  dS = P * (dP * scale - D * scale)
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const int cl = 8 * g + cq;                     // column inside this warpgroup's 64
        float lq[2][2], dq[2][2];                      // [h][e]
        if constexpr (ROWS_ARE_KEYS) {
          const float2 a2 = *reinterpret_cast<const float2*>(st + wg * 64 + cl);
          const float2 b2 = *reinterpret_cast<const float2*>(st + 128 + wg * 64 + cl);
#pragma unroll
          for (int h = 0; h < 2; ++h) { lq[h][0] = a2.x; lq[h][1] = a2.y; dq[h][0] = b2.x; dq[h][1] = b2.y; }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) { lq[h][0] = lq[h][1] = lse_r[h]; dq[h][0] = dq[h][1] = d_r[h]; }
        }
        float pr[4], ds[4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * g + 2 * h + e;
            pr[2 * h + e] = ex2(fmaf(Sa[i], p.scale_log2, -lq[h][e]));
            ds[2 * h + e] = pr[2 * h + e] * fmaf(Pa[i], p.scale, -dq[h][e]);
          }
        if constexpr (ROWS_ARE_KEYS) {
          st_frag_pair(aE1 + wg * 8192, rq, cl, pack_bf16x2(pr[0], pr[1]));
          st_frag_pair(aE1 + wg * 8192, rq + 8, cl, pack_bf16x2(pr[2], pr[3]));
        }
        st_frag_pair(aE2 + wg * 8192, rq, cl, pack_bf16x2(ds[0], ds[1]));
        st_frag_pair(aE2 + wg * 8192, rq + 8, cl, pack_bf16x2(ds[2], ds[3]));
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 256);                          // both halves of E1 / E2 are published
      wgmma_fence();
      if constexpr (ROWS_ARE_KEYS) {
        // dV += P^T . dO_i (warpgroup 0) | dK += dS^T . Q_i (warpgroup 1); B MN-major, chunks kTile apart
        const uint32_t aE = wg == 0 ? aE1 : aE2;
        const uint32_t aB = wg == 0 ? aC2 : aC1;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          wgmma_m64n128k16<0, 1>(A, gmma_desc_sw128(aE + (k >> 2) * 8192 + (k & 3) * 32, 16, 1024),
                                 gmma_desc_sw128(aB + k * 2048, kTile, 1024));
      } else {
        // dQ[:, 64 wg ..] += dS . K_j[:, 64 wg ..]: B = channel chunk wg of K_j
#pragma unroll
        for (int k = 0; k < 8; ++k)
          wgmma_m64n64k16<0, 1>(A, gmma_desc_sw128(aE2 + (k >> 2) * 8192 + (k & 3) * 32, 16, 1024),
                                gmma_desc_sw128(aC1 + wg * kTile + k * 2048, kTile, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (wg_leader) mbar_arrive(&c_empty[s]);
    }
    // epilogue: fragment rows -> bf16
    __nv_bfloat16* base;
    long long ld;
    if constexpr (ROWS_ARE_KEYS) {
      base = wg == 0 ? p.dv + (long long)b * p.dv_bs : p.dk + (long long)b * p.dk_bs;
      ld = wg == 0 ? p.dv_ld : p.dk_ld;
      base += c0 + cq;
    } else {
      base = p.dq + (long long)b * p.dq_bs + c0 + wg * 64 + cq;
      ld = p.dq_ld;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (row_in[h]) {
        __nv_bfloat16* rp = base + (long long)(r0 + rq + 8 * h) * ld;
#pragma unroll
        for (int g = 0; g < AN / 8; ++g)
          *reinterpret_cast<uint32_t*>(rp + 8 * g) = pack_bf16x2(A[4 * g + 2 * h], A[4 * g + 2 * h + 1]);
      }
    }
  }
}

// ======================================================================================================
// head width 256.  The width-128 design with the key / column side cut to 64-row blocks: a 256-channel operand
// is four 64-channel chunks (four TMA boxes), and a [128 keys][256 ch] K or V tile alone would take 64 KB.
// Fragment layout, quad reductions and the P / dS tiles as above; every chunk of a 64-row operand is
// [64 rows][64 ch] = 8 KB, so the MN-major B operands advance 8 KB per 64 channels.
// ======================================================================================================
constexpr int kChunk64 = 64 * 128;               // bytes of one [64 rows][64 ch] bf16 swizzled chunk
constexpr int kOp256 = 4 * kChunk64;             // [64 rows][256 ch]: 32 KB

// forward, 128 queries per CTA: warpgroup wg owns query rows [64 wg, 64 wg + 64); per 64-key block S = Q K_j^T is
// one m64n64 fragment (32 registers) and O one m64n256 fragment (128 registers); P_j goes through the
// warpgroup's own [64][64] bf16 tile.  Shared memory: Q 64 KB, 2 x (K, V) 128 KB, P 2 x 8 KB.
// SHORT (<= 128 keys): both key blocks are loaded once behind one barrier; otherwise the two stages are a ring.
template <bool SHORT>
__global__ void __launch_bounds__(kBwdThreads, 1)
fdx_attn_fwd256_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                       const __grid_constant__ CUtensorMap mapV, const AttnDev p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  constexpr int NKV = 2;
  uint8_t* sQ = smem;                                 // [4 chunks][128 queries][64 ch]
  uint8_t* sKV = smem + 4 * kTile;                    // NKV x (K, V), each [4 chunks][64 keys][64 ch]
  uint8_t* sP = sKV + NKV * 2 * kOp256;               // per warpgroup [64 queries][64 keys]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 2 * kChunk64);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;          // [NKV]
  uint64_t* kv_empty = bars + 3;         // [NKV]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * 128;
  const int nblk = (p.Lk + 63) / 64;
  const int c0 = head * 256;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapQ); tma_prefetch_desc(&mapK); tma_prefetch_desc(&mapV);
    mbar_init(q_full, 1);
    for (int i = 0; i < NKV; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // setmaxnreg sits inside each role's branch: issued before code both roles run, ptxas ignores it (C7507)
  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(q_full, 4 * kTile);
      for (int c = 0; c < 4; ++c) tma_load_4d(sQ + c * kTile, &mapQ, q_full, c0 + 64 * c, q0, b, 0);
      if constexpr (SHORT) {
        mbar_arrive_expect_tx(&kv_full[0], nblk * 2 * kOp256);
      }
      for (int j = 0; j < nblk; ++j) {
        const int s = j % NKV;
        uint8_t* kv = sKV + s * 2 * kOp256;
        uint64_t* full = &kv_full[SHORT ? 0 : s];
        if constexpr (!SHORT) {
          mbar_wait(&kv_empty[s], ((j / NKV) & 1) ^ 1);
          mbar_arrive_expect_tx(full, 2 * kOp256);
        }
        for (int c = 0; c < 4; ++c) {
          tma_load_4d(kv + c * kChunk64, &mapK, full, c0 + 64 * c, j * 64, b, 0);
          tma_load_4d(kv + kOp256 + c * kChunk64, &mapV, full, c0 + 64 * c, j * 64, b, 0);
        }
      }
    }
  } else {
    consumer_regs();
    const int wg = warp >> 2;
    const int rq = (warp & 3) * 16 + (lane >> 2);      // fragment rows rq, rq + 8 of this warpgroup's 64
    const int cq = 2 * (lane & 3);                     // fragment column offset inside each 8-column group
    const uint32_t aQ = smem_u32(sQ) + wg * 8192;
    const uint32_t aP = smem_u32(sP) + wg * kChunk64;
    float m[2] = {-INFINITY, -INFINITY};               // running row maxima (log2 domain, scaled)
    float l[2] = {0.f, 0.f};                           // running row sums over this thread's columns
    float O[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) O[i] = 0.f;
    mbar_wait(q_full, 0);
    if constexpr (SHORT) mbar_wait(&kv_full[0], 0);

    for (int j = 0; j < nblk; ++j) {
      const int s = j % NKV;
      if constexpr (!SHORT) mbar_wait(&kv_full[s], (j / NKV) & 1);
      const uint32_t aK = smem_u32(sKV + s * 2 * kOp256), aV = aK + kOp256;
      float S[32];                                     // the first K step overwrites it (scale_d = 0)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t kc = (uint32_t)(k & 3) * 32;
        wgmma_m64n64k16<0, 0>(S, gmma_desc_sw128(aQ + (k >> 2) * kTile + kc, 16, 1024),
                              gmma_desc_sw128(aK + (k >> 2) * kChunk64 + kc, 16, 1024), k > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // keys beyond Lk (TMA zero fill; only the last block can be partial) drop out as -inf logits
      const int kvalid = p.Lk - j * 64;
      if (kvalid < 64) {
#pragma unroll
        for (int g = 0; g < 8; ++g)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * g + cq + e >= kvalid) S[4 * g + e] = S[4 * g + 2 + e] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int g = 0; g < 8; ++g)
#pragma unroll
        for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], fmaxf(S[4 * g + 2 * h], S[4 * g + 2 * h + 1]));
      float corr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float m_new = fmaxf(m[h], mx[h] * p.scale_log2);
        corr[h] = ex2(m[h] - m_new);                   // first block: exp2(-inf) = 0
        m[h] = m_new;
      }
      // probabilities -> bf16 -> the K-major swizzled A tile of the PV MMA
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        float pe[4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            pe[2 * h + e] = ex2(fmaf(S[4 * g + 2 * h + e], p.scale_log2, -m[h]));
            rs[h] += pe[2 * h + e];
          }
        st_frag_pair(aP, rq, 8 * g + cq, pack_bf16x2(pe[0], pe[1]));
        st_frag_pair(aP, rq + 8, 8 * g + cq, pack_bf16x2(pe[2], pe[3]));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l[h] = fmaf(l[h], corr[h], rs[h]);
#pragma unroll
      for (int g = 0; g < 32; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) O[4 * g + i] *= corr[i >> 1];
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);                     // every row of this warpgroup's P_j is in shared memory
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)                      // B = V_j, MN-major: 64-channel chunks kChunk64 apart
        wgmma_m64n256k16<0, 1>(O, gmma_desc_sw128(aP + k * 32, 16, 1024),
                               gmma_desc_sw128(aV + k * 2048, kChunk64, 1024));
      wgmma_commit();
      wgmma_wait<0>();
      if constexpr (!SHORT) {
        if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[s]);
      }
    }
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      inv[h] = 1.f / l[h];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = q0 + wg * 64 + rq + 8 * h;
      if (row < p.L) {
        __nv_bfloat16* op = p.o + (long long)b * p.o_bs + (long long)row * p.o_ld + c0 + cq;
#pragma unroll
        for (int g = 0; g < 32; ++g)
          *reinterpret_cast<uint32_t*>(op + 8 * g) = pack_bf16x2(O[4 * g + 2 * h] * inv[h], O[4 * g + 2 * h + 1] * inv[h]);
        if (p.lse && (lane & 3) == 0) p.lse[((long long)b * p.heads + head) * p.L + row] = m[h] * kLn2 + logf(l[h]);
      }
    }
  }
}

// backward at head width 256: the skeleton of fdx_attn_bwd128_kernel with 64-row steps on the column side.  Per
// step each warpgroup computes 32 of the 64 columns of S and dP (m64n32, 16 + 16 registers) and writes its half
// of E1 = P and E2 = dS; then
//   dQ[:, 128 wg .. +128] += dS . K_j[:, 128 wg .. +128]   (m64n128 per warpgroup)    [ROWS_ARE_KEYS = false]
//   dV += P^T . dO_i (warpgroup 0),  dK += dS^T . Q_i (warpgroup 1)   (m64n256)        [ROWS_ARE_KEYS = true]
// Shared memory: R1, R2 2 x 32 KB, a ring of 2 x (C1, C2) 2 x 64 KB, E1, E2 2 x 8 KB.
template <bool ROWS_ARE_KEYS>
__global__ void __launch_bounds__(kBwdThreads, 1)
fdx_attn_bwd256_kernel(const __grid_constant__ CUtensorMap mapR1, const __grid_constant__ CUtensorMap mapR2,
                       const __grid_constant__ CUtensorMap mapC1, const __grid_constant__ CUtensorMap mapC2,
                       const AttnDev p) {
  constexpr int RING = 2;
  constexpr int AN = ROWS_ARE_KEYS ? 256 : 128;        // accumulator columns per warpgroup
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sR1 = smem;                                 // [4 chunks][64 rows][64 ch]
  uint8_t* sR2 = smem + kOp256;
  uint8_t* sC = smem + 2 * kOp256;                     // RING x (C1, C2), each [4 chunks][64 rows][64 ch]
  uint8_t* sE1 = sC + RING * 2 * kOp256;               // [64 rows][64 columns]
  uint8_t* sE2 = sE1 + kChunk64;
  float* sStat = reinterpret_cast<float*>(sE2 + kChunk64);       // 2 x (lse[64], dvec[64]) of the columns
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStat + 2 * 128);
  uint64_t* r_full = bars;
  uint64_t* c_full = bars + 1;            // [RING]
  uint64_t* c_empty = c_full + RING;      // [RING]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, b = blockIdx.z;
  const int r0 = blockIdx.x * 64;
  const int nrows = ROWS_ARE_KEYS ? p.Lk : p.L;
  const int ncols = ROWS_ARE_KEYS ? p.L : p.Lk;
  const int nstep = (ncols + 63) / 64;
  const int c0 = head * 256;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapR1); tma_prefetch_desc(&mapR2); tma_prefetch_desc(&mapC1); tma_prefetch_desc(&mapC2);
    mbar_init(r_full, 1);
    for (int i = 0; i < RING; ++i) { mbar_init(&c_full[i], 1); mbar_init(&c_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // setmaxnreg sits inside each role's branch: issued before code both roles run, ptxas ignores it (C7507)
  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && lane == 0) {
      mbar_arrive_expect_tx(r_full, 2 * kOp256);
      for (int c = 0; c < 4; ++c) {
        tma_load_4d(sR1 + c * kChunk64, &mapR1, r_full, c0 + 64 * c, r0, b, 0);
        tma_load_4d(sR2 + c * kChunk64, &mapR2, r_full, c0 + 64 * c, r0, b, 0);
      }
      for (int j = 0; j < nstep; ++j) {
        const int s = j % RING;
        uint8_t* cp = sC + s * 2 * kOp256;
        mbar_wait(&c_empty[s], ((j / RING) & 1) ^ 1);
        mbar_arrive_expect_tx(&c_full[s], 2 * kOp256);
        for (int c = 0; c < 4; ++c) {
          tma_load_4d(cp + c * kChunk64, &mapC1, &c_full[s], c0 + 64 * c, j * 64, b, 0);
          tma_load_4d(cp + kOp256 + c * kChunk64, &mapC2, &c_full[s], c0 + 64 * c, j * 64, b, 0);
        }
      }
    }
  } else {
    consumer_regs();
    const int wg = warp >> 2;                          // columns [32 wg, 32 wg + 32) of S / dP
    const int rq = (warp & 3) * 16 + (lane >> 2);      // fragment rows rq, rq + 8
    const int cq = 2 * (lane & 3);
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const long long stat_base = ((long long)b * p.heads + head) * p.L;
    const bool row_in[2] = {r0 + rq < nrows, r0 + rq + 8 < nrows};
    // dQ kernel: the statistics of this thread's two query rows; dK/dV kernel: they belong to the COLUMNS
    float lse_r[2] = {0.f, 0.f}, d_r[2] = {0.f, 0.f};
    if constexpr (!ROWS_ARE_KEYS) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (row_in[h]) {
          lse_r[h] = p.lse[stat_base + r0 + rq + 8 * h] * kLog2e;
          d_r[h] = p.dvec[stat_base + r0 + rq + 8 * h] * p.scale;
        }
    }
    const uint32_t aR1 = smem_u32(sR1), aR2 = smem_u32(sR2);
    const uint32_t aE1 = smem_u32(sE1), aE2 = smem_u32(sE2);
    float A[AN / 2];                                   // dQ half | dV (warpgroup 0) or dK (warpgroup 1)
#pragma unroll
    for (int i = 0; i < AN / 2; ++i) A[i] = 0.f;
    mbar_wait(r_full, 0);
    for (int j = 0; j < nstep; ++j) {
      const int s = j % RING;
      const int cbase = j * 64;
      if constexpr (ROWS_ARE_KEYS) {
        // stage the query-side statistics of this step (parity buffer j & 1), 64 threads = 64 columns
        if (threadIdx.x < 64) {
          float* st = sStat + (j & 1) * 128;
          const int t = threadIdx.x;
          const bool ok = cbase + t < p.L;
          st[t] = ok ? p.lse[stat_base + cbase + t] * kLog2e : 0.f;
          st[64 + t] = ok ? p.dvec[stat_base + cbase + t] * p.scale : 0.f;
        }
      }
      mbar_wait(&c_full[s], (j / RING) & 1);
      const uint32_t aC1 = smem_u32(sC + s * 2 * kOp256), aC2 = aC1 + kOp256;
      // S (or S^T) = R1 . C1^T ;  dP (or dP^T) = R2 . C2^T  - this warpgroup's 32 columns (rows 32 wg of C)
      float Sa[16], Pa[16];                            // the first K step overwrites them (scale_d = 0)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t ro = (uint32_t)((k >> 2) * kChunk64 + (k & 3) * 32);
        const uint32_t co = ro + (uint32_t)wg * 4096;
        wgmma_m64n32k16<0, 0>(Sa, gmma_desc_sw128(aR1 + ro, 16, 1024), gmma_desc_sw128(aC1 + co, 16, 1024), k > 0);
        wgmma_m64n32k16<0, 0>(Pa, gmma_desc_sw128(aR2 + ro, 16, 1024), gmma_desc_sw128(aC2 + co, 16, 1024), k > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      // the statistics are staged and the previous step's accumulation has consumed E1 / E2
      named_bar_sync(1, 256);
      const float* st = sStat + (j & 1) * 128;
      // rows / columns outside the tensors (TMA zero fill; only the last row tile or step) drop out as -inf
      // logits: P = 0 and dS = 0 there
      const int col_lim = ncols - cbase - wg * 32;     // columns of this warpgroup inside the tensor
      if (r0 + 64 > nrows || col_lim < 32) {
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (!(row_in[h] && 8 * g + cq + e < col_lim)) Sa[4 * g + 2 * h + e] = -INFINITY;
      }
      // P = exp2(s * scale*log2e - lse*log2e);  dS = P * (dP * scale - D * scale)
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int cl = wg * 32 + 8 * g + cq;           // column inside the step's 64
        float lq[2][2], dq[2][2];                      // [h][e]
        if constexpr (ROWS_ARE_KEYS) {
          const float2 a2 = *reinterpret_cast<const float2*>(st + cl);
          const float2 b2 = *reinterpret_cast<const float2*>(st + 64 + cl);
#pragma unroll
          for (int h = 0; h < 2; ++h) { lq[h][0] = a2.x; lq[h][1] = a2.y; dq[h][0] = b2.x; dq[h][1] = b2.y; }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) { lq[h][0] = lq[h][1] = lse_r[h]; dq[h][0] = dq[h][1] = d_r[h]; }
        }
        float pr[4], ds[4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int i = 4 * g + 2 * h + e;
            pr[2 * h + e] = ex2(fmaf(Sa[i], p.scale_log2, -lq[h][e]));
            ds[2 * h + e] = pr[2 * h + e] * fmaf(Pa[i], p.scale, -dq[h][e]);
          }
        if constexpr (ROWS_ARE_KEYS) {
          st_frag_pair(aE1, rq, cl, pack_bf16x2(pr[0], pr[1]));
          st_frag_pair(aE1, rq + 8, cl, pack_bf16x2(pr[2], pr[3]));
        }
        st_frag_pair(aE2, rq, cl, pack_bf16x2(ds[0], ds[1]));
        st_frag_pair(aE2, rq + 8, cl, pack_bf16x2(ds[2], ds[3]));
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 256);                          // both halves of E1 / E2 are published
      wgmma_fence();
      if constexpr (ROWS_ARE_KEYS) {
        // dV += P^T . dO_i (warpgroup 0) | dK += dS^T . Q_i (warpgroup 1); B MN-major, chunks kChunk64 apart
        const uint32_t aE = wg == 0 ? aE1 : aE2;
        const uint32_t aB = wg == 0 ? aC2 : aC1;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n256k16<0, 1>(A, gmma_desc_sw128(aE + k * 32, 16, 1024),
                                 gmma_desc_sw128(aB + k * 2048, kChunk64, 1024));
      } else {
        // dQ[:, 128 wg ..] += dS . K_j[:, 128 wg ..]: B = channel chunks 2 wg, 2 wg + 1 of K_j
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n128k16<0, 1>(A, gmma_desc_sw128(aE2 + k * 32, 16, 1024),
                                 gmma_desc_sw128(aC1 + wg * 2 * kChunk64 + k * 2048, kChunk64, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (wg_leader) mbar_arrive(&c_empty[s]);
    }
    // epilogue: fragment rows -> bf16
    __nv_bfloat16* base;
    long long ld;
    if constexpr (ROWS_ARE_KEYS) {
      base = wg == 0 ? p.dv + (long long)b * p.dv_bs : p.dk + (long long)b * p.dk_bs;
      ld = wg == 0 ? p.dv_ld : p.dk_ld;
      base += c0 + cq;
    } else {
      base = p.dq + (long long)b * p.dq_bs + c0 + wg * 128 + cq;
      ld = p.dq_ld;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (row_in[h]) {
        __nv_bfloat16* rp = base + (long long)(r0 + rq + 8 * h) * ld;
#pragma unroll
        for (int g = 0; g < AN / 8; ++g)
          *reinterpret_cast<uint32_t*>(rp + 8 * g) = pack_bf16x2(A[4 * g + 2 * h], A[4 * g + 2 * h + 1]);
      }
    }
  }
}

int make_map(CUtensorMap* m, const void* ptr, int hd, int rows, int B, long long ld, long long bs,
             int box_rows = 128) {
  uint64_t dims[4] = {(uint64_t)hd, (uint64_t)rows, (uint64_t)B, 1};
  uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)bs * 2, (uint64_t)bs * 2 * (uint64_t)B};
  uint32_t box[4] = {64, (uint32_t)box_rows, 1, 1};
  uint32_t est[4] = {1, 1, 1, 1};
  return fdx_make_tmap_bf16(m, ptr, 4, dims, str, box, est, 1);
}

int check_desc(const fdx_attn_desc* a, const char* who) {
  FDX_REQUIRE(a && a->q && a->k && a->v, "%s: null tensor", who);
  FDX_REQUIRE(a->B > 0 && a->heads > 0 && a->L > 0 && a->Lk > 0, "%s: bad sizes", who);
  FDX_REQUIRE(a->dh == 32 || a->dh == 64 || a->dh == 128 || a->dh == 256,
              "%s: head width %d (stored) must be 32 or 64, or 128 or 256 - zero-pad narrower heads", who, a->dh);
  FDX_REQUIRE((a->heads * a->dh) % 64 == 0, "%s: heads * dh must be a multiple of 64", who);
  FDX_REQUIRE(a->q_ld % 8 == 0, "%s: q_ld must be a multiple of 8 elements", who);
  FDX_REQUIRE(a->k_ld % 8 == 0, "%s: k_ld must be a multiple of 8 elements", who);
  FDX_REQUIRE(a->v_ld % 8 == 0, "%s: v_ld must be a multiple of 8 elements", who);
  FDX_REQUIRE(a->q_bs % 8 == 0, "%s: q_bs must be a multiple of 8 elements", who);
  FDX_REQUIRE(a->k_bs % 8 == 0, "%s: k_bs must be a multiple of 8 elements", who);
  FDX_REQUIRE(a->v_bs % 8 == 0, "%s: v_bs must be a multiple of 8 elements", who);
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(a->q) & 15) == 0, "%s: q must be 16-byte aligned", who);
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(a->k) & 15) == 0, "%s: k must be 16-byte aligned", who);
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(a->v) & 15) == 0, "%s: v must be 16-byte aligned", who);
  return FDX_OK;
}

// o, d_o, dq, dk, dv are written / read with 16-byte vector accesses (and TMA needs 16-byte aligned rows): the
// base pointer must be 16-byte aligned and both strides multiples of 8 bf16 elements, or some row starts off a
// 16-byte boundary and the access faults
int check_io(const void* ptr, long long ld, long long bs, const char* name, const char* ld_name, const char* bs_name,
             const char* who) {
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "%s: %s must be 16-byte aligned", who, name);
  FDX_REQUIRE(ld % 8 == 0, "%s: %s must be a multiple of 8 elements", who, ld_name);
  FDX_REQUIRE(bs % 8 == 0, "%s: %s must be a multiple of 8 elements", who, bs_name);
  return FDX_OK;
}

// argument checks, TMA maps and kernel parameters of both forward entry points
int fwd_prepare(const fdx_attn_desc* a, const char* who, CUtensorMap* mQ, CUtensorMap* mK, CUtensorMap* mV,
                AttnDev* d) {
  int s = check_desc(a, who);
  if (s != FDX_OK) return s;
  FDX_REQUIRE(a->o, "%s: null output", who);
  if ((s = check_io(a->o, a->o_ld, a->o_bs, "o", "o_ld", "o_bs", who)) != FDX_OK) return s;
  const int hd = a->heads * a->dh;
  if ((s = make_map(mQ, a->q, hd, a->L, a->B, a->q_ld, a->q_bs)) != FDX_OK) return s;
  if ((s = make_map(mK, a->k, hd, a->Lk, a->B, a->k_ld, a->k_bs)) != FDX_OK) return s;
  if ((s = make_map(mV, a->v, hd, a->Lk, a->B, a->v_ld, a->v_bs)) != FDX_OK) return s;
  *d = AttnDev{};
  d->B = a->B; d->heads = a->heads; d->L = a->L; d->Lk = a->Lk; d->dh = a->dh;
  d->scale = a->scale; d->scale_log2 = a->scale * kLog2e;
  d->o = (__nv_bfloat16*)a->o; d->o_ld = a->o_ld; d->o_bs = a->o_bs;
  d->lse = a->lse;
  return FDX_OK;
}

}  // namespace

extern "C" {

int fdx_attention_fwd(const fdx_attn_desc* a, void* stream) {
  CUtensorMap mQ, mK, mV;
  AttnDev d;
  int s = fwd_prepare(a, "attention_fwd", &mQ, &mK, &mV, &d);
  if (s != FDX_OK) return s;
  const bool short_keys = a->Lk <= 128;
  if (a->dh == 256) {
    // K and V come in 64-key blocks: their maps get 64-row boxes
    CUtensorMap mK64, mV64;
    if ((s = make_map(&mK64, a->k, a->heads * 256, a->Lk, a->B, a->k_ld, a->k_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&mV64, a->v, a->heads * 256, a->Lk, a->B, a->v_ld, a->v_bs, 64)) != FDX_OK) return s;
    const int smem256 = 4 * kTile + 2 * 2 * kOp256 + 2 * kChunk64 + 1024 + 64;
    dim3 grid256((a->L + 127) / 128, a->heads, a->B);
    static bool attr256[2] = {false, false};
    if (short_keys) {
      if (!attr256[0]) {
        FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd256_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem256));
        attr256[0] = true;
      }
      fdx_attn_fwd256_kernel<true><<<grid256, kBwdThreads, smem256, (cudaStream_t)stream>>>(mQ, mK64, mV64, d);
    } else {
      if (!attr256[1]) {
        FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd256_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem256));
        attr256[1] = true;
      }
      fdx_attn_fwd256_kernel<false><<<grid256, kBwdThreads, smem256, (cudaStream_t)stream>>>(mQ, mK64, mV64, d);
    }
    fdx_note_kernel(FDX_KERNEL_ATTN_FWD);
    FDX_LAUNCH_CHECK();
    return FDX_OK;
  }
  if (a->dh == 128) {
    const int smem128 = (2 + 2 * (short_keys ? 1 : 2)) * kWTile + 1024 + 64;
    dim3 grid128((a->L + 127) / 128, a->heads, a->B);
    static bool attr128[2] = {false, false};
    if (short_keys) {
      if (!attr128[0]) {
        FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd128_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem128));
        attr128[0] = true;
      }
      fdx_attn_fwd128_kernel<true><<<grid128, kFwd128Threads, smem128, (cudaStream_t)stream>>>(mQ, mK, mV, d);
    } else {
      if (!attr128[1]) {
        FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd128_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem128));
        attr128[1] = true;
      }
      fdx_attn_fwd128_kernel<false><<<grid128, kFwd128Threads, smem128, (cudaStream_t)stream>>>(mQ, mK, mV, d);
    }
    fdx_note_kernel(FDX_KERNEL_ATTN_FWD);
    FDX_LAUNCH_CHECK();
    return FDX_OK;
  }
  const int smem = (1 + 2 * (short_keys ? 1 : kKV) + 2) * kTile + kAccXchgBytes + 1024 + 256;
  dim3 grid((a->L + 127) / 128, a->heads, a->B);
  static bool attr[4] = {false, false, false, false};
#define FDX_ATTN_FWD_LAUNCH(DHV, SH, IDX)                                                                         \
  {                                                                                                               \
    if (!attr[IDX]) {                                                                                             \
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd_kernel<DHV, SH>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                    smem));                                                                       \
      attr[IDX] = true;                                                                                           \
    }                                                                                                             \
    fdx_attn_fwd_kernel<DHV, SH><<<grid, kThreads, smem, (cudaStream_t)stream>>>(mQ, mK, mV, d);                  \
  }
  if (a->dh == 64) {
    if (short_keys) FDX_ATTN_FWD_LAUNCH(64, true, 0)
    else FDX_ATTN_FWD_LAUNCH(64, false, 1)
  } else {
    if (short_keys) FDX_ATTN_FWD_LAUNCH(32, true, 2)
    else FDX_ATTN_FWD_LAUNCH(32, false, 3)
  }
#undef FDX_ATTN_FWD_LAUNCH
  fdx_note_kernel(FDX_KERNEL_ATTN_FWD);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_attention_fwd_masked(const fdx_attn_desc* a, int causal, const int32_t* key_mask, void* stream) {
  if (a && (a->dh == 128 || a->dh == 256)) {
    fdx_set_error("attention_fwd_masked: head width %d is not supported (32 or 64)", a->dh);
    return FDX_ERR_UNSUPPORTED;
  }
  CUtensorMap mQ, mK, mV;
  AttnDev d;
  int s = fwd_prepare(a, "attention_fwd_masked", &mQ, &mK, &mV, &d);
  if (s != FDX_OK) return s;
  d.key_mask = key_mask;
  d.causal = causal ? 1 : 0;
  const bool short_keys = a->Lk <= 128;
  const int smem = (1 + 2 * (short_keys ? 1 : kKV) + 2) * kTile + kAccXchgBytes + 1024 + 256;
  dim3 grid((a->L + 127) / 128, a->heads, a->B);
  static bool attr[4] = {false, false, false, false};
#define FDX_ATTN_FWD_MASKED_LAUNCH(DHV, SH, IDX)                                                                  \
  {                                                                                                               \
    if (!attr[IDX]) {                                                                                             \
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_fwd_kernel<DHV, SH, true>,                                           \
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, smem));                          \
      attr[IDX] = true;                                                                                           \
    }                                                                                                             \
    fdx_attn_fwd_kernel<DHV, SH, true><<<grid, kThreads, smem, (cudaStream_t)stream>>>(mQ, mK, mV, d);            \
  }
  if (a->dh == 64) {
    if (short_keys) FDX_ATTN_FWD_MASKED_LAUNCH(64, true, 0)
    else FDX_ATTN_FWD_MASKED_LAUNCH(64, false, 1)
  } else {
    if (short_keys) FDX_ATTN_FWD_MASKED_LAUNCH(32, true, 2)
    else FDX_ATTN_FWD_MASKED_LAUNCH(32, false, 3)
  }
#undef FDX_ATTN_FWD_MASKED_LAUNCH
  fdx_note_kernel(FDX_KERNEL_ATTN_FWD);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_attention_bwd(const fdx_attn_desc* a, void* stream) {
  int s = check_desc(a, "attention_bwd");
  if (s != FDX_OK) return s;
  FDX_REQUIRE(a->o && a->d_o && a->lse && a->dvec_ws && a->dq && a->dk && a->dv, "attention_bwd: null pointer");
  const char* who = "attention_bwd";
  if ((s = check_io(a->o, a->o_ld, a->o_bs, "o", "o_ld", "o_bs", who)) != FDX_OK) return s;
  if ((s = check_io(a->d_o, a->do_ld, a->do_bs, "d_o", "do_ld", "do_bs", who)) != FDX_OK) return s;
  if ((s = check_io(a->dq, a->dq_ld, a->dq_bs, "dq", "dq_ld", "dq_bs", who)) != FDX_OK) return s;
  if ((s = check_io(a->dk, a->dk_ld, a->dk_bs, "dk", "dk_ld", "dk_bs", who)) != FDX_OK) return s;
  if ((s = check_io(a->dv, a->dv_ld, a->dv_bs, "dv", "dv_ld", "dv_bs", who)) != FDX_OK) return s;
  const int hd = a->heads * a->dh;
  CUtensorMap mQ, mK, mV, mDO;
  if ((s = make_map(&mQ, a->q, hd, a->L, a->B, a->q_ld, a->q_bs)) != FDX_OK) return s;
  if ((s = make_map(&mK, a->k, hd, a->Lk, a->B, a->k_ld, a->k_bs)) != FDX_OK) return s;
  if ((s = make_map(&mV, a->v, hd, a->Lk, a->B, a->v_ld, a->v_bs)) != FDX_OK) return s;
  if ((s = make_map(&mDO, a->d_o, hd, a->L, a->B, a->do_ld, a->do_bs)) != FDX_OK) return s;
  AttnDev d{};
  d.B = a->B; d.heads = a->heads; d.L = a->L; d.Lk = a->Lk; d.dh = a->dh;
  d.scale = a->scale; d.scale_log2 = a->scale * kLog2e;
  d.lse = a->lse; d.dvec = a->dvec_ws;
  d.d_o = (const __nv_bfloat16*)a->d_o; d.do_ld = a->do_ld; d.do_bs = a->do_bs;
  d.o_in = (const __nv_bfloat16*)a->o; d.oin_ld = a->o_ld; d.oin_bs = a->o_bs;
  d.dq = (__nv_bfloat16*)a->dq; d.dq_ld = a->dq_ld; d.dq_bs = a->dq_bs;
  d.dk = (__nv_bfloat16*)a->dk; d.dk_ld = a->dk_ld; d.dk_bs = a->dk_bs;
  d.dv = (__nv_bfloat16*)a->dv; d.dv_ld = a->dv_ld; d.dv_bs = a->dv_bs;
  cudaStream_t st = (cudaStream_t)stream;
  {
    const long long total = (long long)a->B * a->L * a->heads;
    attn_dvec_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d);
    FDX_LAUNCH_CHECK();
  }
  if (a->dh == 256) {
    // both sides of both kernels come in 64-row blocks
    CUtensorMap rQ, rK, rV, rDO;
    if ((s = make_map(&rQ, a->q, hd, a->L, a->B, a->q_ld, a->q_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rK, a->k, hd, a->Lk, a->B, a->k_ld, a->k_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rV, a->v, hd, a->Lk, a->B, a->v_ld, a->v_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rDO, a->d_o, hd, a->L, a->B, a->do_ld, a->do_bs, 64)) != FDX_OK) return s;
    const int smem256 = 2 * kOp256 + 2 * 2 * kOp256 + 2 * kChunk64 + 2 * 128 * 4 + 1024 + 64;
    static bool attr256 = false;
    if (!attr256) {
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_bwd256_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    smem256));
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_bwd256_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    smem256));
      attr256 = true;
    }
    // dQ: rows = queries (Q, dO), loop (K_j, V_j);  dK/dV: rows = keys (K, V), loop (Q_i, dO_i)
    fdx_attn_bwd256_kernel<false><<<dim3((a->L + 63) / 64, a->heads, a->B), kBwdThreads, smem256, st>>>(
        rQ, rDO, rK, rV, d);
    fdx_note_kernel(FDX_KERNEL_ATTN_BWD);
    FDX_LAUNCH_CHECK();
    fdx_attn_bwd256_kernel<true><<<dim3((a->Lk + 63) / 64, a->heads, a->B), kBwdThreads, smem256, st>>>(
        rK, rV, rQ, rDO, d);
    fdx_note_kernel(FDX_KERNEL_ATTN_BWD);
    FDX_LAUNCH_CHECK();
    return FDX_OK;
  }
  if (a->dh == 128) {
    // the row side of a 64-row tile comes in 64-row boxes; the looped column side keeps the 128-row maps
    CUtensorMap rQ, rK, rV, rDO;
    if ((s = make_map(&rQ, a->q, hd, a->L, a->B, a->q_ld, a->q_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rK, a->k, hd, a->Lk, a->B, a->k_ld, a->k_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rV, a->v, hd, a->Lk, a->B, a->v_ld, a->v_bs, 64)) != FDX_OK) return s;
    if ((s = make_map(&rDO, a->d_o, hd, a->L, a->B, a->do_ld, a->do_bs, 64)) != FDX_OK) return s;
    const int smem128 = 4 * kTile + 2 * 2 * kWTile + 2 * 256 * 4 + 1024 + 64;
    static bool attr128 = false;
    if (!attr128) {
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_bwd128_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    smem128));
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_bwd128_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    smem128));
      attr128 = true;
    }
    // dQ: rows = queries (Q, dO), loop (K_j, V_j);  dK/dV: rows = keys (K, V), loop (Q_i, dO_i)
    fdx_attn_bwd128_kernel<false><<<dim3((a->L + 63) / 64, a->heads, a->B), kBwdThreads, smem128, st>>>(
        rQ, rDO, mK, mV, d);
    fdx_note_kernel(FDX_KERNEL_ATTN_BWD);
    FDX_LAUNCH_CHECK();
    fdx_attn_bwd128_kernel<true><<<dim3((a->Lk + 63) / 64, a->heads, a->B), kBwdThreads, smem128, st>>>(
        rK, rV, mQ, mDO, d);
    fdx_note_kernel(FDX_KERNEL_ATTN_BWD);
    FDX_LAUNCH_CHECK();
    return FDX_OK;
  }
  const int smem = (2 + 2 * 2 + 4) * kTile + 2 * 256 * 4 + 2 * kAccXchgBytes + 1024 + 256;
  static bool attr[4] = {false, false, false, false};
#define FDX_ATTN_BWD_LAUNCH(DHV, RK, IDX, GRIDX, M1, M2, M3, M4)                                                  \
  {                                                                                                                \
    if (!attr[IDX]) {                                                                                              \
      FDX_CUDA(cudaFuncSetAttribute(fdx_attn_bwd_kernel<DHV, RK>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                    smem));                                                                        \
      attr[IDX] = true;                                                                                            \
    }                                                                                                              \
    dim3 grid((GRIDX + 127) / 128, a->heads, a->B);                                                                \
    fdx_attn_bwd_kernel<DHV, RK><<<grid, kBwdThreads, smem, st>>>(M1, M2, M3, M4, d);                              \
    fdx_note_kernel(FDX_KERNEL_ATTN_BWD);                                                                          \
    FDX_LAUNCH_CHECK();                                                                                            \
  }
  if (a->dh == 64) {
    FDX_ATTN_BWD_LAUNCH(64, false, 0, a->L, mQ, mDO, mK, mV)      // dQ: rows = queries (Q, dO), loop (K_j, V_j)
    FDX_ATTN_BWD_LAUNCH(64, true, 1, a->Lk, mK, mV, mQ, mDO)      // dK/dV: rows = keys (K, V), loop (Q_i, dO_i)
  } else {
    FDX_ATTN_BWD_LAUNCH(32, false, 2, a->L, mQ, mDO, mK, mV)
    FDX_ATTN_BWD_LAUNCH(32, true, 3, a->Lk, mK, mV, mQ, mDO)
  }
#undef FDX_ATTN_BWD_LAUNCH
  return FDX_OK;
}

}  // extern "C"
