// fdx_mmdit.cu -- the HBM-bound kernels of the SimpleMMDiT block (flaxdiff/models/simple_mmdit.py:17-158) that sit
// around the GEMM engine and the fused attention.  The MMDiT block is a parallel block: ONE LayerNorm of the block input
// is modulated twice (attention chunks as they are, MLP chunks clipped to [-10, 10]) and both branches are added onto
// the same residual.  These kernels fuse exactly that: one pass over x writes both modulated rows, one pass over dout
// forms both branch gradients, one pass forms the LayerNorm backward of both.
//
// ada / d_ada rows hold six C-wide chunks in the reference's split order: scale_mlp 0, shift_mlp 1, gate_mlp 2,
// scale_attn 3, shift_attn 4, gate_attn 5.  bf16 activations, f32 statistics and sums, 16-byte vectors.  Every
// per-sample column sum is formed in a fixed order (per-chunk partial sums, then an ordered reduction): no atomics, so
// a step is bit-reproducible.
#include "fdx_common.cuh"
#include "../../include/fdx.h"

namespace {

inline int stream_grid(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = (long long)fdx_num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void ld8f(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// MMAdaLNZero's jnp.clip(v, -10, 10) (simple_mmdit.py:81-82) and its derivative under JAX's autodiff: clip is
// min(max(v, lo), hi), and lax.max / lax.min split the cotangent evenly between equal operands, so the derivative is
// 1 inside, 0 outside and 1/2 at exactly -10 or 10.
constexpr float kClip = 10.f;
__device__ __forceinline__ float clip10(float v) { return fminf(fmaxf(v, -kClip), kClip); }
__device__ __forceinline__ float clip10_grad(float v) {
  return (v > -kClip && v < kClip) ? 1.f : ((v == -kClip || v == kClip) ? 0.5f : 0.f);
}

enum { kScaleM = 0, kShiftM = 1, kGateM = 2, kScaleA = 3, kShiftA = 4, kGateA = 5 };   // ada chunk order

constexpr int kV = 6;               // one warp holds a row of up to 6 x 32 x 8 = 1536 channels
constexpr int kColSlab = 64;        // columns per column-sum block (8 threads x 8 channels)

// ---- one LayerNorm, two modulations: one warp per token ----------------------------------------------------------
// xhat = (x - mean) * rstd;  y_attn = xhat (1 + scale_attn) + shift_attn;  y_mlp = xhat (1 + clip(scale_mlp)) +
// clip(shift_mlp).  The row stays in registers between the mean and the centred-variance pass.
__global__ void __launch_bounds__(256)
mmdit_adaln_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int L, int C, const float* __restrict__ ada,
                       long long ada_ld, float eps, __nv_bfloat16* __restrict__ ya, __nv_bfloat16* __restrict__ ym,
                       float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    float f[kV][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < kV; ++v) {
      if (v * 32 + lane < nv) {
        ld8(x + r * C + (v * 32 + lane) * 8, f[v]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[v][j];
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < kV; ++v) {
      if (v * 32 + lane < nv) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          f[v][j] -= mean;
          q = fmaf(f[v][j], f[v][j], q);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
    if (lane == 0 && mean_out) {
      mean_out[r] = mean;
      rstd_out[r] = rstd;
    }
    const float* arow = ada + (r / L) * ada_ld;
#pragma unroll
    for (int v = 0; v < kV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float sa[8], ha[8], sm[8], hm[8], o[8];
        ld8f(arow + kScaleA * C + c, sa);
        ld8f(arow + kShiftA * C + c, ha);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(f[v][j] * rstd, 1.f + sa[j], ha[j]);
        st8(ya + r * C + c, o);
        ld8f(arow + kScaleM * C + c, sm);
        ld8f(arow + kShiftM * C + c, hm);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(f[v][j] * rstd, 1.f + clip10(sm[j]), clip10(hm[j]));
        st8(ym + r * C + c, o);
      }
    }
  }
}

// ---- its data gradient: one warp per token ------------------------------------------------------------------------
// g = dy_attn (1 + scale_attn) + dy_mlp (1 + clip(scale_mlp));  dx = rstd (g - mean(g) - xhat mean(g xhat)) (+ addend).
// dx may alias addend.
__global__ void __launch_bounds__(256)
mmdit_adaln_bwd_dx_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dya,
                          const __nv_bfloat16* __restrict__ dym, long long rows, int L, int C,
                          const float* __restrict__ ada, long long ada_ld, const float* __restrict__ mean,
                          const float* __restrict__ rstd, const __nv_bfloat16* addend, __nv_bfloat16* dx) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    const float mu = mean[r], rs = rstd[r];
    const float* arow = ada + (r / L) * ada_ld;
    float xh[kV][8], g[kV][8];
    float a = 0.f, q = 0.f;
#pragma unroll
    for (int v = 0; v < kV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float gm[8], sa[8], sm[8];
        ld8(x + r * C + c, xh[v]);
        ld8(dya + r * C + c, g[v]);
        ld8(dym + r * C + c, gm);
        ld8f(arow + kScaleA * C + c, sa);
        ld8f(arow + kScaleM * C + c, sm);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[v][j] = (xh[v][j] - mu) * rs;
          g[v][j] = fmaf(g[v][j], 1.f + sa[j], gm[j] * (1.f + clip10(sm[j])));
          a += g[v][j];
          q = fmaf(g[v][j], xh[v][j], q);
        }
      }
    }
    const float ma = warp_sum(a) / (float)C, mq = warp_sum(q) / (float)C;
#pragma unroll
    for (int v = 0; v < kV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float ad[8], o[8];
        if (addend) {
          ld8(addend + r * C + c, ad);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) ad[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(rs, g[v][j] - ma - xh[v][j] * mq, ad[j]);
        st8(dx + r * C + c, o);
      }
    }
  }
}

// ---- per-sample column sums over a sample's tokens, first stage -------------------------------------------------
// Block (slab of 64 columns, token chunk k, sample b): 8 threads x 8 channels across, 32 token rows down; the 32 row
// partials are added in row order.  ws[b][k][NS][C].
//   MODE_LN   (NS 4): dy_attn xhat, dy_attn, dy_mlp xhat, dy_mlp            (a0 = dy_attn, a1 = dy_mlp, x the input)
//   MODE_GATE (NS 2): dout y_attn, dout y_mlp; writes dy_attn = gate_attn dout and dy_mlp = gate_mlp dout
//                     (a0 = dout, x = y_attn, a1 = y_mlp)
enum { MODE_LN = 0, MODE_GATE = 1 };

template <int MODE>
__global__ void __launch_bounds__(256)
mmdit_colsum_kernel(const __nv_bfloat16* __restrict__ a0, const __nv_bfloat16* __restrict__ a1,
                    const __nv_bfloat16* __restrict__ x, const float* __restrict__ mean,
                    const float* __restrict__ rstd, int L, int C, int nchunk, const float* __restrict__ ada,
                    long long ada_ld, __nv_bfloat16* __restrict__ dya, __nv_bfloat16* __restrict__ dym,
                    float* __restrict__ ws) {
  constexpr int NS = MODE == MODE_LN ? 4 : 2;
  __shared__ float red[NS][32][kColSlab];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int k = blockIdx.y, b = blockIdx.z;
  const int c = blockIdx.x * kColSlab + tx * 8;
  const int per = (L + nchunk - 1) / nchunk;
  const int t0 = k * per, t1 = min(L, t0 + per);
  float s[NS][8];
#pragma unroll
  for (int i = 0; i < NS; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s[i][j] = 0.f;
  if (c < C) {
    float ga[8], gm[8];
    if (MODE == MODE_GATE) {
      ld8f(ada + (long long)b * ada_ld + kGateA * C + c, ga);
      ld8f(ada + (long long)b * ada_ld + kGateM * C + c, gm);
    }
    for (int t = t0 + ty; t < t1; t += 32) {
      const long long r = (long long)b * L + t;
      float u[8], w[8], xv[8];
      ld8(a0 + r * C + c, u);
      ld8(a1 + r * C + c, w);
      ld8(x + r * C + c, xv);
      if constexpr (MODE == MODE_LN) {
        const float mu = mean[r], rs = rstd[r];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xv[j] - mu) * rs;
          s[0][j] = fmaf(u[j], xh, s[0][j]);
          s[1][j] += u[j];
          s[2][j] = fmaf(w[j], xh, s[2][j]);
          s[3][j] += w[j];
        }
      } else {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s[0][j] = fmaf(u[j], xv[j], s[0][j]);
          s[1][j] = fmaf(u[j], w[j], s[1][j]);
          o[j] = ga[j] * u[j];
        }
        st8(dya + r * C + c, o);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = gm[j] * u[j];
        st8(dym + r * C + c, o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NS; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[i][ty][tx * 8 + j] = s[i][j];
  __syncthreads();
  if (threadIdx.x < NS * kColSlab) {
    const int which = threadIdx.x / kColSlab, col = threadIdx.x % kColSlab;
    const int cc = blockIdx.x * kColSlab + col;
    if (cc < C) {
      float sum = 0.f;
      for (int i = 0; i < 32; ++i) sum += red[which][i][col];
      ws[(((long long)b * nchunk + k) * NS + which) * C + cc] = sum;
    }
  }
}

// Second stage: d_ada[b][chunk(j) * C + c] = mask_j * sum_k ws[b][k][j][c], the chunks in stage-one order; the mlp
// chunks' mask is clip10_grad of the forward value.
template <int MODE>
__global__ void mmdit_colsum_finish_kernel(const float* __restrict__ ws, int B, int nchunk, int C,
                                           const float* __restrict__ ada, long long ada_ld, float* __restrict__ d_ada,
                                           long long d_ld) {
  constexpr int NS = MODE == MODE_LN ? 4 : 2;
  const long long total = (long long)B * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / C), c = (int)(i % C);
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      float sum = 0.f;
      for (int k = 0; k < nchunk; ++k) sum += ws[(((long long)b * nchunk + k) * NS + j) * C + c];
      int chunk;
      if (MODE == MODE_LN) {
        chunk = j == 0 ? kScaleA : j == 1 ? kShiftA : j == 2 ? kScaleM : kShiftM;
        if (j >= 2) sum *= clip10_grad(ada[(long long)b * ada_ld + chunk * C + c]);
      } else {
        chunk = j == 0 ? kGateA : kGateM;
      }
      d_ada[(long long)b * d_ld + chunk * C + c] = sum;
    }
  }
}

// ---- the parallel block's residual: out = x + gate_attn y_attn + gate_mlp y_mlp, one rounding (out may alias x) ----
__global__ void mmdit_gate_fwd_kernel(const __nv_bfloat16* x, const __nv_bfloat16* __restrict__ ya,
                                      const __nv_bfloat16* __restrict__ ym, long long rows, int L, int C,
                                      const float* __restrict__ ada, long long ada_ld, __nv_bfloat16* out) {
  const int v = C / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    const float* arow = ada + (r / L) * ada_ld;
    float xv[8], a[8], m[8], ga[8], gm[8];
    ld8(x + r * C + c, xv);
    ld8(ya + r * C + c, a);
    ld8(ym + r * C + c, m);
    ld8f(arow + kGateA * C + c, ga);
    ld8f(arow + kGateM * C + c, gm);
#pragma unroll
    for (int j = 0; j < 8; ++j) xv[j] = fmaf(gm[j], m[j], fmaf(ga[j], a[j], xv[j]));
    st8(out + r * C + c, xv);
  }
}

template <int MODE>
int colsum_launch(const void* a0, const void* a1, const void* x, const float* mean, const float* rstd, int B, int L,
                  int C, const float* ada, long long ada_ld, void* dya, void* dym, float* ws, int nchunk, float* d_ada,
                  long long d_ld, cudaStream_t st) {
  FDX_REQUIRE(ws && nchunk > 0 && nchunk <= 65535 && B <= 65535, "mmdit colsum: bad workspace / sizes");
  const dim3 grid((C + kColSlab - 1) / kColSlab, nchunk, B);
  mmdit_colsum_kernel<MODE><<<grid, 256, 0, st>>>(
      (const __nv_bfloat16*)a0, (const __nv_bfloat16*)a1, (const __nv_bfloat16*)x, mean, rstd, L, C, nchunk, ada,
      ada_ld, (__nv_bfloat16*)dya, (__nv_bfloat16*)dym, ws);
  FDX_LAUNCH_CHECK();
  mmdit_colsum_finish_kernel<MODE><<<stream_grid((long long)B * C, 256), 256, 0, st>>>(ws, B, nchunk, C, ada, ada_ld,
                                                                                       d_ada, d_ld);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

inline bool row_ok(int C) { return C > 0 && C % 8 == 0 && C <= 32 * 8 * kV; }
inline bool ada_ok(const float* ada, long long ld, int C) { return ada && aligned16(ada) && ld % 4 == 0 && ld >= 6LL * C; }


// ---- affine LayerNorm over wide rows with 2x2 assembly: HierarchicalMMDiT's PatchMerging / PatchExpanding / fusion --
// A logical row r of C columns (C a multiple of 8, <= 6144) is assembled from, or scattered to, token rows:
//   LN_GATHER  : row r = coarse patch (b, h, w) of an HPc x WPc grid; column c = (p1, p2, cc), cc < Cf = C / 4, reads
//                fine row b HP WP + (2h + p1) WP + (2w + p2) of src0 (HP = 2 HPc, WP = 2 WPc); y is [rows][C].
//   LN_CONCAT  : columns [0, C0) from src0 [rows][C0], [C0, C) from src1 [rows][C - C0]; y is [rows][C].
//   LN_SCATTER : src0 is [rows][C]; column (p1, p2, cc) of row (b, h, w) is written to fine row
//                b HP WP + (2h + p1) WP + (2w + p2), channel cc, of y [4 rows][Cf].
// One CTA per row (256 threads x up to 3 vectors of 8 channels in registers); block sums in a fixed order.
enum { LN_GATHER = 0, LN_CONCAT = 1, LN_SCATTER = 2 };
constexpr int kRowV = 3;
constexpr int kRowMax = 256 * 8 * kRowV;

struct RowMap {
  int mode, C, C0, HPc, WPc;
  // element offset of column c of logical row r in the assembled side (gather / scatter: fine rows, width C / 4)
  __device__ __forceinline__ long long fine(long long r, int c) const {
    const int Cf = C >> 2;
    const int p1 = c / (2 * Cf), p2 = (c / Cf) & 1, cc = c % Cf;
    const long long per = (long long)HPc * WPc;
    const long long b = r / per;
    const int hw = (int)(r % per), h = hw / WPc, w = hw % WPc;
    return ((b * 2 * HPc + 2 * h + p1) * (2LL * WPc) + 2 * w + p2) * Cf + cc;
  }
};

__device__ __forceinline__ float block_sum256(float v, float* sh) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += sh[i];
  return t;
}

// input column c of row r (the un-normalised value) as 8 floats
__device__ __forceinline__ void ln_load(const RowMap& m, const __nv_bfloat16* src0, const __nv_bfloat16* src1,
                                        long long r, int c, float (&f)[8]) {
  if (m.mode == LN_GATHER)
    ld8(src0 + m.fine(r, c), f);
  else if (m.mode == LN_CONCAT)
    c < m.C0 ? ld8(src0 + r * m.C0 + c, f) : ld8(src1 + r * (m.C - m.C0) + (c - m.C0), f);
  else
    ld8(src0 + r * m.C + c, f);
}

__global__ void __launch_bounds__(256)
ln_rows_fwd_kernel(RowMap m, const __nv_bfloat16* __restrict__ src0, const __nv_bfloat16* __restrict__ src1,
                   long long rows, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  __shared__ float sh[8];
  const int nv = m.C >> 3;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    float f[kRowV][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < kRowV; ++v) {
      const int vi = v * 256 + threadIdx.x;
      if (vi < nv) {
        ln_load(m, src0, src1, r, vi * 8, f[v]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[v][j];
      }
    }
    const float mean = block_sum256(s, sh) / (float)m.C;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < kRowV; ++v) {
      if (v * 256 + (int)threadIdx.x < nv) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          f[v][j] -= mean;
          q = fmaf(f[v][j], f[v][j], q);
        }
      }
    }
    const float rstd = rsqrtf(block_sum256(q, sh) / (float)m.C + eps);
    if (threadIdx.x == 0) {
      mean_out[r] = mean;
      rstd_out[r] = rstd;
    }
#pragma unroll
    for (int v = 0; v < kRowV; ++v) {
      const int vi = v * 256 + threadIdx.x;
      if (vi < nv) {
        const int c = vi * 8;
        float g[8], b[8], o[8];
        ld8f(gamma + c, g);
        ld8f(beta + c, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(f[v][j] * rstd, g[j], b[j]);
        st8(y + (m.mode == LN_SCATTER ? m.fine(r, c) : r * m.C + c), o);
      }
    }
  }
}

// Backward: CTA k takes rows [k per, (k + 1) per), writes dx (the input's layout; each destination (+)= by its flag)
// and its partial sums of dy xhat and dy per column into ws[k][2][C].
__global__ void __launch_bounds__(256)
ln_rows_bwd_kernel(RowMap m, const __nv_bfloat16* __restrict__ src0, const __nv_bfloat16* __restrict__ src1,
                   const __nv_bfloat16* __restrict__ dy, long long rows, long long per,
                   const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                   __nv_bfloat16* dx0, int acc0, __nv_bfloat16* dx1, int acc1, float* __restrict__ ws) {
  __shared__ float sh[8];
  const int nv = m.C >> 3;
  float pg[kRowV][8], pb[kRowV][8];
#pragma unroll
  for (int v = 0; v < kRowV; ++v)
#pragma unroll
    for (int j = 0; j < 8; ++j) pg[v][j] = pb[v][j] = 0.f;
  const long long r0 = blockIdx.x * per, r1 = min(rows, r0 + per);
  for (long long r = r0; r < r1; ++r) {
    const float mu = mean[r], rs = rstd[r];
    float xh[kRowV][8], g[kRowV][8];
    float a = 0.f, q = 0.f;
#pragma unroll
    for (int v = 0; v < kRowV; ++v) {
      const int vi = v * 256 + threadIdx.x;
      if (vi < nv) {
        const int c = vi * 8;
        float ga[8];
        ln_load(m, src0, src1, r, c, xh[v]);
        ld8(dy + (m.mode == LN_SCATTER ? m.fine(r, c) : r * m.C + c), g[v]);
        ld8f(gamma + c, ga);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[v][j] = (xh[v][j] - mu) * rs;
          pg[v][j] = fmaf(g[v][j], xh[v][j], pg[v][j]);
          pb[v][j] += g[v][j];
          g[v][j] *= ga[j];
          a += g[v][j];
          q = fmaf(g[v][j], xh[v][j], q);
        }
      }
    }
    const float ma = block_sum256(a, sh) / (float)m.C, mq = block_sum256(q, sh) / (float)m.C;
#pragma unroll
    for (int v = 0; v < kRowV; ++v) {
      const int vi = v * 256 + threadIdx.x;
      if (vi < nv) {
        const int c = vi * 8;
        __nv_bfloat16* d;
        int acc;
        if (m.mode == LN_GATHER) {
          d = dx0 + m.fine(r, c);
          acc = acc0;
        } else if (m.mode == LN_CONCAT && c >= m.C0) {
          d = dx1 + r * (m.C - m.C0) + (c - m.C0);
          acc = acc1;
        } else {
          d = dx0 + r * (m.mode == LN_CONCAT ? m.C0 : m.C) + c;
          acc = acc0;
        }
        float o[8];
        if (acc) {
          ld8(d, o);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(rs, g[v][j] - ma - xh[v][j] * mq, o[j]);
        st8(d, o);
      }
    }
  }
#pragma unroll
  for (int v = 0; v < kRowV; ++v) {
    const int vi = v * 256 + threadIdx.x;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ws[((long long)blockIdx.x * 2) * m.C + vi * 8 + j] = pg[v][j];
        ws[((long long)blockIdx.x * 2 + 1) * m.C + vi * 8 + j] = pb[v][j];
      }
    }
  }
}

// dgamma[c] += sum_k ws[k][0][c], dbeta[c] += sum_k ws[k][1][c], in chunk order
__global__ void ln_rows_param_finish_kernel(const float* __restrict__ ws, int nchunk, int C, float* dgamma,
                                            float* dbeta) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float sg = 0.f, sb = 0.f;
    for (int k = 0; k < nchunk; ++k) {
      sg += ws[(2LL * k) * C + c];
      sb += ws[(2LL * k + 1) * C + c];
    }
    dgamma[c] += sg;
    dbeta[c] += sb;
  }
}

inline int rowmap_check(RowMap& m, int mode, long long rows, int C, int C0, int HPc, int WPc) {
  m.mode = mode; m.C = C; m.C0 = C0; m.HPc = HPc; m.WPc = WPc;
  FDX_REQUIRE(mode >= LN_GATHER && mode <= LN_SCATTER, "layernorm_rows: mode %d", mode);
  FDX_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && C <= kRowMax, "layernorm_rows: C=%d must be a multiple of 8, <= %d",
              C, kRowMax);
  if (mode == LN_CONCAT)
    FDX_REQUIRE(C0 > 0 && C0 < C && C0 % 8 == 0, "layernorm_rows: concat split C0=%d", C0);
  else
    FDX_REQUIRE(C % 32 == 0 && HPc > 0 && WPc > 0 && rows % ((long long)HPc * WPc) == 0,
                "layernorm_rows: 2x2 modes need C a multiple of 32 and rows a multiple of HPc * WPc");
  return FDX_OK;
}
}  // namespace

extern "C" {

int fdx_mmdit_adaln_fwd(const void* x_bf16, long long rows, int L, int C, const float* ada, long long ada_ld,
                        float eps, void* y_attn_bf16, void* y_mlp_bf16, float* mean, float* rstd, void* stream) {
  FDX_REQUIRE(x_bf16 && y_attn_bf16 && y_mlp_bf16, "mmdit_adaln_fwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && row_ok(C),
              "mmdit_adaln_fwd: C=%d must be a multiple of 8, <= %d; rows a multiple of L", C, 32 * 8 * kV);
  FDX_REQUIRE(ada_ok(ada, ada_ld, C), "mmdit_adaln_fwd: ada rows must hold 6 C floats, 16-byte aligned");
  FDX_REQUIRE((mean == nullptr) == (rstd == nullptr), "mmdit_adaln_fwd: mean and rstd go together");
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_attn_bf16) && aligned16(y_mlp_bf16),
              "mmdit_adaln_fwd: tensors must be 16-byte aligned");
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  mmdit_adaln_fwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, rows, L, C, ada, ada_ld, eps, (__nv_bfloat16*)y_attn_bf16,
      (__nv_bfloat16*)y_mlp_bf16, mean, rstd);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_mmdit_adaln_bwd(const void* x_bf16, const void* dy_attn_bf16, const void* dy_mlp_bf16, long long rows, int L,
                        int C, const float* ada, long long ada_ld, const float* mean, const float* rstd,
                        const void* addend_bf16, void* dx_bf16, float* ws, int nchunk, float* d_ada,
                        long long d_ada_ld, void* stream) {
  FDX_REQUIRE(x_bf16 && dy_attn_bf16 && dy_mlp_bf16 && dx_bf16 && mean && rstd && d_ada,
              "mmdit_adaln_bwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && row_ok(C),
              "mmdit_adaln_bwd: C=%d must be a multiple of 8, <= %d; rows a multiple of L", C, 32 * 8 * kV);
  FDX_REQUIRE(ada_ok(ada, ada_ld, C) && d_ada_ld >= 6LL * C,
              "mmdit_adaln_bwd: ada / d_ada rows must hold 6 C floats, ada 16-byte aligned");
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(dy_attn_bf16) && aligned16(dy_mlp_bf16) && aligned16(dx_bf16) &&
                  (!addend_bf16 || aligned16(addend_bf16)),
              "mmdit_adaln_bwd: tensors must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int s = colsum_launch<MODE_LN>(dy_attn_bf16, dy_mlp_bf16, x_bf16, mean, rstd, (int)(rows / L), L, C, ada,
                                       ada_ld, nullptr, nullptr, ws, nchunk, d_ada, d_ada_ld, st);
  if (s != FDX_OK) return s;
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  mmdit_adaln_bwd_dx_kernel<<<(int)grid, 256, 0, st>>>(
      (const __nv_bfloat16*)x_bf16, (const __nv_bfloat16*)dy_attn_bf16, (const __nv_bfloat16*)dy_mlp_bf16, rows, L, C,
      ada, ada_ld, mean, rstd, (const __nv_bfloat16*)addend_bf16, (__nv_bfloat16*)dx_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_mmdit_gate_fwd(const void* x_bf16, const void* y_attn_bf16, const void* y_mlp_bf16, long long rows, int L,
                       int C, const float* ada, long long ada_ld, void* out_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && y_attn_bf16 && y_mlp_bf16 && out_bf16, "mmdit_gate_fwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && C > 0 && C % 8 == 0, "mmdit_gate_fwd: bad sizes (C=%d)", C);
  FDX_REQUIRE(ada_ok(ada, ada_ld, C), "mmdit_gate_fwd: ada rows must hold 6 C floats, 16-byte aligned");
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_attn_bf16) && aligned16(y_mlp_bf16) && aligned16(out_bf16),
              "mmdit_gate_fwd: tensors must be 16-byte aligned");
  mmdit_gate_fwd_kernel<<<stream_grid(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, (const __nv_bfloat16*)y_attn_bf16, (const __nv_bfloat16*)y_mlp_bf16, rows, L, C,
      ada, ada_ld, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_mmdit_gate_bwd(const void* dout_bf16, const void* y_attn_bf16, const void* y_mlp_bf16, long long rows, int L,
                       int C, const float* ada, long long ada_ld, void* dy_attn_bf16, void* dy_mlp_bf16, float* ws,
                       int nchunk, float* d_ada, long long d_ada_ld, void* stream) {
  FDX_REQUIRE(dout_bf16 && y_attn_bf16 && y_mlp_bf16 && dy_attn_bf16 && dy_mlp_bf16 && d_ada,
              "mmdit_gate_bwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && C > 0 && C % 8 == 0, "mmdit_gate_bwd: bad sizes (C=%d)", C);
  FDX_REQUIRE(ada_ok(ada, ada_ld, C) && d_ada_ld >= 6LL * C,
              "mmdit_gate_bwd: ada / d_ada rows must hold 6 C floats, ada 16-byte aligned");
  FDX_REQUIRE(aligned16(dout_bf16) && aligned16(y_attn_bf16) && aligned16(y_mlp_bf16) && aligned16(dy_attn_bf16) &&
                  aligned16(dy_mlp_bf16),
              "mmdit_gate_bwd: tensors must be 16-byte aligned");
  return colsum_launch<MODE_GATE>(dout_bf16, y_mlp_bf16, y_attn_bf16, nullptr, nullptr, (int)(rows / L), L, C, ada,
                                  ada_ld, dy_attn_bf16, dy_mlp_bf16, ws, nchunk, d_ada, d_ada_ld,
                                  (cudaStream_t)stream);
}


int fdx_layernorm_rows_fwd(int mode, const void* src0_bf16, const void* src1_bf16, long long rows, int C, int C0,
                           int HPc, int WPc, const float* gamma, const float* beta, float eps, void* y_bf16,
                           float* mean, float* rstd, void* stream) {
  RowMap m;
  const int st = rowmap_check(m, mode, rows, C, C0, HPc, WPc);
  if (st != FDX_OK) return st;
  FDX_REQUIRE(src0_bf16 && (mode != LN_CONCAT || src1_bf16) && gamma && beta && y_bf16 && mean && rstd,
              "layernorm_rows_fwd: null pointer");
  FDX_REQUIRE(aligned16(src0_bf16) && (!src1_bf16 || aligned16(src1_bf16)) && aligned16(y_bf16) && aligned16(gamma) &&
                  aligned16(beta), "layernorm_rows_fwd: tensors must be 16-byte aligned");
  long long grid = rows < (long long)fdx_num_sms() * 8 ? rows : (long long)fdx_num_sms() * 8;
  ln_rows_fwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(
      m, (const __nv_bfloat16*)src0_bf16, (const __nv_bfloat16*)src1_bf16, rows, gamma, beta, eps,
      (__nv_bfloat16*)y_bf16, mean, rstd);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_layernorm_rows_bwd(int mode, const void* src0_bf16, const void* src1_bf16, const void* dy_bf16,
                           long long rows, int C, int C0, int HPc, int WPc, const float* gamma, const float* mean,
                           const float* rstd, void* dx0_bf16, int accumulate0, void* dx1_bf16, int accumulate1,
                           float* ws, int nchunk, float* dgamma, float* dbeta, void* stream) {
  RowMap m;
  const int st = rowmap_check(m, mode, rows, C, C0, HPc, WPc);
  if (st != FDX_OK) return st;
  FDX_REQUIRE(src0_bf16 && (mode != LN_CONCAT || (src1_bf16 && dx1_bf16)) && dy_bf16 && gamma && mean && rstd &&
                  dx0_bf16 && ws && dgamma && dbeta, "layernorm_rows_bwd: null pointer");
  FDX_REQUIRE(nchunk > 0 && nchunk <= 65535, "layernorm_rows_bwd: nchunk=%d", nchunk);
  FDX_REQUIRE(aligned16(src0_bf16) && (!src1_bf16 || aligned16(src1_bf16)) && aligned16(dy_bf16) &&
                  aligned16(dx0_bf16) && (!dx1_bf16 || aligned16(dx1_bf16)) && aligned16(gamma),
              "layernorm_rows_bwd: tensors must be 16-byte aligned");
  const long long per = (rows + nchunk - 1) / nchunk;
  const int nblk = (int)((rows + per - 1) / per);
  cudaStream_t s = (cudaStream_t)stream;
  ln_rows_bwd_kernel<<<nblk, 256, 0, s>>>(m, (const __nv_bfloat16*)src0_bf16, (const __nv_bfloat16*)src1_bf16,
                                          (const __nv_bfloat16*)dy_bf16, rows, per, gamma, mean, rstd,
                                          (__nv_bfloat16*)dx0_bf16, accumulate0, (__nv_bfloat16*)dx1_bf16,
                                          accumulate1, ws);
  FDX_LAUNCH_CHECK();
  ln_rows_param_finish_kernel<<<(C + 255) / 256, 256, 0, s>>>(ws, nblk, C, dgamma, dbeta);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
