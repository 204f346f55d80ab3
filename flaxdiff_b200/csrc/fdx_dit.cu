// fdx_dit.cu -- the HBM-bound kernels of the SimpleDiT denoiser (flaxdiff/models/simple_dit.py:23-306) that sit around
// the GEMM engine (fdx_gemm) and the fused attention (fdx_attention_fwd / _bwd): adaLN LayerNorm forward / backward,
// the gated residual, RoPE on the fused QKV output, the tanh-gelu of the MLP, patchify / unpatchify and the Fourier
// timestep features.  bf16 activations, f32 statistics and sums, 16-byte vectors wherever a row allows it.  Every
// column sum is formed in a fixed order (per-chunk partial sums, then an ordered reduction): no atomics, so a step is
// bit-reproducible.
#include "fdx_common.cuh"
#include "../../include/fdx.h"
#include <math.h>

namespace {

inline int stream_grid(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = (long long)fdx_num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

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
// f = p[0..8) or `fill` when p is null
__device__ __forceinline__ void ld8f_or(const float* p, float fill, float (&f)[8]) {
  if (p) {
    ld8f(p, f);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = fill;
  }
}

constexpr int kDitV = 6;            // one warp holds a row of up to 6 x 32 x 8 = 1536 channels
constexpr int kColSlab = 64;        // columns per column-sum block (8 threads x 8 channels)

// ---- adaLN LayerNorm forward: one warp per token ----------------------------------------------------------------
// y = (xhat * gamma + beta) * (1 + ada[b][scale_off + c]) + ada[b][shift_off + c], xhat = (x - mean) * rstd; a null
// gamma / beta / ada drops its term.  The row stays in registers between the mean and the centred-variance pass.
__global__ void __launch_bounds__(256)
dit_adaln_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int L, int C, const float* __restrict__ ada,
                     long long ada_ld, int scale_off, int shift_off, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    float f[kDitV][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < kDitV; ++v) {
      if (v * 32 + lane < nv) {
        ld8(x + r * C + (v * 32 + lane) * 8, f[v]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[v][j];
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < kDitV; ++v) {
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
    const float* arow = ada ? ada + (r / L) * ada_ld : nullptr;
#pragma unroll
    for (int v = 0; v < kDitV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float g[8], b[8], sc[8], sh[8], o[8];
        ld8f_or(gamma ? gamma + c : nullptr, 1.f, g);
        ld8f_or(beta ? beta + c : nullptr, 0.f, b);
        ld8f_or(arow ? arow + scale_off + c : nullptr, 0.f, sc);
        ld8f_or(arow ? arow + shift_off + c : nullptr, 0.f, sh);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(fmaf(f[v][j] * rstd, g[j], b[j]), 1.f + sc[j], sh[j]);
        st8(y + r * C + c, o);
      }
    }
  }
}

// ---- adaLN LayerNorm backward, data gradient: one warp per token --------------------------------------------------
// dxhat = dy * gamma * (1 + scale[b]);  dx = rstd * (dxhat - mean(dxhat) - xhat * mean(dxhat * xhat)) (+ addend).
// dx may alias addend.
__global__ void __launch_bounds__(256)
dit_adaln_bwd_dx_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, long long rows,
                        int L, int C, const float* __restrict__ ada, long long ada_ld, int scale_off,
                        const float* __restrict__ gamma, const float* __restrict__ mean,
                        const float* __restrict__ rstd, const __nv_bfloat16* addend, __nv_bfloat16* dx) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    const float mu = mean[r], rs = rstd[r];
    const float* arow = ada ? ada + (r / L) * ada_ld : nullptr;
    float xh[kDitV][8], g[kDitV][8];
    float a = 0.f, q = 0.f;
#pragma unroll
    for (int v = 0; v < kDitV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float ga[8], sc[8];
        ld8(x + r * C + c, xh[v]);
        ld8(dy + r * C + c, g[v]);
        ld8f_or(gamma ? gamma + c : nullptr, 1.f, ga);
        ld8f_or(arow ? arow + scale_off + c : nullptr, 0.f, sc);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[v][j] = (xh[v][j] - mu) * rs;
          g[v][j] *= ga[j] * (1.f + sc[j]);
          a += g[v][j];
          q = fmaf(g[v][j], xh[v][j], q);
        }
      }
    }
    const float ma = warp_sum(a) / (float)C, mq = warp_sum(q) / (float)C;
#pragma unroll
    for (int v = 0; v < kDitV; ++v) {
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
// partials are added in row order.  ws[b][k][2][C].
//   MODE_LN   : s0 += dy * xhat, s1 += dy               (a = dy, x = the normalised input, mean / rstd per token)
//   MODE_GATE : s0 += dout * y, and dy_out = gate[b] * dout is written (a = dout, x = y)
//   MODE_SUM  : s0 += a
enum { MODE_LN = 0, MODE_GATE = 1, MODE_SUM = 2 };

template <int MODE>
__global__ void __launch_bounds__(256)
dit_colsum_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ x,
                  const float* __restrict__ mean, const float* __restrict__ rstd, int L, int C, int nchunk,
                  const float* __restrict__ gate, long long gate_ld, __nv_bfloat16* __restrict__ dy_out,
                  float* __restrict__ ws) {
  __shared__ float red[2][32][kColSlab];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int k = blockIdx.y, b = blockIdx.z;
  const int c = blockIdx.x * kColSlab + tx * 8;
  const int per = (L + nchunk - 1) / nchunk;
  const int t0 = k * per, t1 = min(L, t0 + per);
  float s0[8], s1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s0[j] = s1[j] = 0.f;
  if (c < C) {
    float gt[8];
    if (MODE == MODE_GATE) ld8f(gate + (long long)b * gate_ld + c, gt);
    for (int t = t0 + ty; t < t1; t += 32) {
      const long long r = (long long)b * L + t;
      float av[8];
      ld8(a + r * C + c, av);
      if (MODE == MODE_SUM) {
#pragma unroll
        for (int j = 0; j < 8; ++j) s0[j] += av[j];
      } else if (MODE == MODE_LN) {
        float xv[8];
        ld8(x + r * C + c, xv);
        const float mu = mean[r], rs = rstd[r];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s0[j] = fmaf(av[j], (xv[j] - mu) * rs, s0[j]);
          s1[j] += av[j];
        }
      } else {
        float xv[8], o[8];
        ld8(x + r * C + c, xv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s0[j] = fmaf(av[j], xv[j], s0[j]);
          o[j] = gt[j] * av[j];
        }
        st8(dy_out + r * C + c, o);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][ty][tx * 8 + j] = s0[j];
    red[1][ty][tx * 8 + j] = s1[j];
  }
  __syncthreads();
  if (threadIdx.x < 2 * kColSlab) {
    const int which = threadIdx.x / kColSlab, col = threadIdx.x % kColSlab;
    const int cc = blockIdx.x * kColSlab + col;
    if (cc < C && (which == 0 || MODE == MODE_LN)) {
      float s = 0.f;
      for (int i = 0; i < 32; ++i) s += red[which][i][col];
      ws[(((long long)b * nchunk + k) * 2 + which) * C + cc] = s;
    }
  }
}

// Second stage: out0[b][c] (+)= scale * sum_k ws[b][k][0][c] (out1 from [1]); reduce_b: out[c] sums every sample too,
// in sample order.
__global__ void dit_colsum_finish_kernel(const float* __restrict__ ws, int B, int nchunk, int C, float scale,
                                         float* out0, long long ld0, float* out1, long long ld1, int reduce_b,
                                         int accumulate) {
  const int nb = reduce_b ? 1 : B;
  const long long total = (long long)nb * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / C), c = (int)(i % C);
    const int b0 = reduce_b ? 0 : b, b1 = reduce_b ? B : b + 1;
    float s0 = 0.f, s1 = 0.f;
    for (int bb = b0; bb < b1; ++bb)
      for (int k = 0; k < nchunk; ++k) {
        const long long base = ((long long)bb * nchunk + k) * 2 * C + c;
        s0 += ws[base];
        if (out1) s1 += ws[base + C];
      }
    float* p0 = out0 + (long long)b * ld0 + c;
    *p0 = accumulate ? *p0 + scale * s0 : scale * s0;
    if (out1) {
      float* p1 = out1 + (long long)b * ld1 + c;
      *p1 = accumulate ? *p1 + scale * s1 : scale * s1;
    }
  }
}

// ---- gated residual: out = x + gate[b][c] * y (out may alias x) ---------------------------------------------------
__global__ void dit_gate_fwd_kernel(const __nv_bfloat16* x, const __nv_bfloat16* __restrict__ y, long long rows,
                                    int L, int C, const float* __restrict__ gate, long long gate_ld,
                                    __nv_bfloat16* out) {
  const int v = C / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    float xv[8], yv[8], g[8];
    ld8(x + r * C + c, xv);
    ld8(y + r * C + c, yv);
    ld8f(gate + (r / L) * gate_ld + c, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) xv[j] = fmaf(g[j], yv[j], xv[j]);
    st8(out + r * C + c, xv);
  }
}

// ---- RoPE (vit_common.py:56-80, 96-104), in place: one warp per (token, head, matrix) ------------------------------
// Pair i < d/2 of a head: (x1, x2) = (x[i], x[i + d/2]) -> (x1 cos - x2 sin, x2 cos + x1 sin) with angle
// l * 10000^(-2i/d), l = token index in its sample; `inverse` applies the transposed rotation (the backward).
// Channels [d, dp) of each dp-wide head are written as zeros.
__global__ void dit_rope_kernel(__nv_bfloat16* __restrict__ base, long long rows, int L, long long ld, int heads,
                                int d, int dp, int nmat, long long mat_off, int inverse) {
  const int lane = threadIdx.x & 31;
  const long long items = rows * heads * nmat;
  const int half = d / 2;
  const float sgn = inverse ? -1.f : 1.f;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < items;
       w += ((long long)gridDim.x * blockDim.x) >> 5) {
    const int m = (int)(w % nmat);
    const long long rh = w / nmat;
    const int h = (int)(rh % heads);
    const long long r = rh / heads;
    const float pos = (float)(r % L);
    __nv_bfloat16* p = base + r * ld + m * mat_off + (long long)h * dp;
    for (int i = lane; i < half; i += 32) {
      const float inv = 1.f / powf(10000.f, (float)(2 * i) / (float)d);
      float sn, cs;
      sincosf(pos * inv, &sn, &cs);
      sn *= sgn;
      const float x1 = __bfloat162float(p[i]), x2 = __bfloat162float(p[i + half]);
      p[i] = __float2bfloat16(x1 * cs - x2 * sn);
      p[i + half] = __float2bfloat16(x2 * cs + x1 * sn);
    }
    for (int j = d + lane; j < dp; j += 32) p[j] = __float2bfloat16(0.f);
  }
}

// ---- tanh-approximated gelu (jax.nn.gelu's default) ----------------------------------------------------------------
constexpr float kGeluK = 0.7978845608028654f;   // sqrt(2 / pi)
constexpr float kGeluC = 0.044715f;

__global__ void dit_bias_gelu_tanh_kernel(const __nv_bfloat16* x, long long rows, int C,
                                          const float* __restrict__ bias, __nv_bfloat16* y) {
  const int v = C / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    float f[8], b[8];
    ld8(x + r * C + c, f);
    ld8f_or(bias ? bias + c : nullptr, 0.f, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = f[j] + b[j];
      f[j] = 0.5f * z * (1.f + tanhf(kGeluK * fmaf(kGeluC * z, z * z, z)));
    }
    st8(y + r * C + c, f);
  }
}

// dx = dy * gelu_tanh'(x + bias)
__global__ void dit_bias_gelu_tanh_bwd_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C,
                                              const float* __restrict__ bias, const __nv_bfloat16* dy,
                                              __nv_bfloat16* dx) {
  const int v = C / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    float f[8], b[8], g[8];
    ld8(x + r * C + c, f);
    ld8(dy + r * C + c, g);
    ld8f_or(bias ? bias + c : nullptr, 0.f, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = f[j] + b[j];
      const float th = tanhf(kGeluK * fmaf(kGeluC * z, z * z, z));
      const float dth = (1.f - th * th) * kGeluK * fmaf(3.f * kGeluC, z * z, 1.f);
      g[j] *= 0.5f * (1.f + th) + 0.5f * z * dth;
    }
    st8(dx + r * C + c, g);
  }
}

// ---- patchify / unpatchify (raster patch order) -------------------------------------------------------------------
// dst[b * L + hp * WP + wp][(p1 * p + p2) * C + c] = src[b][hp * p + p1][wp * p + p2][c]; columns [p*p*C, ld) = 0.
template <typename T>
__global__ void dit_patchify_kernel(const T* __restrict__ src, int B, int H, int W, int C, int p, int ld,
                                    __nv_bfloat16* __restrict__ dst) {
  const int HP = H / p, WP = W / p, K = p * p * C, v = ld / 8;
  const long long total = (long long)B * HP * WP * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / v;
    const int c0 = (int)(i % v) * 8;
    const int wp = (int)(row % WP), hp = (int)((row / WP) % HP), b = (int)(row / ((long long)WP * HP));
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = c0 + j;
      float val = 0.f;
      if (col < K) {
        const int c = col % C, p2 = (col / C) % p, p1 = col / (C * p);
        const long long s = (((long long)b * H + hp * p + p1) * W + wp * p + p2) * C + c;
        if constexpr (sizeof(T) == 4)
          val = src[s];
        else
          val = __bfloat162float(src[s]);
      }
      f[j] = val;
    }
    st8(dst + row * ld + c0, f);
  }
}

// dst[b][h][w][c] = src[b * L + (h / p) * WP + w / p][((h % p) * p + w % p) * C + c]  (f32 -> f32)
__global__ void dit_unpatchify_kernel(const float* __restrict__ src, int ld, int B, int H, int W, int C, int p,
                                      float* __restrict__ dst) {
  const int WP = W / p, HP = H / p;
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
    const long long row = ((long long)b * HP + h / p) * WP + w / p;
    dst[i] = src[row * ld + ((h % p) * p + w % p) * C + c];
  }
}

// ---- Fourier timestep features (models/common.py:97-110): [sin(t w), cos(t w)], w = 2 pi freqs --------------------
__global__ void dit_fourier_kernel(const float* __restrict__ t, int B, const float* __restrict__ freqs, int half,
                                   __nv_bfloat16* __restrict__ out) {
  const long long total = (long long)B * 2 * half;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / (2 * half)), j = (int)(i % (2 * half));
    const float w = 6.283185307179586f * freqs[j % half];
    const float arg = t[b] * w;
    out[i] = __float2bfloat16(j < half ? sinf(arg) : cosf(arg));
  }
}

int colsum_launch(int mode, const void* a, const void* x, const float* mean, const float* rstd, int B, int L, int C,
                  const float* gate, long long gate_ld, void* dy_out, float* ws, int nchunk, float scale, float* out0,
                  long long ld0, float* out1, long long ld1, int reduce_b, int accumulate, cudaStream_t st) {
  FDX_REQUIRE(ws && nchunk > 0 && nchunk <= 65535 && B <= 65535, "dit colsum: bad workspace / sizes");
  const dim3 grid((C + kColSlab - 1) / kColSlab, nchunk, B);
  const __nv_bfloat16* a16 = (const __nv_bfloat16*)a;
  const __nv_bfloat16* x16 = (const __nv_bfloat16*)x;
  if (mode == MODE_LN)
    dit_colsum_kernel<MODE_LN><<<grid, 256, 0, st>>>(a16, x16, mean, rstd, L, C, nchunk, nullptr, 0, nullptr, ws);
  else if (mode == MODE_GATE)
    dit_colsum_kernel<MODE_GATE><<<grid, 256, 0, st>>>(a16, x16, nullptr, nullptr, L, C, nchunk, gate, gate_ld,
                                                       (__nv_bfloat16*)dy_out, ws);
  else
    dit_colsum_kernel<MODE_SUM><<<grid, 256, 0, st>>>(a16, nullptr, nullptr, nullptr, L, C, nchunk, nullptr, 0,
                                                      nullptr, ws);
  FDX_LAUNCH_CHECK();
  dit_colsum_finish_kernel<<<stream_grid((long long)(reduce_b ? 1 : B) * C, 256), 256, 0, st>>>(
      ws, B, nchunk, C, scale, out0, ld0, out1, ld1, reduce_b, accumulate);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

inline bool row_ok(int C) { return C > 0 && C % 8 == 0 && C <= 32 * 8 * kDitV; }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// fdx_bias_act's FDX_ACT_GELU_TANH (declared in fdx_clip.cu, which owns the entry point)
int fdx_dit_bias_gelu_tanh(const void* x_bf16, long long rows, int C, const float* bias, void* y_bf16, void* stream) {
  dit_bias_gelu_tanh_kernel<<<stream_grid(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, rows, C, bias, (__nv_bfloat16*)y_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

extern "C" {

int fdx_dit_adaln_fwd(const void* x_bf16, long long rows, int L, int C, const float* ada, long long ada_ld,
                      int scale_off, int shift_off, const float* gamma, const float* beta, float eps, void* y_bf16,
                      float* mean, float* rstd, void* stream) {
  FDX_REQUIRE(x_bf16 && y_bf16, "dit_adaln_fwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && row_ok(C),
              "dit_adaln_fwd: C=%d must be a multiple of 8, <= %d; rows a multiple of L", C, 32 * 8 * kDitV);
  FDX_REQUIRE(!(ada && gamma), "dit_adaln_fwd: either the ada modulation or the affine parameters, not both");
  FDX_REQUIRE(!ada || (ada_ld % 4 == 0 && scale_off % 8 == 0 && shift_off % 8 == 0 && aligned16(ada)),
              "dit_adaln_fwd: ada rows and chunk offsets must be 32-byte aligned");
  FDX_REQUIRE((mean == nullptr) == (rstd == nullptr), "dit_adaln_fwd: mean and rstd go together");
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_bf16) && (!gamma || aligned16(gamma)) && (!beta || aligned16(beta)),
              "dit_adaln_fwd: tensors must be 16-byte aligned");
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  dit_adaln_fwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, rows, L, C, ada, ada_ld, scale_off, shift_off, gamma, beta, eps,
      (__nv_bfloat16*)y_bf16, mean, rstd);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_adaln_bwd(const void* x_bf16, const void* dy_bf16, long long rows, int L, int C, const float* ada,
                      long long ada_ld, int scale_off, const float* gamma, const float* mean, const float* rstd,
                      const void* addend_bf16, void* dx_bf16, float* ws, int nchunk, float* d0, long long d0_ld,
                      float* d1, long long d1_ld, int reduce_samples, int accumulate, void* stream) {
  FDX_REQUIRE(x_bf16 && dy_bf16 && dx_bf16 && mean && rstd && d0 && d1, "dit_adaln_bwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && row_ok(C),
              "dit_adaln_bwd: C=%d must be a multiple of 8, <= %d; rows a multiple of L", C, 32 * 8 * kDitV);
  FDX_REQUIRE(!(ada && gamma), "dit_adaln_bwd: either the ada modulation or the affine parameters, not both");
  FDX_REQUIRE(!ada || (ada_ld % 4 == 0 && scale_off % 8 == 0 && aligned16(ada)),
              "dit_adaln_bwd: ada rows and chunk offsets must be 32-byte aligned");
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(dy_bf16) && aligned16(dx_bf16) &&
                  (!addend_bf16 || aligned16(addend_bf16)) && (!gamma || aligned16(gamma)),
              "dit_adaln_bwd: tensors must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int s = colsum_launch(MODE_LN, dy_bf16, x_bf16, mean, rstd, (int)(rows / L), L, C, nullptr, 0, nullptr, ws,
                              nchunk, 1.f, d0, d0_ld, d1, d1_ld, reduce_samples, accumulate, st);
  if (s != FDX_OK) return s;
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  dit_adaln_bwd_dx_kernel<<<(int)grid, 256, 0, st>>>(
      (const __nv_bfloat16*)x_bf16, (const __nv_bfloat16*)dy_bf16, rows, L, C, ada, ada_ld, scale_off, gamma, mean,
      rstd, (const __nv_bfloat16*)addend_bf16, (__nv_bfloat16*)dx_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_gate_fwd(const void* x_bf16, const void* y_bf16, long long rows, int L, int C, const float* gate,
                     long long gate_ld, void* out_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && y_bf16 && gate && out_bf16, "dit_gate_fwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && C > 0 && C % 8 == 0 && gate_ld % 4 == 0,
              "dit_gate_fwd: bad sizes (C=%d a multiple of 8)", C);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_bf16) && aligned16(gate) && aligned16(out_bf16),
              "dit_gate_fwd: tensors must be 16-byte aligned");
  dit_gate_fwd_kernel<<<stream_grid(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, (const __nv_bfloat16*)y_bf16, rows, L, C, gate, gate_ld,
      (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_gate_bwd(const void* dout_bf16, const void* y_bf16, long long rows, int L, int C, const float* gate,
                     long long gate_ld, void* dy_bf16, float* ws, int nchunk, float* dgate, long long dgate_ld,
                     void* stream) {
  FDX_REQUIRE(dout_bf16 && y_bf16 && gate && dy_bf16 && dgate, "dit_gate_bwd: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && C > 0 && C % 8 == 0 && gate_ld % 4 == 0,
              "dit_gate_bwd: bad sizes (C=%d a multiple of 8)", C);
  FDX_REQUIRE(aligned16(dout_bf16) && aligned16(y_bf16) && aligned16(gate) && aligned16(dy_bf16),
              "dit_gate_bwd: tensors must be 16-byte aligned");
  return colsum_launch(MODE_GATE, dout_bf16, y_bf16, nullptr, nullptr, (int)(rows / L), L, C, gate, gate_ld, dy_bf16,
                       ws, nchunk, 1.f, dgate, dgate_ld, nullptr, 0, 0, 0, (cudaStream_t)stream);
}

int fdx_dit_token_mean(const void* x_bf16, int B, int T, int C, float* ws, int nchunk, float* out, void* stream) {
  FDX_REQUIRE(x_bf16 && out, "dit_token_mean: null pointer");
  FDX_REQUIRE(B > 0 && T > 0 && C > 0 && C % 8 == 0 && aligned16(x_bf16), "dit_token_mean: bad sizes (C=%d)", C);
  return colsum_launch(MODE_SUM, x_bf16, nullptr, nullptr, nullptr, B, T, C, nullptr, 0, nullptr, ws, nchunk,
                       1.f / (float)T, out, C, nullptr, 0, 0, 0, (cudaStream_t)stream);
}

int fdx_dit_rope(void* base_bf16, long long rows, int L, long long ld, int heads, int d, int dp, int nmat,
                 long long mat_off, int inverse, void* stream) {
  FDX_REQUIRE(base_bf16, "dit_rope: null pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && heads > 0 && d > 0 && d % 2 == 0 && dp >= d && nmat >= 1,
              "dit_rope: bad sizes (d=%d must be even, <= dp=%d)", d, dp);
  FDX_REQUIRE(ld >= (long long)(nmat - 1) * mat_off + (long long)heads * dp, "dit_rope: row stride too small");
  const long long warps = rows * heads * nmat;
  dit_rope_kernel<<<stream_grid(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)base_bf16, rows, L, ld, heads, d, dp, nmat, mat_off, inverse);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_bias_act_bwd(const void* x_bf16, long long rows, int C, const float* bias, int act, const void* dy_bf16,
                     void* dx_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && dy_bf16 && dx_bf16, "bias_act_bwd: null pointer");
  FDX_REQUIRE(act == FDX_ACT_GELU_TANH, "bias_act_bwd: activation %d has no backward (only tanh-gelu)", act);
  FDX_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, "bias_act_bwd: C=%d must be a multiple of 8", C);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(dy_bf16) && aligned16(dx_bf16) && (!bias || aligned16(bias)),
              "bias_act_bwd: tensors must be 16-byte aligned");
  dit_bias_gelu_tanh_bwd_kernel<<<stream_grid(rows * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, rows, C, bias, (const __nv_bfloat16*)dy_bf16, (__nv_bfloat16*)dx_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_patchify(const void* src, int src_f32, int B, int H, int W, int C, int p, int ld, void* dst_bf16,
                     void* stream) {
  FDX_REQUIRE(src && dst_bf16, "dit_patchify: null pointer");
  FDX_REQUIRE(B > 0 && C > 0 && p > 0 && H > 0 && W > 0 && H % p == 0 && W % p == 0,
              "dit_patchify: H=%d, W=%d must be multiples of the patch size %d", H, W, p);
  FDX_REQUIRE(ld >= p * p * C && ld % 8 == 0 && aligned16(dst_bf16), "dit_patchify: ld=%d must be >= p*p*C and a "
              "multiple of 8, dst 16-byte aligned", ld);
  const long long items = (long long)B * (H / p) * (W / p) * (ld / 8);
  const int grid = stream_grid(items, 256);
  if (src_f32)
    dit_patchify_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)src, B, H, W, C, p, ld,
                                                                       (__nv_bfloat16*)dst_bf16);
  else
    dit_patchify_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)src, B, H, W, C, p, ld, (__nv_bfloat16*)dst_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_unpatchify(const float* src, int ld, int B, int H, int W, int C, int p, float* dst, void* stream) {
  FDX_REQUIRE(src && dst, "dit_unpatchify: null pointer");
  FDX_REQUIRE(B > 0 && C > 0 && p > 0 && H > 0 && W > 0 && H % p == 0 && W % p == 0 && ld >= p * p * C,
              "dit_unpatchify: bad sizes (H=%d, W=%d, p=%d, ld=%d)", H, W, p, ld);
  dit_unpatchify_kernel<<<stream_grid((long long)B * H * W * C, 256), 256, 0, (cudaStream_t)stream>>>(
      src, ld, B, H, W, C, p, dst);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_dit_fourier(const float* t, int B, const float* freqs, int half, void* out_bf16, void* stream) {
  FDX_REQUIRE(t && freqs && out_bf16 && B > 0 && half > 0, "dit_fourier: bad arguments");
  dit_fourier_kernel<<<stream_grid((long long)B * 2 * half, 256), 256, 0, (cudaStream_t)stream>>>(
      t, B, freqs, half, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
