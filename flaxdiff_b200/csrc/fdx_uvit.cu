// fdx_uvit.cu -- the glue kernels of UViT (flaxdiff/models/simple_vit.py:18-250) that sit around the GEMM engine, the
// fused attention and the UNet's transformer-block program:
//   * the token sequence [patches + pos | time | text] and its gradient's split, with the learned position table's
//     batch-reduced gradient;
//   * the optional output head's per-pixel LayerNorm over 64 channels fused with swish or mish, and its backward;
//   * the 6-channel im2col that feeds final_conv1 over concat([x, x_image]) without writing the concat.
// bf16 activations, f32 statistics and sums, 16-byte vectors.  Every reduction runs in a fixed order (per-block
// partial sums, then an ordered pass): no atomics, so a step is bit-reproducible.
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
__device__ __forceinline__ void st8f(float* p, const float (&f)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

// ---- sequence assembly ---------------------------------------------------------------------------------------------
// Row r = b L + s of the stream (L = N + 1 + T): s < N is bf16(f32(patch[b N + s]) + pos[s]) (simple_vit.py:194, the
// bf16 patches promoted by the f32 table and rounded once to the stream's storage), s = N the time token, the rest
// text_proj's rows.  One thread per 8 columns.
__global__ void __launch_bounds__(256)
uvit_assemble_fwd_kernel(const __nv_bfloat16* __restrict__ patch, const float* __restrict__ pos,
                         const __nv_bfloat16* __restrict__ time_tok, const __nv_bfloat16* __restrict__ text, int B,
                         int N, int T, int F, __nv_bfloat16* __restrict__ out) {
  const int L = N + 1 + T, F8 = F / 8;
  const long long total = (long long)B * L * F8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / F8;
    const int c = (int)(i - r * F8) * 8;
    const int b = (int)(r / L), s = (int)(r - (long long)b * L);
    __nv_bfloat16* dst = out + r * F + c;
    if (s < N) {
      float v[8], p[8];
      ld8(patch + ((long long)b * N + s) * F + c, v);
      ld8f(pos + (long long)s * F + c, p);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += p[j];
      st8(dst, v);
    } else {
      const __nv_bfloat16* src = s == N ? time_tok + (long long)b * F + c
                                        : text + ((long long)b * T + (s - N - 1)) * F + c;
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    }
  }
}

// The stream gradient's rows go back to where they came from: the patch rows (bf16, for the embedding's GEMMs), the
// time token (f32, for fdx_time_embed_bwd) and the text rows (bf16, for text_proj's GEMMs).
__global__ void __launch_bounds__(256)
uvit_split_bwd_kernel(const __nv_bfloat16* __restrict__ dx, int B, int N, int T, int F,
                      __nv_bfloat16* __restrict__ dpatch, float* __restrict__ dtime, __nv_bfloat16* __restrict__ dtext) {
  const int L = N + 1 + T, F8 = F / 8;
  const long long total = (long long)B * L * F8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / F8;
    const int c = (int)(i - r * F8) * 8;
    const int b = (int)(r / L), s = (int)(r - (long long)b * L);
    const uint4 u = *reinterpret_cast<const uint4*>(dx + r * F + c);
    if (s < N) {
      *reinterpret_cast<uint4*>(dpatch + ((long long)b * N + s) * F + c) = u;
    } else if (s == N) {
      if (dtime) {
        float v[8];
        ld8(dx + r * F + c, v);
        st8f(dtime + (long long)b * F + c, v);
      }
    } else if (dtext) {
      *reinterpret_cast<uint4*>(dtext + ((long long)b * T + (s - N - 1)) * F + c) = u;
    }
  }
}

// d pos[s] = sum_b dx[b, s] for s < N, in two ordered stages: split g sums the samples [g per, (g + 1) per) in order
// into ws[g][s][:], then one pass adds the nsplit partials in split order onto dpos.
__global__ void __launch_bounds__(256)
uvit_pos_partial_kernel(const __nv_bfloat16* __restrict__ dx, int B, int N, int L, int F, int per,
                        float* __restrict__ ws) {
  const int F8 = F / 8;
  const long long items = (long long)N * F8;
  const int g = blockIdx.y;
  const int b0 = g * per, b1 = min(B, b0 + per);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items;
       i += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(i / F8), c = (int)(i - (long long)s * F8) * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int b = b0; b < b1; ++b) {
      float v[8];
      ld8(dx + ((long long)b * L + s) * F + c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
    st8f(ws + ((long long)g * N + s) * F + c, acc);
  }
}

__global__ void __launch_bounds__(256)
uvit_pos_finish_kernel(const float* __restrict__ ws, int nsplit, long long items, float* __restrict__ dpos) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items;
       i += (long long)gridDim.x * blockDim.x) {
    float a = dpos[i];
    for (int g = 0; g < nsplit; ++g) a += ws[(long long)g * items + i];
    dpos[i] = a;
  }
}

// ---- the output head's LayerNorm(64) + activation --------------------------------------------------------------------
// final_norm_conv + activation (simple_vit.py:240-241): per pixel, y = act(xhat gamma + beta) over C = 64 channels,
// xhat = (x - mean) rstd with f32 centred statistics.  Eight threads hold a pixel's row (8 channels each); a 256-thread
// block works on 32 pixels at a time.
constexpr int kC = 64;
constexpr int kPixPerIter = 32;
enum { ACT_SWISH = 1, ACT_MISH = 2 };

__device__ __forceinline__ float group8_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  return v;
}
__device__ __forceinline__ float sigmoid_f(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }
template <int ACT>
__device__ __forceinline__ float act_f(float z) {
  return ACT == ACT_MISH ? mish_f(z) : z * sigmoid_f(z);
}
template <int ACT>
__device__ __forceinline__ float act_grad(float z) {
  if (ACT == ACT_MISH) return mish_grad(z);
  const float s = sigmoid_f(z);
  return fmaf(z * s, 1.f - s, s);
}

// the row's statistics: two passes over the registers (mean, then the centred variance)
__device__ __forceinline__ void row_stats(const float (&v)[8], float eps, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) s += v[j];
  mean = group8_sum(s) * (1.f / kC);
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float d = v[j] - mean;
    q = fmaf(d, d, q);
  }
  rstd = rsqrtf(group8_sum(q) * (1.f / kC) + eps);
}

template <int ACT>
__global__ void __launch_bounds__(256)
uvit_head_norm_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long pixels, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y) {
  const int c = (threadIdx.x & 7) * 8;
  float g[8], bb[8];
  ld8f(gamma + c, g);
  ld8f(beta + c, bb);
  // every lane of a warp runs the same number of iterations (the shuffles need the full warp)
  for (long long base = (long long)blockIdx.x * kPixPerIter; base < pixels; base += (long long)gridDim.x * kPixPerIter) {
    const long long p = base + (threadIdx.x >> 3);
    const bool ok = p < pixels;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (ok) ld8(x + p * kC + c, v);
    float mean, rstd;
    row_stats(v, eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = act_f<ACT>(fmaf((v[j] - mean) * rstd, g[j], bb[j]));
    if (ok) st8(y + p * kC + c, v);
  }
}

// dz = dy act'(z), dxhat = dz gamma, dx = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)).  Block k owns the pixels
// [k per, (k + 1) per) and writes its dgamma / dbeta partial sums to ws[k][2][64] in a fixed order; the finish kernel
// adds the blocks' partials in block order.
template <int ACT>
__global__ void __launch_bounds__(256)
uvit_head_norm_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, long long pixels,
                          long long per, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          __nv_bfloat16* __restrict__ dx, float* __restrict__ ws) {
  __shared__ float red[2][256 / 8][kC];
  const int c = (threadIdx.x & 7) * 8, grp = threadIdx.x >> 3;
  float ag[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ab[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const long long p0 = (long long)blockIdx.x * per;
  const long long p1 = p0 + per < pixels ? p0 + per : pixels;
  for (long long base = p0; base < p1; base += kPixPerIter) {
    const long long p = base + grp;
    const bool ok = p < p1;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (ok) {
      ld8(x + p * kC + c, v);
      ld8(dy + p * kC + c, d);
    }
    float mean, rstd;
    row_stats(v, eps, mean, rstd);
    float g[8], bb[8];      // re-read from L1 each pixel: kept live across the loop they push the kernel into spills
    ld8f(gamma + c, g);
    ld8f(beta + c, bb);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float xh = (v[j] - mean) * rstd;
      const float dz = d[j] * act_grad<ACT>(fmaf(xh, g[j], bb[j]));
      ag[j] = fmaf(dz, xh, ag[j]);
      ab[j] += dz;
      const float dxh = dz * g[j];
      s1 += dxh;
      s2 = fmaf(dxh, xh, s2);
      v[j] = xh;
      d[j] = dxh;
    }
    s1 = group8_sum(s1) * (1.f / kC);
    s2 = group8_sum(s2) * (1.f / kC);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = rstd * (d[j] - s1 - v[j] * s2);
    if (ok) st8(dx + p * kC + c, d);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][grp][c + j] = ag[j];
    red[1][grp][c + j] = ab[j];
  }
  __syncthreads();
  if (threadIdx.x < 2 * kC) {
    const int k = threadIdx.x / kC, ch = threadIdx.x % kC;
    float a = 0.f;
    for (int r = 0; r < 256 / 8; ++r) a += red[k][r][ch];
    ws[((long long)blockIdx.x * 2 + k) * kC + ch] = a;
  }
}

__global__ void __launch_bounds__(128)
uvit_head_norm_finish_kernel(const float* __restrict__ ws, int nblk, float* __restrict__ dgamma,
                             float* __restrict__ dbeta) {
  const int k = threadIdx.x / kC, ch = threadIdx.x % kC;
  float a = 0.f;
  for (int i = 0; i < nblk; ++i) a += ws[((long long)i * 2 + k) * kC + ch];
  float* dst = k == 0 ? dgamma : dbeta;
  dst[ch] += a;
}

// ---- im2col over two 3-channel tensors --------------------------------------------------------------------------------
// col[p][t*3 + k] = bf16(src0[p + d(t)][k]) and col[p][32 + t*3 + k] = bf16(src1[p + d(t)][k]), d(t) = (t/3 - 1,
// t%3 - 1), zero outside the image and in columns 27..31 and 59..63: final_conv1's K = 64 operand over concat([src0,
// src1], -1) with its 54 real taps, the concatenation never written.
template <bool F32>
__device__ __forceinline__ float ld_in(const void* p, long long i) {
  if (F32) return __bfloat162float(__float2bfloat16_rn(reinterpret_cast<const float*>(p)[i]));
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}

template <bool F32_0, bool F32_1>
__global__ void __launch_bounds__(256)
uvit_im2col_c6_kernel(const void* __restrict__ src0, const void* __restrict__ src1, int N, int H, int W,
                      __nv_bfloat16* __restrict__ col) {
  const long long npix = (long long)N * H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix;
       p += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    float v[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) v[j] = 0.f;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int sy = py + t / 3 - 1, sx = px + t % 3 - 1;
      if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
      const long long q = (p + (long long)(t / 3 - 1) * W + (t % 3 - 1)) * 3;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        v[t * 3 + k] = ld_in<F32_0>(src0, q + k);
        v[32 + t * 3 + k] = ld_in<F32_1>(src1, q + k);
      }
    }
    uint4* o = reinterpret_cast<uint4*>(col + p * 64);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint4 u;
      u.x = pack_bf16x2(v[8 * j], v[8 * j + 1]); u.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
      u.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]); u.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
      o[j] = u;
    }
  }
}

template <bool F32_0>
void im2col_c6_launch(const void* src0, const void* src1, int src1_is_f32, int N, int H, int W, void* col, int grid,
                      cudaStream_t s) {
  if (src1_is_f32)
    uvit_im2col_c6_kernel<F32_0, true><<<grid, 256, 0, s>>>(src0, src1, N, H, W, (__nv_bfloat16*)col);
  else
    uvit_im2col_c6_kernel<F32_0, false><<<grid, 256, 0, s>>>(src0, src1, N, H, W, (__nv_bfloat16*)col);
}

}  // namespace

extern "C" {

int fdx_uvit_assemble_fwd(const void* patch_bf16, const float* pos, const void* time_bf16, const void* text_bf16,
                          int B, int N, int T, int F, void* out_bf16, void* stream) {
  FDX_REQUIRE(patch_bf16 && pos && time_bf16 && out_bf16 && (T == 0 || text_bf16), "uvit_assemble_fwd: null pointer");
  FDX_REQUIRE(B > 0 && N > 0 && T >= 0 && F > 0 && F % 8 == 0,
              "uvit_assemble_fwd: bad sizes B=%d N=%d T=%d F=%d (F a multiple of 8)", B, N, T, F);
  FDX_REQUIRE(aligned16(patch_bf16) && aligned16(pos) && aligned16(time_bf16) && aligned16(out_bf16) &&
                  (!text_bf16 || aligned16(text_bf16)), "uvit_assemble_fwd: tensors must be 16-byte aligned");
  uvit_assemble_fwd_kernel<<<stream_grid((long long)B * (N + 1 + T) * (F / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)patch_bf16, pos, (const __nv_bfloat16*)time_bf16, (const __nv_bfloat16*)text_bf16, B, N,
      T, F, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_uvit_assemble_bwd(const void* dx_bf16, int B, int N, int T, int F, void* dpatch_bf16, float* dtime,
                          void* dtext_bf16, float* ws, int nsplit, float* dpos, void* stream) {
  FDX_REQUIRE(dx_bf16 && dpatch_bf16 && ws && dpos, "uvit_assemble_bwd: null pointer");
  FDX_REQUIRE(B > 0 && N > 0 && T >= 0 && F > 0 && F % 8 == 0,
              "uvit_assemble_bwd: bad sizes B=%d N=%d T=%d F=%d (F a multiple of 8)", B, N, T, F);
  FDX_REQUIRE(nsplit > 0 && nsplit <= B && nsplit <= 65535, "uvit_assemble_bwd: nsplit=%d must be in [1, B]", nsplit);
  FDX_REQUIRE(aligned16(dx_bf16) && aligned16(dpatch_bf16) && aligned16(ws) && aligned16(dpos) &&
                  (!dtime || aligned16(dtime)) && (!dtext_bf16 || aligned16(dtext_bf16)),
              "uvit_assemble_bwd: tensors must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int L = N + 1 + T;
  uvit_split_bwd_kernel<<<stream_grid((long long)B * L * (F / 8), 256), 256, 0, s>>>(
      (const __nv_bfloat16*)dx_bf16, B, N, T, F, (__nv_bfloat16*)dpatch_bf16, dtime, (__nv_bfloat16*)dtext_bf16);
  FDX_LAUNCH_CHECK();
  const int per = (B + nsplit - 1) / nsplit;
  const int used = (B + per - 1) / per;
  const long long items8 = (long long)N * (F / 8);
  long long gx = (items8 + 255) / 256;
  const long long cap = ((long long)fdx_num_sms() * 8 + used - 1) / used;
  if (gx > cap) gx = cap;
  uvit_pos_partial_kernel<<<dim3((unsigned)gx, (unsigned)used), 256, 0, s>>>((const __nv_bfloat16*)dx_bf16, B, N, L,
                                                                             F, per, ws);
  FDX_LAUNCH_CHECK();
  uvit_pos_finish_kernel<<<stream_grid((long long)N * F, 256), 256, 0, s>>>(ws, used, (long long)N * F, dpos);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_uvit_head_norm_fwd(const void* x_bf16, long long pixels, const float* gamma, const float* beta, float eps,
                           int act, void* y_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && gamma && beta && y_bf16, "uvit_head_norm_fwd: null pointer");
  FDX_REQUIRE(pixels > 0, "uvit_head_norm_fwd: pixels=%lld", pixels);
  FDX_REQUIRE(act == ACT_SWISH || act == ACT_MISH, "uvit_head_norm_fwd: act=%d (1 = swish, 2 = mish)", act);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(gamma) && aligned16(beta) && aligned16(y_bf16),
              "uvit_head_norm_fwd: tensors must be 16-byte aligned");
  long long grid = (pixels + kPixPerIter - 1) / kPixPerIter;
  if (grid > (long long)fdx_num_sms() * 8) grid = (long long)fdx_num_sms() * 8;
  cudaStream_t s = (cudaStream_t)stream;
  if (act == ACT_MISH)
    uvit_head_norm_fwd_kernel<ACT_MISH><<<(int)grid, 256, 0, s>>>((const __nv_bfloat16*)x_bf16, pixels, gamma, beta,
                                                                  eps, (__nv_bfloat16*)y_bf16);
  else
    uvit_head_norm_fwd_kernel<ACT_SWISH><<<(int)grid, 256, 0, s>>>((const __nv_bfloat16*)x_bf16, pixels, gamma, beta,
                                                                   eps, (__nv_bfloat16*)y_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_uvit_head_norm_bwd(const void* x_bf16, const void* dy_bf16, long long pixels, const float* gamma,
                           const float* beta, float eps, int act, void* dx_bf16, float* ws, int nchunk, float* dgamma,
                           float* dbeta, void* stream) {
  FDX_REQUIRE(x_bf16 && dy_bf16 && gamma && beta && dx_bf16 && ws && dgamma && dbeta,
              "uvit_head_norm_bwd: null pointer");
  FDX_REQUIRE(pixels > 0, "uvit_head_norm_bwd: pixels=%lld", pixels);
  FDX_REQUIRE(act == ACT_SWISH || act == ACT_MISH, "uvit_head_norm_bwd: act=%d (1 = swish, 2 = mish)", act);
  FDX_REQUIRE(nchunk > 0 && nchunk <= 65535, "uvit_head_norm_bwd: nchunk=%d", nchunk);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(dy_bf16) && aligned16(gamma) && aligned16(beta) && aligned16(dx_bf16),
              "uvit_head_norm_bwd: tensors must be 16-byte aligned");
  long long per = (pixels + nchunk - 1) / nchunk;
  per = (per + kPixPerIter - 1) / kPixPerIter * kPixPerIter;
  const int nblk = (int)((pixels + per - 1) / per);
  cudaStream_t s = (cudaStream_t)stream;
  if (act == ACT_MISH)
    uvit_head_norm_bwd_kernel<ACT_MISH><<<nblk, 256, 0, s>>>((const __nv_bfloat16*)x_bf16,
                                                             (const __nv_bfloat16*)dy_bf16, pixels, per, gamma, beta,
                                                             eps, (__nv_bfloat16*)dx_bf16, ws);
  else
    uvit_head_norm_bwd_kernel<ACT_SWISH><<<nblk, 256, 0, s>>>((const __nv_bfloat16*)x_bf16,
                                                              (const __nv_bfloat16*)dy_bf16, pixels, per, gamma, beta,
                                                              eps, (__nv_bfloat16*)dx_bf16, ws);
  FDX_LAUNCH_CHECK();
  uvit_head_norm_finish_kernel<<<1, 2 * kC, 0, s>>>(ws, nblk, dgamma, dbeta);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_im2col3x3_c6(const void* src0, int src0_is_f32, const void* src1, int src1_is_f32, int N, int H, int W,
                     void* col_bf16, void* stream) {
  FDX_REQUIRE(src0 && src1 && col_bf16, "im2col3x3_c6: null pointer");
  FDX_REQUIRE(N > 0 && H > 0 && W > 0, "im2col3x3_c6: bad sizes N=%d H=%d W=%d", N, H, W);
  FDX_REQUIRE(aligned16(col_bf16), "im2col3x3_c6: col must be 16-byte aligned");
  const int grid = stream_grid((long long)N * H * W, 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (src0_is_f32)
    im2col_c6_launch<true>(src0, src1, src1_is_f32, N, H, W, col_bf16, grid, s);
  else
    im2col_c6_launch<false>(src0, src1, src1_is_f32, N, H, W, col_bf16, grid, s);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
