// fdx_misc.cu -- timestep embedding MLP and attention softmax.
//
//   FourierEmbedding + TimeProjection      flaxdiff/models/common.py:97-124
//       emb = [sin, cos](t * (2*pi*freqs));  Dense(256) -> gelu(tanh) -> Dense(256) -> gelu
//       (TimeProjection passes no dtype => f32 arithmetic in the reference; f32 here too)
//   softmax of nn.dot_product_attention     flaxdiff/models/attention.py:170-174
// The MLP is ~0.26 MFLOP per sample: one CTA per sample, f32 on CUDA cores.
#include "fdx_common.cuh"
#include "../../include/fdx.h"

namespace {

__device__ __forceinline__ float gelu_tanh(float x) {
  const float k = 0.7978845608028654f;   // sqrt(2/pi)
  return 0.5f * x * (1.f + tanhf(k * (x + 0.044715f * x * x * x)));
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k = 0.7978845608028654f;
  const float u = k * (x + 0.044715f * x * x * x);
  const float th = tanhf(u);
  return 0.5f * (1.f + th) + 0.5f * x * (1.f - th * th) * k * (1.f + 3.f * 0.044715f * x * x);
}

// one block of D threads per sample; D = emb features (256)
__global__ void time_embed_fwd_kernel(const float* __restrict__ t, const float* __restrict__ freqs,
                                      const float* __restrict__ W1, const float* __restrict__ b1,
                                      const float* __restrict__ W2, const float* __restrict__ b2,
                                      int D, float* __restrict__ four, float* __restrict__ h1,
                                      float* __restrict__ h2, float* __restrict__ emb,
                                      __nv_bfloat16* __restrict__ emb_bf16) {
  extern __shared__ float sh[];   // [D]
  const int b = blockIdx.x, j = threadIdx.x, half = D / 2;
  const float tv = t[b];
  {
    const float f = freqs[j < half ? j : j - half];
    const float w = 6.283185307179586f * f;   // (2*pi*freqs) rounded to f32 first, as jnp does
    const float ph = tv * w;
    const float v = j < half ? sinf(ph) : cosf(ph);
    sh[j] = v;
    four[(long long)b * D + j] = v;
  }
  __syncthreads();
  float a = b1[j];
  for (int k = 0; k < D; ++k) a += sh[k] * W1[(long long)k * D + j];
  h1[(long long)b * D + j] = a;
  const float g1 = gelu_tanh(a);
  __syncthreads();
  sh[j] = g1;
  __syncthreads();
  float c = b2[j];
  for (int k = 0; k < D; ++k) c += sh[k] * W2[(long long)k * D + j];
  h2[(long long)b * D + j] = c;
  const float g2 = gelu_tanh(c);
  emb[(long long)b * D + j] = g2;
  if (emb_bf16) emb_bf16[(long long)b * D + j] = __float2bfloat16(g2);
}

// per-sample backward: dh2 = demb * gelu'(h2); da1 = dh2 W2^T; dh1 = da1 * gelu'(h1)
__global__ void time_embed_bwd_kernel(const float* __restrict__ demb, const float* __restrict__ h1,
                                      const float* __restrict__ h2, const float* __restrict__ W2,
                                      int D, float* __restrict__ dh1, float* __restrict__ dh2) {
  extern __shared__ float sh[];
  const int b = blockIdx.x, j = threadIdx.x;
  const float d2 = demb[(long long)b * D + j] * gelu_tanh_grad(h2[(long long)b * D + j]);
  dh2[(long long)b * D + j] = d2;
  sh[j] = d2;
  __syncthreads();
  float a = 0.f;
  const float* wrow = W2 + (long long)j * D;   // da1[j] = sum_n dh2[n] * W2[j][n]
  for (int n = 0; n < D; ++n) a += sh[n] * wrow[n];
  dh1[(long long)b * D + j] = a * gelu_tanh_grad(h1[(long long)b * D + j]);
}

// dW[k][j] += sum_b in[b][k] * dout[b][j] ; db[j] += sum_b dout[b][j]
// grid = (D/16 row blocks, batch slices); partial sums are combined with f32 atomics
__global__ void dense_wgrad_small_kernel(const float* __restrict__ in, int apply_gelu,
                                         const float* __restrict__ dout, int B, int D,
                                         float* __restrict__ dW, float* __restrict__ db) {
  const int j = threadIdx.x, k0 = blockIdx.x * 16;
  const int per = (B + gridDim.y - 1) / gridDim.y;
  const int b0 = blockIdx.y * per, b1 = min(B, b0 + per);
  float acc[16];
#pragma unroll
  for (int r = 0; r < 16; ++r) acc[r] = 0.f;
  float accb = 0.f;
  for (int b = b0; b < b1; ++b) {
    const float d = dout[(long long)b * D + j];
    accb += d;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float v = in[(long long)b * D + k0 + r];
      if (apply_gelu) v = gelu_tanh(v);
      acc[r] += v * d;
    }
  }
#pragma unroll
  for (int r = 0; r < 16; ++r) atomicAdd(&dW[(long long)(k0 + r) * D + j], acc[r]);
  if (blockIdx.x == 0) atomicAdd(&db[j], accb);
}

// ---- softmax over the last dim; one warp per row; S f32 -> P bf16.  Rows have Lp (padded) columns of
//      which the first L are real: padded logits are ignored and padded probabilities written as 0.
__global__ void __launch_bounds__(256)
softmax_fwd_kernel(const float* __restrict__ S, long long rows, int L, int Lp, __nv_bfloat16* __restrict__ P) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    const float* s = S + r * Lp;
    float mx = -INFINITY;
    for (int i = lane; i < L; i += 32) mx = fmaxf(mx, s[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int i = lane; i < L; i += 32) sum += __expf(s[i] - mx);
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    __nv_bfloat16* p = P + r * Lp;
    for (int i = lane; i < Lp; i += 32) p[i] = __float2bfloat16(i < L ? __expf(s[i] - mx) * inv : 0.f);
  }
}

// dS = P * (dP - sum_k dP*P) * scale ; dP f32 -> dS bf16 (padded columns -> 0)
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const __nv_bfloat16* __restrict__ P, const float* __restrict__ dP,
                   long long rows, int L, int Lp, float scale, __nv_bfloat16* __restrict__ dS) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    const __nv_bfloat16* p = P + r * Lp;
    const float* d = dP + r * Lp;
    float dot = 0.f;
    for (int i = lane; i < L; i += 32) dot += __bfloat162float(p[i]) * d[i];
    dot = warp_sum(dot);
    __nv_bfloat16* o = dS + r * Lp;
    for (int i = lane; i < Lp; i += 32)
      o[i] = __float2bfloat16(i < L ? __bfloat162float(p[i]) * (d[i] - dot) * scale : 0.f);
  }
}

}  // namespace

extern "C" {

int fdx_time_embed_fwd(const float* t, const float* freqs, const float* W1, const float* b1,
                       const float* W2, const float* b2, int B, int D, float* four, float* h1,
                       float* h2, float* emb, void* emb_bf16, void* stream) {
  FDX_REQUIRE(t && freqs && W1 && b1 && W2 && b2 && four && h1 && h2 && emb,
              "time_embed_fwd: null pointer");
  FDX_REQUIRE(B > 0 && D >= 32 && D <= 1024 && D % 32 == 0, "time_embed_fwd: bad D=%d", D);
  time_embed_fwd_kernel<<<B, D, sizeof(float) * D, (cudaStream_t)stream>>>(
      t, freqs, W1, b1, W2, b2, D, four, h1, h2, emb, (__nv_bfloat16*)emb_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_time_embed_bwd(const float* demb, const float* four, const float* h1, const float* h2,
                       const float* W2, int B, int D, float* dh1_ws, float* dh2_ws, float* dW1,
                       float* db1, float* dW2, float* db2, void* stream) {
  FDX_REQUIRE(demb && four && h1 && h2 && W2 && dh1_ws && dh2_ws && dW1 && db1 && dW2 && db2,
              "time_embed_bwd: null pointer");
  FDX_REQUIRE(B > 0 && D >= 32 && D <= 1024 && D % 32 == 0, "time_embed_bwd: bad D=%d", D);
  cudaStream_t st = (cudaStream_t)stream;
  time_embed_bwd_kernel<<<B, D, sizeof(float) * D, st>>>(demb, h1, h2, W2, D, dh1_ws, dh2_ws);
  FDX_LAUNCH_CHECK();
  const int bs = B >= 64 ? 16 : (B >= 8 ? 4 : 1);
  dense_wgrad_small_kernel<<<dim3(D / 16, bs), D, 0, st>>>(h1, 1, dh2_ws, B, D, dW2, db2);
  FDX_LAUNCH_CHECK();
  dense_wgrad_small_kernel<<<dim3(D / 16, bs), D, 0, st>>>(four, 0, dh1_ws, B, D, dW1, db1);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_softmax_fwd(const float* S, long long rows, int L, int Lp, void* P_bf16, void* stream) {
  FDX_REQUIRE(S && P_bf16 && rows > 0 && L > 0 && Lp >= L, "softmax_fwd: bad arguments");
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 16) grid = fdx_num_sms() * 16;
  softmax_fwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(S, rows, L, Lp,
                                                                 (__nv_bfloat16*)P_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_softmax_bwd(const void* P_bf16, const float* dP, long long rows, int L, int Lp, float scale,
                    void* dS_bf16, void* stream) {
  FDX_REQUIRE(P_bf16 && dP && dS_bf16 && rows > 0 && L > 0 && Lp >= L, "softmax_bwd: bad arguments");
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 16) grid = fdx_num_sms() * 16;
  softmax_bwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)P_bf16, dP, rows, L, Lp, scale, (__nv_bfloat16*)dS_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
