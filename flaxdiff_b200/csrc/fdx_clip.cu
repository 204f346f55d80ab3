// fdx_clip.cu -- the pieces of the CLIP text tower (FlaxCLIPTextModel, flaxdiff/inputs/encoders.py) that are not
// GEMMs or attention: token + position embedding, LayerNorm forward, and the MLP's bias + activation.  All three
// are HBM-bound streaming kernels with 16-byte vectors; the tower's GEMMs run on fdx_gemm and its attention on
// fdx_attention_fwd_masked.
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

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void load8f(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// out[b][t][:] = bf16(tok[ids[b][t]] + pos[t]); an id outside [0, vocab) gives a NaN row (jnp.take's fill mode)
__global__ void token_embed_kernel(const int32_t* __restrict__ ids, long long rows, int T,
                                   const float* __restrict__ tok, int vocab, const float* __restrict__ pos, int D,
                                   __nv_bfloat16* __restrict__ out) {
  const int v = D / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    const int t = (int)(r % T);
    const int id = ids[r];
    float o[8];
    if (id >= 0 && id < vocab) {
      float a[8], b[8];
      load8f(tok + (long long)id * D + c, a);
      load8f(pos + (long long)t * D + c, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = a[j] + b[j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = __int_as_float(0x7fc00000);
    }
    store8(out + r * D + c, o);
  }
}

// nn.LayerNorm over the last axis, one warp per row: the row stays in registers between the mean pass and the
// centred variance pass
constexpr int kLnV = 5;   // up to 5 x 32 x 8 = 1280 channels

__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    float f[kLnV][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < kLnV; ++v) {
      if (v * 32 + lane < nv) {
        load8(x + r * C + (v * 32 + lane) * 8, f[v]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[v][j];
      }
    }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < kLnV; ++v) {
      if (v * 32 + lane < nv) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          f[v][j] -= mean;
          q = fmaf(f[v][j], f[v][j], q);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
    for (int v = 0; v < kLnV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float g[8], b[8], o[8];
        load8f(gamma + c, g);
        load8f(beta + c, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(f[v][j] * rstd, g[j], b[j]);
        store8(y + r * C + c, o);
      }
    }
  }
}

// y = act(x + bias): quick_gelu(z) = z sigmoid(1.702 z) (the openai CLIP towers), gelu(z) = z Phi(z) exactly
// (erf form, OpenCLIP configs).  x == y is allowed.
template <int ACT>
__global__ void bias_act_kernel(const __nv_bfloat16* x, long long rows, int C, const float* __restrict__ bias,
                                __nv_bfloat16* y) {
  const int v = C / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    float f[8], b[8];
    load8(x + r * C + c, f);
    if (bias) {
      load8f(bias + c, b);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = f[j] + b[j];
      if (ACT == FDX_ACT_QUICK_GELU)
        f[j] = z / (1.f + expf(-1.702f * z));
      else
        f[j] = 0.5f * z * (1.f + erff(z * 0.70710678118654752f));
    }
    store8(y + r * C + c, f);
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int fdx_token_embed(const int32_t* ids, int B, int T, const float* tok, int vocab, const float* pos, int D,
                    void* out_bf16, void* stream) {
  FDX_REQUIRE(ids && tok && pos && out_bf16, "token_embed: null pointer");
  FDX_REQUIRE(B > 0 && T > 0 && vocab > 0 && D > 0 && D % 8 == 0, "token_embed: bad sizes (D=%d must be a multiple of 8)",
              D);
  FDX_REQUIRE(aligned16(tok) && aligned16(pos) && aligned16(out_bf16), "token_embed: tables and output must be "
              "16-byte aligned");
  const long long rows = (long long)B * T;
  token_embed_kernel<<<stream_grid(rows * (D / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      ids, rows, T, tok, vocab, pos, D, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_layernorm_fwd(const void* x_bf16, long long rows, int C, const float* gamma, const float* beta, float eps,
                      void* y_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && y_bf16 && gamma && beta, "layernorm_fwd: null pointer");
  FDX_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && C <= 32 * 8 * kLnV,
              "layernorm_fwd: C=%d must be a multiple of 8, <= %d", C, 32 * 8 * kLnV);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_bf16) && aligned16(gamma) && aligned16(beta),
              "layernorm_fwd: tensors must be 16-byte aligned");
  long long grid = (rows + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  layernorm_fwd_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x_bf16, rows, C, gamma,
                                                                    beta, eps, (__nv_bfloat16*)y_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_bias_act(const void* x_bf16, long long rows, int C, const float* bias, int act, void* y_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && y_bf16, "bias_act: null pointer");
  FDX_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, "bias_act: C=%d must be a multiple of 8", C);
  FDX_REQUIRE(act == FDX_ACT_QUICK_GELU || act == FDX_ACT_GELU, "bias_act: unknown activation %d", act);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_bf16) && (!bias || aligned16(bias)),
              "bias_act: tensors must be 16-byte aligned");
  const int grid = stream_grid(rows * (C / 8), 256);
  if (act == FDX_ACT_QUICK_GELU)
    bias_act_kernel<FDX_ACT_QUICK_GELU><<<grid, 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_bf16, rows, C, bias, (__nv_bfloat16*)y_bf16);
  else
    bias_act_kernel<FDX_ACT_GELU><<<grid, 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_bf16, rows, C, bias, (__nv_bfloat16*)y_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
