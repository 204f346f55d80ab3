// fdx_geglu.cu -- FlaxGEGLU of the full transformer block (flaxdiff/models/attention.py:179-205):
//   u = proj(x) = [hidden_linear | hidden_gelu]  (2 * inner columns) ;  g = hidden_linear * gelu(hidden_gelu)
// with jax.nn.gelu's default tanh approximation, and its backward.  HBM-bound streaming kernels, 16-byte
// vectors: forward reads 4 B and writes 2 B per output element, backward reads 6 B and writes 4 B.
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

// gelu_tanh(x) = 0.5 x (1 + tanh(c (x + 0.044715 x^3))),  c = sqrt(2/pi)
__device__ __forceinline__ float gelu_tanh_f(float x, float* dgelu) {
  const float c = 0.7978845608028654f, a = 0.044715f;
  const float inner = c * (x + a * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(inner));
  if (dgelu) *dgelu = 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * c * (1.f + 3.f * a * x * x);
  return 0.5f * x * (1.f + t);
}

__global__ void geglu_fwd_kernel(const __nv_bfloat16* __restrict__ u, long long rows, int inner,
                                 __nv_bfloat16* __restrict__ g) {
  const int v = inner / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    const uint4 ul = *reinterpret_cast<const uint4*>(u + r * 2 * inner + c);
    const uint4 ug = *reinterpret_cast<const uint4*>(u + r * 2 * inner + inner + c);
    const uint32_t wl[4] = {ul.x, ul.y, ul.z, ul.w}, wg[4] = {ug.x, ug.y, ug.z, ug.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16x2(wl[j]), b = unpack_bf16x2(wg[j]);
      o[j] = pack_bf16x2(a.x * gelu_tanh_f(b.x, nullptr), a.y * gelu_tanh_f(b.y, nullptr));
    }
    *reinterpret_cast<uint4*>(g + r * inner + c) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ u, const __nv_bfloat16* __restrict__ dg,
                                 long long rows, int inner, __nv_bfloat16* __restrict__ du) {
  const int v = inner / 8;
  const long long total = rows * v;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / v;
    const int c = (int)(i % v) * 8;
    const uint4 ul = *reinterpret_cast<const uint4*>(u + r * 2 * inner + c);
    const uint4 ug = *reinterpret_cast<const uint4*>(u + r * 2 * inner + inner + c);
    const uint4 dd = *reinterpret_cast<const uint4*>(dg + r * inner + c);
    const uint32_t wl[4] = {ul.x, ul.y, ul.z, ul.w}, wg[4] = {ug.x, ug.y, ug.z, ug.w},
                   wd[4] = {dd.x, dd.y, dd.z, dd.w};
    uint32_t ol[4], og[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = unpack_bf16x2(wl[j]), b = unpack_bf16x2(wg[j]), d = unpack_bf16x2(wd[j]);
      float d0, d1;
      const float g0 = gelu_tanh_f(b.x, &d0), g1 = gelu_tanh_f(b.y, &d1);
      ol[j] = pack_bf16x2(d.x * g0, d.y * g1);                 // d hidden_linear
      og[j] = pack_bf16x2(d.x * a.x * d0, d.y * a.y * d1);     // d hidden_gelu
    }
    *reinterpret_cast<uint4*>(du + r * 2 * inner + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    *reinterpret_cast<uint4*>(du + r * 2 * inner + inner + c) = make_uint4(og[0], og[1], og[2], og[3]);
  }
}

}  // namespace

extern "C" {

int fdx_geglu_fwd(const void* u_bf16, long long rows, int inner, void* g_bf16, void* stream) {
  FDX_REQUIRE(u_bf16 && g_bf16 && rows > 0 && inner > 0 && inner % 8 == 0, "geglu_fwd: bad arguments");
  geglu_fwd_kernel<<<stream_grid(rows * (inner / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)u_bf16, rows, inner, (__nv_bfloat16*)g_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_geglu_bwd(const void* u_bf16, const void* dg_bf16, long long rows, int inner, void* du_bf16,
                  void* stream) {
  FDX_REQUIRE(u_bf16 && dg_bf16 && du_bf16 && rows > 0 && inner > 0 && inner % 8 == 0, "geglu_bwd: bad arguments");
  geglu_bwd_kernel<<<stream_grid(rows * (inner / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)u_bf16, (const __nv_bfloat16*)dg_bf16, rows, inner, (__nv_bfloat16*)du_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
