// fdx_clip.cu -- the pieces of the CLIP towers that are not GEMMs or attention.  Text tower (FlaxCLIPTextModel,
// flaxdiff/inputs/encoders.py): token + position embedding, LayerNorm forward, and the MLP's bias + activation, all
// HBM-bound streaming kernels with 16-byte vectors.  CLIP metrics (flaxdiff/metrics/images.py:32-112): the image
// preprocessing (quantise, PIL bicubic resize, crop, normalise, patchify), the vision embedding + pre-LayerNorm, the
// pooled row of either tower and the cosine.  The towers' GEMMs run on fdx_gemm and their attention on
// fdx_attention_fwd (vision) / fdx_attention_fwd_masked (text).
#include "fdx_common.cuh"
#include "../../include/fdx.h"
#include <limits.h>
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

// Normalise the row a warp holds in f (lane owns the 8-channel vectors v * 32 + lane < C / 8, in channel order) and
// store it as bf16: the sum in the order the vectors were loaded, then the centred squares, f32 throughout.
__device__ __forceinline__ void layernorm_row_store(float (&f)[kLnV][8], int C, int lane, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float eps,
                                                    __nv_bfloat16* __restrict__ y) {
  const int nv = C >> 3;
  float s = 0.f;
#pragma unroll
  for (int v = 0; v < kLnV; ++v) {
    if (v * 32 + lane < nv) {
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
      store8(y + c, o);
    }
  }
}

__global__ void __launch_bounds__(256)
layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long rows, int C, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int nv = C >> 3;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    float f[kLnV][8];
#pragma unroll
    for (int v = 0; v < kLnV; ++v)
      if (v * 32 + lane < nv) load8(x + r * C + (v * 32 + lane) * 8, f[v]);
    layernorm_row_store(f, C, lane, gamma, beta, eps, y + r * C);
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

// ---- CLIP image metrics (flaxdiff/metrics/images.py:32-112) ----------------------------------------------------

// ((g + 1) / 2) * 255 as f32 (each operation rounded on its own), truncated to uint8; clamped to [0, 255], NaN -> 0
__device__ __forceinline__ int quantise_u8(float g) {
  const float t = __fmul_rn(__fmul_rn(__fadd_rn(g, 1.f), 0.5f), 255.f);
  return t > 0.f ? (t < 255.f ? (int)t : 255) : 0;
}

// PIL's clip8: the 22-fraction-bit accumulator shifted down and clamped to uint8
__device__ __forceinline__ int clip8(int acc) { return min(max(acc >> 22, 0), 255); }

// The crop window of PIL's two-pass 8-bit bicubic resize, one output element per (patch row, column) and 8 columns per
// thread.  tab = [crop][2 + ksy] rows then [crop][2 + ksx] columns: first source index, tap count, int32 taps.  A pass
// PIL skips has the identity table (one tap of 1 << 22), which reproduces its input exactly.
__global__ void __launch_bounds__(256)
clip_image_prep_kernel(const float* __restrict__ x, int B, int H, int W, const int32_t* __restrict__ tab, int ksy,
                       int ksx, const float* __restrict__ lut, int crop, int p, int ld,
                       __nv_bfloat16* __restrict__ patches, uint8_t* __restrict__ u8) {
  const int G = crop / p, pp = p * p, K = 3 * pp, nvec = ld / 8;
  const int32_t* tabx = tab + (long long)crop * (2 + ksy);
  const long long total = (long long)B * G * G * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / nvec;
    const int c0 = (int)(i % nvec) * 8;
    const int b = (int)(row / (G * G)), g = (int)(row % (G * G)), gy = g / G, gx = g % G;
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int col = c0 + e;
      if (col >= K) {
        o[e] = 0.f;
        continue;
      }
      const int c = col / pp, ky = (col % pp) / p, kx = col % p;
      const int Y = gy * p + ky, X = gx * p + kx;
      const int32_t* ty = tab + (long long)Y * (2 + ksy);
      const int32_t* tx = tabx + (long long)X * (2 + ksx);
      const int y0 = ty[0], ny = ty[1], x0 = tx[0], nx = tx[1];
      int acc = 1 << 21;
      for (int j = 0; j < ny; ++j) {
        const float* src = x + (((long long)b * H + y0 + j) * W + x0) * 3 + c;
        int h = 1 << 21;
        for (int t = 0; t < nx; ++t) h += quantise_u8(src[3 * t]) * tx[2 + t];
        acc += clip8(h) * ty[2 + j];
      }
      const int v = clip8(acc);
      o[e] = lut[c * 256 + v];
      if (u8) u8[(((long long)b * crop + Y) * crop + X) * 3 + c] = (uint8_t)v;
    }
    store8(patches + row * ld + c0, o);
  }
}

// h[b][t] = LN(t == 0 ? cls : patch[b][t - 1]) + pos[t]) in f32, rounded to bf16 once; one warp per token
__global__ void __launch_bounds__(256)
clip_vision_embed_kernel(const float* __restrict__ patch, int B, int G2, int D, const float* __restrict__ cls,
                         const float* __restrict__ pos, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int nv = D >> 3, T = G2 + 1;
  const long long rows = (long long)B * T;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long nw = (long long)gridDim.x * 8;
  for (long long r = wid; r < rows; r += nw) {
    const int t = (int)(r % T);
    const float* src = t == 0 ? cls : patch + ((r / T) * G2 + t - 1) * D;
    float f[kLnV][8];
#pragma unroll
    for (int v = 0; v < kLnV; ++v) {
      if (v * 32 + lane < nv) {
        const int c = (v * 32 + lane) * 8;
        float a[8];
        load8f(src + c, f[v]);
        load8f(pos + (long long)t * D + c, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[v][j] += a[j];
      }
    }
    layernorm_row_store(f, D, lane, gamma, beta, eps, y + r * D);
  }
}

// out[b] = [LN](x[b][row_b]); row_b = 0, or the first position of the largest id of sequence b.  One warp per sequence.
__global__ void __launch_bounds__(256)
clip_pool_kernel(const __nv_bfloat16* __restrict__ x, int B, int T, int D, const int32_t* __restrict__ ids,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                 __nv_bfloat16* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int nv = D >> 3;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  int best = 0;
  if (ids) {
    int bv = INT_MIN;
    best = T;
    for (int t = lane; t < T; t += 32) {
      const int v = ids[(long long)b * T + t];
      if (v > bv) { bv = v; best = t; }             // t ascends: the first position of the lane's maximum
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int ov = __shfl_xor_sync(0xffffffffu, bv, o), ot = __shfl_xor_sync(0xffffffffu, best, o);
      if (ov > bv || (ov == bv && ot < best)) { bv = ov; best = ot; }
    }
  }
  const __nv_bfloat16* src = x + ((long long)b * T + best) * D;
  if (!gamma) {
    for (int c = lane * 8; c < D; c += 256)
      *reinterpret_cast<uint4*>(out + (long long)b * D + c) = *reinterpret_cast<const uint4*>(src + c);
    return;
  }
  float f[kLnV][8];
#pragma unroll
  for (int v = 0; v < kLnV; ++v)
    if (v * 32 + lane < nv) load8(src + (v * 32 + lane) * 8, f[v]);
  layernorm_row_store(f, D, lane, gamma, beta, eps, out + (long long)b * D);
}

// cos[b] = <a / (|a| + 1e-6), t / (|t| + 1e-6)>, f32; one block, one warp per sample, then the two means over the
// batch in a fixed order: out2 = {mean(1 - cos), mean(100 max(cos, 0))}
constexpr int kSimThreads = 1024;

__global__ void __launch_bounds__(kSimThreads)
clip_similarity_kernel(const float* __restrict__ img, const float* __restrict__ txt, int B, int P,
                       float* __restrict__ cos, float* __restrict__ out2) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = warp; b < B; b += kSimThreads / 32) {
    const float* a = img + (long long)b * P;
    const float* t = txt + (long long)b * P;
    float dot = 0.f, aa = 0.f, tt = 0.f;
    for (int c = lane; c < P; c += 32) {
      const float u = a[c], v = t[c];
      dot = fmaf(u, v, dot);
      aa = fmaf(u, u, aa);
      tt = fmaf(v, v, tt);
    }
    dot = warp_sum(dot);
    aa = warp_sum(aa);
    tt = warp_sum(tt);
    if (lane == 0) cos[b] = dot / (sqrtf(aa) + 1e-6f) / (sqrtf(tt) + 1e-6f);
  }
  __syncthreads();
  if (warp == 0) {
    float s = 0.f, sc = 0.f;
    for (int b = lane; b < B; b += 32) {
      const float c = cos[b];
      s += 1.f - c;
      sc += 100.f * fmaxf(c, 0.f);
    }
    s = warp_sum(s);
    sc = warp_sum(sc);
    if (lane == 0) {
      out2[0] = s / (float)B;
      out2[1] = sc / (float)B;
    }
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// the tanh-gelu of the DiT's MLP lives with its backward in fdx_dit.cu
int fdx_dit_bias_gelu_tanh(const void* x_bf16, long long rows, int C, const float* bias, void* y_bf16, void* stream);

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
  FDX_REQUIRE(act == FDX_ACT_QUICK_GELU || act == FDX_ACT_GELU || act == FDX_ACT_GELU_TANH,
              "bias_act: unknown activation %d", act);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(y_bf16) && (!bias || aligned16(bias)),
              "bias_act: tensors must be 16-byte aligned");
  if (act == FDX_ACT_GELU_TANH) return fdx_dit_bias_gelu_tanh(x_bf16, rows, C, bias, y_bf16, stream);
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

int fdx_clip_image_prep(const float* x, int B, int H, int W, const int32_t* tables, int ksize_y, int ksize_x,
                        const float* lut, int crop, int patch, int ld, void* patches_bf16, uint8_t* u8_out,
                        void* stream) {
  FDX_REQUIRE(x && tables && lut && patches_bf16, "clip_image_prep: null pointer");
  FDX_REQUIRE(B > 0 && H > 0 && W > 0 && ksize_y > 0 && ksize_x > 0, "clip_image_prep: bad sizes");
  FDX_REQUIRE(patch > 0 && crop > 0 && crop % patch == 0, "clip_image_prep: crop %d is not a multiple of the patch %d",
              crop, patch);
  FDX_REQUIRE(ld % 8 == 0 && ld >= 3 * patch * patch, "clip_image_prep: ld=%d must be a multiple of 8, >= %d", ld,
              3 * patch * patch);
  FDX_REQUIRE(aligned16(patches_bf16), "clip_image_prep: patches must be 16-byte aligned");
  const int G = crop / patch;
  clip_image_prep_kernel<<<stream_grid((long long)B * G * G * (ld / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      x, B, H, W, tables, ksize_y, ksize_x, lut, crop, patch, ld, (__nv_bfloat16*)patches_bf16, u8_out);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_clip_vision_embed(const float* patch_f32, int B, int G2, int D, const float* cls, const float* pos,
                          const float* gamma, const float* beta, float eps, void* out_bf16, void* stream) {
  FDX_REQUIRE(patch_f32 && cls && pos && gamma && beta && out_bf16, "clip_vision_embed: null pointer");
  FDX_REQUIRE(B > 0 && G2 > 0 && D > 0 && D % 8 == 0 && D <= 32 * 8 * kLnV,
              "clip_vision_embed: D=%d must be a multiple of 8, <= %d", D, 32 * 8 * kLnV);
  FDX_REQUIRE(aligned16(patch_f32) && aligned16(cls) && aligned16(pos) && aligned16(gamma) && aligned16(beta) &&
              aligned16(out_bf16), "clip_vision_embed: tensors must be 16-byte aligned");
  long long grid = ((long long)B * (G2 + 1) + 7) / 8;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  clip_vision_embed_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(patch_f32, B, G2, D, cls, pos, gamma, beta,
                                                                        eps, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_clip_pool(const void* x_bf16, int B, int T, int D, const int32_t* ids, const float* gamma, const float* beta,
                  float eps, void* out_bf16, void* stream) {
  FDX_REQUIRE(x_bf16 && out_bf16, "clip_pool: null pointer");
  FDX_REQUIRE(!gamma == !beta, "clip_pool: gamma and beta are given together or not at all");
  FDX_REQUIRE(B > 0 && T > 0 && D > 0 && D % 8 == 0 && D <= 32 * 8 * kLnV,
              "clip_pool: D=%d must be a multiple of 8, <= %d", D, 32 * 8 * kLnV);
  FDX_REQUIRE(aligned16(x_bf16) && aligned16(out_bf16) && (!gamma || (aligned16(gamma) && aligned16(beta))),
              "clip_pool: tensors must be 16-byte aligned");
  clip_pool_kernel<<<(B + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x_bf16, B, T, D, ids, gamma,
                                                                  beta, eps, (__nv_bfloat16*)out_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_clip_similarity(const float* img, const float* txt, int B, int P, float* cos, float* out2, void* stream) {
  FDX_REQUIRE(img && txt && cos && out2, "clip_similarity: null pointer");
  FDX_REQUIRE(B > 0 && P > 0, "clip_similarity: bad sizes");
  clip_similarity_kernel<<<1, kSimThreads, 0, (cudaStream_t)stream>>>(img, txt, B, P, cos, out2);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
