// fdx_stream.cu -- HBM-bound streaming kernels of the diffusion step.
//
// Reference call sites replaced (XLA fusions, or un-jitted jnp op chains in the samplers):
//   image normalise + forward_diffusion + c_in      trainer/general_diffusion_trainer.py:258,285-291
//                                                   predictors/__init__.py:19-24,43-44,67-71,93-96
//   pred_transform + l2_loss + weights + mean        general_diffusion_trainer.py:295-302,
//                                                   predictors/__init__.py:84-91
//   sampler update rules / CFG combine / x0,eps      samplers/{euler,ddim,ddpm,heun_sampler}.py,
//                                                   samplers/common.py:93-96
//   optax adam/adamw + apply_ema                     trainer/diffusion_trainer.py:31-37, training.py:594-608
//   jax.image.resize(nearest) x2                     models/common.py:214-215
// All are one pass over their operands: 128-bit vector accesses, grid-stride loops sized
// to a multiple of the SM count.
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

// ---------------------------------------------------------------------------
// noise-add / precondition
// ---------------------------------------------------------------------------
template <bool U8>
__global__ void diffuse_forward_kernel(const void* __restrict__ x0_, const float* __restrict__ eps,
                                       const float* __restrict__ alpha,
                                       const float* __restrict__ sigma,
                                       const float* __restrict__ c_in, int B, long long E,
                                       int normalize, int target_kind, float* __restrict__ x_t,
                                       float* __restrict__ target,
                                       __nv_bfloat16* __restrict__ model_in) {
  // E (elements per sample) is a multiple of 4; one thread handles 4 elements.
  const long long total4 = (long long)B * E / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    const int b = (int)(e / E);
    const float a = alpha[b], s = sigma[b], ci = c_in[b];
    float x[4];
    if (U8) {
      const uchar4 u = reinterpret_cast<const uchar4*>(x0_)[i];
      x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w;
    } else {
      const float4 u = reinterpret_cast<const float4*>(x0_)[i];
      x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w;
    }
    const float4 n4 = reinterpret_cast<const float4*>(eps)[i];
    const float n[4] = {n4.x, n4.y, n4.z, n4.w};
    float xt[4], tg[4];
    const float inv_sd = rsqrtf(a * a + s * s);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (normalize) x[j] = (x[j] - 127.5f) / 127.5f;
      xt[j] = a * x[j] + s * n[j];
      tg[j] = target_kind == 0 ? x[j] : target_kind == 1 ? n[j] : (a * n[j] - s * x[j]) * inv_sd;
    }
    reinterpret_cast<float4*>(x_t)[i] = make_float4(xt[0], xt[1], xt[2], xt[3]);
    reinterpret_cast<float4*>(target)[i] = make_float4(tg[0], tg[1], tg[2], tg[3]);
    uint2 o;
    o.x = pack_bf16x2(xt[0] * ci, xt[1] * ci);
    o.y = pack_bf16x2(xt[2] * ci, xt[3] * ci);
    reinterpret_cast<uint2*>(model_in)[i] = o;
  }
}

// ---------------------------------------------------------------------------
// loss forward + seed of the backward pass
// ---------------------------------------------------------------------------
__global__ void loss_kernel(const float* __restrict__ F, const float* __restrict__ x_t,
                            const float* __restrict__ target, const float* __restrict__ c_out,
                            const float* __restrict__ c_skip, const float* __restrict__ weight,
                            int B, long long E, float inv_count, float* __restrict__ loss_sum,
                            float* __restrict__ dF) {
  const long long total4 = (long long)B * E / 4;
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)((i * 4) / E);
    const float co = c_out[b], cs = c_skip[b], w = weight[b];
    const float4 f = reinterpret_cast<const float4*>(F)[i];
    const float4 x = reinterpret_cast<const float4*>(x_t)[i];
    const float4 t = reinterpret_cast<const float4*>(target)[i];
    const float d0 = co * f.x + cs * x.x - t.x, d1 = co * f.y + cs * x.y - t.y;
    const float d2 = co * f.z + cs * x.z - t.z, d3 = co * f.w + cs * x.w - t.w;
    acc += 0.5f * w * (d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3);
    if (dF) {
      const float g = w * co * inv_count;
      reinterpret_cast<float4*>(dF)[i] = make_float4(g * d0, g * d1, g * d2, g * d3);
    }
  }
  acc = warp_sum(acc);
  __shared__ float sh[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) sh[wid] = acc;
  __syncthreads();
  if (wid == 0) {
    float v = lane < (blockDim.x >> 5) ? sh[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) atomicAdd(loss_sum, v * inv_count);
  }
}

// ---------------------------------------------------------------------------
// affine combination of up to 6 f32 tensors with per-sample coefficients:
//   out1 = sum_i a[i][b] * in_i ; out2 = sum_i c[i][b] * in_i ; out_bf16 = bf16(out1 * s[b])
// Covers x0/eps recovery, CFG mixing and every sampler update rule in one pass.
// ---------------------------------------------------------------------------
struct AffineArgs {
  const float* in[6];
  int n_in;
  const float* a;   // [n_in][B]
  const float* c;   // [n_in][B] or null
  const float* s;   // [B] or null
  float* out1;
  float* out2;
  __nv_bfloat16* out_bf16;
  float clip_lo, clip_hi;
  int clip;
};

__global__ void affine_kernel(const AffineArgs p, int B, long long E) {
  const long long total4 = (long long)B * E / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)((i * 4) / E);
    float o1[4] = {0.f, 0.f, 0.f, 0.f}, o2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      if (k < p.n_in) {
        const float4 v = reinterpret_cast<const float4*>(p.in[k])[i];
        const float a = p.a[(long long)k * B + b];
        o1[0] += a * v.x; o1[1] += a * v.y; o1[2] += a * v.z; o1[3] += a * v.w;
        if (p.c) {
          const float c = p.c[(long long)k * B + b];
          o2[0] += c * v.x; o2[1] += c * v.y; o2[2] += c * v.z; o2[3] += c * v.w;
        }
      }
    }
    if (p.clip) {
#pragma unroll
      for (int j = 0; j < 4; ++j) o1[j] = fminf(fmaxf(o1[j], p.clip_lo), p.clip_hi);
    }
    if (p.out1) reinterpret_cast<float4*>(p.out1)[i] = make_float4(o1[0], o1[1], o1[2], o1[3]);
    if (p.out2) reinterpret_cast<float4*>(p.out2)[i] = make_float4(o2[0], o2[1], o2[2], o2[3]);
    if (p.out_bf16) {
      const float s = p.s ? p.s[b] : 1.f;
      uint2 o;
      o.x = pack_bf16x2(o1[0] * s, o1[1] * s);
      o.y = pack_bf16x2(o1[2] * s, o1[3] * s);
      reinterpret_cast<uint2*>(p.out_bf16)[i] = o;
    }
  }
}

// (the optimiser kernels live in fdx_optim.cu)
__global__ void cast_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                 long long n) {
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(dst)[i] = o;
  }
}

// ---------------------------------------------------------------------------
// nearest x2 upsample (and its adjoint), NHWC bf16, 16-byte channel vectors
// ---------------------------------------------------------------------------
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, long long xps, int N, int H,
                                  int W, int C, __nv_bfloat16* __restrict__ y, long long yps) {
  const int vpp = C >> 3;
  const long long total = (long long)N * (2 * H) * (2 * W) * vpp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vpp);
    long long p = i / vpp;
    const int ox = (int)(p % (2 * W)); p /= (2 * W);
    const int oy = (int)(p % (2 * H));
    const int n = (int)(p / (2 * H));
    const long long src = ((long long)(n * H + (oy >> 1)) * W + (ox >> 1)) * xps + cv * 8;
    const long long dst = ((long long)(n * 2 * H + oy) * (2 * W) + ox) * yps + cv * 8;
    *reinterpret_cast<uint4*>(y + dst) = *reinterpret_cast<const uint4*>(x + src);
  }
}

__global__ void upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, long long dps, int N,
                                      int H, int W, int C, __nv_bfloat16* __restrict__ dx,
                                      long long xps, int accumulate) {
  const int vpp = C >> 3;
  const long long total = (long long)N * H * W * vpp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vpp);
    long long p = i / vpp;
    const int x = (int)(p % W); p /= W;
    const int y = (int)(p % H);
    const int n = (int)(p / H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dyy = 0; dyy < 2; ++dyy)
#pragma unroll
      for (int dxx = 0; dxx < 2; ++dxx) {
        const long long src =
            ((long long)(n * 2 * H + 2 * y + dyy) * (2 * W) + 2 * x + dxx) * dps + cv * 8;
        const uint4 u = *reinterpret_cast<const uint4*>(dy + src);
        float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
               d = unpack_bf16x2(u.w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      }
    const long long dst = ((long long)(n * H + y) * W + x) * xps + cv * 8;
    if (accumulate) {
      const uint4 u = *reinterpret_cast<const uint4*>(dx + dst);
      float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
             d = unpack_bf16x2(u.w);
      acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
      acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(dx + dst) = o;
  }
}

// dst (+)= src on strided NHWC bf16 views
__global__ void act_add_kernel(const __nv_bfloat16* __restrict__ a, long long aps,
                               const __nv_bfloat16* __restrict__ b, long long bps,
                               __nv_bfloat16* __restrict__ o, long long ops, long long npix, int C) {
  const int vpp = C >> 3;
  const long long total = npix * vpp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vpp);
    const long long p = i / vpp;
    const uint4 ua = *reinterpret_cast<const uint4*>(a + p * aps + cv * 8);
    const uint4 ub = *reinterpret_cast<const uint4*>(b + p * bps + cv * 8);
    uint4 r;
    float2 x, y;
#define ADD2(F) x = unpack_bf16x2(ua.F); y = unpack_bf16x2(ub.F); r.F = pack_bf16x2(x.x + y.x, x.y + y.y);
    ADD2(x) ADD2(y) ADD2(z) ADD2(w)
#undef ADD2
    *reinterpret_cast<uint4*>(o + p * ops + cv * 8) = r;
  }
}

// per-image (or whole-batch) column sums of an NHWC bf16 tensor -> f32 atomics.
// Whole-batch mode (out_img_stride == 0): gridDim.y < N and every block walks several images, so each
// output address sees at most ~300 atomics instead of one per (image, pixel block).
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, long long xps, int N, int HW, int C,
              float* __restrict__ out, long long out_img_stride) {
  const int vpp = C >> 3, rows = 256 / vpp;
  const int tid = threadIdx.x;
  extern __shared__ float sh[];   // [rows*C]
  const int cv = tid % vpp, r = tid / vpp;
  const bool live = tid < rows * vpp;
  const int stride = gridDim.x * rows;
  for (int n0 = blockIdx.y; n0 < N; n0 += gridDim.y) {
    f32x2_t acc[4] = {f2_pack(0.f, 0.f), f2_pack(0.f, 0.f), f2_pack(0.f, 0.f), f2_pack(0.f, 0.f)};
    const int n_end = out_img_stride ? n0 + 1 : N;
    const int n_step = out_img_stride ? 1 : gridDim.y;
    if (live) {
      for (int n = n0; n < n_end; n += n_step) {
        const __nv_bfloat16* base = x + (long long)n * HW * xps + cv * 8;
        for (int p0 = blockIdx.x * rows + r; p0 < HW; p0 += 4 * stride) {
          uint4 u[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int p = p0 + k * stride;
            u[k] = make_uint4(0, 0, 0, 0);
            if (p < HW) u[k] = *reinterpret_cast<const uint4*>(base + (long long)p * xps);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            acc[0] = f2_add(acc[0], f2_from_bf16x2(u[k].x));
            acc[1] = f2_add(acc[1], f2_from_bf16x2(u[k].y));
            acc[2] = f2_add(acc[2], f2_from_bf16x2(u[k].z));
            acc[3] = f2_add(acc[3], f2_from_bf16x2(u[k].w));
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float lo, hi;
        f2_unpack(acc[j], lo, hi);
        sh[r * C + cv * 8 + 2 * j] = lo;
        sh[r * C + cv * 8 + 2 * j + 1] = hi;
      }
    }
    __syncthreads();
    for (int c = tid; c < C; c += 256) {
      float v = 0.f;
      for (int rr = 0; rr < rows; ++rr) v += sh[rr * C + c];
      atomicAdd(&out[(long long)n0 * out_img_stride + c], v);
    }
    __syncthreads();
    if (!out_img_stride) break;     // whole-batch mode consumed all its images in the inner loop
  }
}

}  // namespace

extern "C" {

int fdx_diffuse_forward(const void* x0, int x0_is_u8, const float* eps, const float* alpha,
                        const float* sigma, const float* c_in, int B, long long E, int normalize,
                        int target_kind, float* x_t, float* target, void* model_in_bf16,
                        void* stream) {
  FDX_REQUIRE(x0 && eps && alpha && sigma && c_in && x_t && target && model_in_bf16,
              "diffuse_forward: null pointer");
  FDX_REQUIRE(B > 0 && E > 0 && E % 4 == 0, "diffuse_forward: E=%lld must be a multiple of 4", E);
  FDX_REQUIRE(target_kind >= 0 && target_kind <= 2, "diffuse_forward: bad target kind");
  const long long t4 = (long long)B * E / 4;
  const int grid = stream_grid(t4, 256);
  if (x0_is_u8)
    diffuse_forward_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(
        x0, eps, alpha, sigma, c_in, B, E, normalize, target_kind, x_t, target,
        (__nv_bfloat16*)model_in_bf16);
  else
    diffuse_forward_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(
        x0, eps, alpha, sigma, c_in, B, E, normalize, target_kind, x_t, target,
        (__nv_bfloat16*)model_in_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_loss_fwd_bwd(const float* F, const float* x_t, const float* target, const float* c_out,
                     const float* c_skip, const float* weight, int B, long long E,
                     float* loss_sum, float* dF, void* stream) {
  FDX_REQUIRE(F && x_t && target && c_out && c_skip && weight && loss_sum, "loss: null pointer");
  FDX_REQUIRE(B > 0 && E > 0 && E % 4 == 0, "loss: E=%lld must be a multiple of 4", E);
  cudaStream_t st = (cudaStream_t)stream;
  FDX_CUDA(cudaMemsetAsync(loss_sum, 0, sizeof(float), st));
  const long long t4 = (long long)B * E / 4;
  loss_kernel<<<stream_grid(t4, 256), 256, 0, st>>>(F, x_t, target, c_out, c_skip, weight, B, E,
                                                    1.f / ((float)B * (float)E), loss_sum, dF);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_affine_combine(int n_in, const float* const* inputs, const float* coef1, const float* coef2,
                       const float* bf16_scale, int B, long long E, float* out1, float* out2,
                       void* out_bf16, int clip, float clip_lo, float clip_hi, void* stream) {
  FDX_REQUIRE(n_in >= 1 && n_in <= 6 && inputs && coef1, "affine_combine: bad inputs");
  FDX_REQUIRE(B > 0 && E > 0 && E % 4 == 0, "affine_combine: E=%lld must be a multiple of 4", E);
  FDX_REQUIRE(!out2 || coef2, "affine_combine: out2 needs coef2");
  AffineArgs a{};
  for (int i = 0; i < n_in; ++i) {
    FDX_REQUIRE(inputs[i], "affine_combine: null input %d", i);
    a.in[i] = inputs[i];
  }
  a.n_in = n_in; a.a = coef1; a.c = out2 ? coef2 : nullptr; a.s = bf16_scale;
  a.out1 = out1; a.out2 = out2; a.out_bf16 = (__nv_bfloat16*)out_bf16;
  a.clip = clip; a.clip_lo = clip_lo; a.clip_hi = clip_hi;
  const long long t4 = (long long)B * E / 4;
  affine_kernel<<<stream_grid(t4, 256), 256, 0, (cudaStream_t)stream>>>(a, B, E);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_cast_f32_bf16(const float* src, void* dst, long long n, void* stream) {
  FDX_REQUIRE(src && dst && n > 0 && n % 4 == 0, "cast: bad arguments (n %% 4 == 0 required)");
  cast_bf16_kernel<<<stream_grid(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(
      src, (__nv_bfloat16*)dst, n);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_upsample2x(const fdx_act* x, const fdx_act* y, void* stream) {
  FDX_REQUIRE(x && y && x->ptr && y->ptr, "upsample2x: null tensor");
  FDX_REQUIRE(y->n == x->n && y->h == 2 * x->h && y->w == 2 * x->w && y->c == x->c && x->c % 8 == 0,
              "upsample2x: shape mismatch");
  const long long total = (long long)y->n * y->h * y->w * (x->c / 8);
  upsample2x_kernel<<<stream_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x->ptr, x->pix_stride, x->n, x->h, x->w, x->c, (__nv_bfloat16*)y->ptr,
      y->pix_stride);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_upsample2x_bwd(const fdx_act* dy, const fdx_act* dx, int accumulate, void* stream) {
  FDX_REQUIRE(dx && dy && dx->ptr && dy->ptr, "upsample2x_bwd: null tensor");
  FDX_REQUIRE(dy->n == dx->n && dy->h == 2 * dx->h && dy->w == 2 * dx->w && dy->c == dx->c &&
                  dx->c % 8 == 0,
              "upsample2x_bwd: shape mismatch");
  const long long total = (long long)dx->n * dx->h * dx->w * (dx->c / 8);
  upsample2x_bwd_kernel<<<stream_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)dy->ptr, dy->pix_stride, dx->n, dx->h, dx->w, dx->c,
      (__nv_bfloat16*)dx->ptr, dx->pix_stride, accumulate);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_act_add(const fdx_act* a, const fdx_act* b, const fdx_act* out, void* stream) {
  FDX_REQUIRE(a && b && out && a->ptr && b->ptr && out->ptr, "act_add: null tensor");
  FDX_REQUIRE(a->c == b->c && a->c == out->c && a->c % 8 == 0, "act_add: channel mismatch");
  const long long npix = (long long)a->n * a->h * a->w;
  FDX_REQUIRE(npix == (long long)b->n * b->h * b->w && npix == (long long)out->n * out->h * out->w,
              "act_add: shape mismatch");
  act_add_kernel<<<stream_grid(npix * (a->c / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)a->ptr, a->pix_stride, (const __nv_bfloat16*)b->ptr, b->pix_stride,
      (__nv_bfloat16*)out->ptr, out->pix_stride, npix, a->c);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_colsum(const fdx_act* x, float* out, int per_image, void* stream) {
  FDX_REQUIRE(x && x->ptr && out, "colsum: null pointer");
  FDX_REQUIRE(x->c % 8 == 0 && x->c / 8 <= 256, "colsum: bad channel count %d", x->c);
  const int HW = x->h * x->w;
  const int rows = 256 / (x->c / 8);
  int bx = (HW + 4 * rows - 1) / (4 * rows);
  int target = (16 * fdx_num_sms() + x->n - 1) / x->n;
  if (bx > target) bx = target;
  if (bx < 1) bx = 1;
  cudaStream_t st = (cudaStream_t)stream;
  FDX_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * x->c * (per_image ? x->n : 1), st));
  int gy = x->n;
  if (!per_image) {
    gy = 592 / bx;     // ~4 blocks per SM; every output address then sees < 600 atomics
    if (gy < 1) gy = 1;
    if (gy > x->n) gy = x->n;
  }
  colsum_kernel<<<dim3(bx, gy), 256, sizeof(float) * rows * x->c, st>>>(
      (const __nv_bfloat16*)x->ptr, x->pix_stride, x->n, HW, x->c, out, per_image ? x->c : 0);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
