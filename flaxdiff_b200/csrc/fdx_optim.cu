// fdx_optim.cu -- the O(parameters) streaming stage of a training step over ONE flat f32 buffer:
//   optax.adam / adamw / lamb  (+ optax.clip_by_global_norm)        /root/reference/training.py:263-267,594-608
//   flax TrainState.apply_gradients                                  trainer/general_diffusion_trainer.py:311,327
//   TrainState.apply_ema                                             trainer/diffusion_trainer.py:31-37
//   flax.training.dynamic_scale.DynamicScale step semantics          trainer/general_diffusion_trainer.py:305-318
// HBM-bound: 16-byte vector accesses, grid = 8 resident blocks per SM, one pass per kernel.
//   adam / adamw : p, g, m, v, ema read + p, m, v, ema, bf16 shadow written = 38 B per parameter, ONE kernel
//   lamb         : the trust ratio ||p|| / ||u|| is per parameter TENSOR, so the step is two passes: pass 1
//                  updates m, v, writes the un-scaled update u and accumulates per-tensor ||p||^2, ||u||^2
//                  (segment = binary search of the element index in the layout's offset table), pass 2
//                  applies p -= lr * ratio[seg] * u and the EMA / shadow refresh.
//                  The per-tensor norms run over whole 64-element slots, so the alignment gaps between
//                  tensors must be zero in p, g, m and v (then they stay zero in m, v and u): the trainer
//                  zeroes the gradient buffer before every backward pass, and parameters and moments
//                  start zero-filled.  A non-zero gap would enter its tensor's trust ratio.
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

// gradient multiplier shared by every optimiser kernel: 1/world (grad_scale), 1/loss-scale (DynamicScale)
// and optax.clip_by_global_norm's min(1, clip / ||g||); `skip` = this step's gradients are not finite.
struct GradScale {
  float mul;
  bool skip;
};
__device__ __forceinline__ GradScale grad_scale_of(float gscale, const float* __restrict__ gstats,
                                                    float clip_norm, const float* __restrict__ dynscale) {
  GradScale r;
  r.mul = gscale;
  r.skip = false;
  if (dynscale) {
    r.mul /= dynscale[0];
    r.skip = gstats && gstats[1] > 0.f;
  }
  if (gstats && clip_norm > 0.f) {
    // gstats[0] = sum (g / loss scale)^2: fdx_grad_stats unscaled before squaring, so the norm stays finite
    // at any loss scale; grad_scale is applied here
    const float nrm = sqrtf(gstats[0]) * gscale;          // norm of the TRUE (averaged, unscaled) gradient
    if (nrm > clip_norm) r.mul *= clip_norm / nrm;
  }
  return r;
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, float* __restrict__ ema, __nv_bfloat16* __restrict__ shadow,
                            long long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2,
                            float ema_decay, float gscale, const float* __restrict__ gstats, float clip_norm,
                            const float* __restrict__ dyn, const float* __restrict__ dynscale) {
  if (dyn) { lr = dyn[0]; bc1 = dyn[1]; bc2 = dyn[2]; }
  const GradScale gs = grad_scale_of(gscale, gstats, clip_norm, dynscale);
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    float pp[4] = {P.x, P.y, P.z, P.w};
    if (!gs.skip) {
      const float4 G = reinterpret_cast<const float4*>(g)[i];
      float4 M = reinterpret_cast<float4*>(m)[i];
      float4 V = reinterpret_cast<float4*>(v)[i];
      float gg[4] = {G.x, G.y, G.z, G.w}, mm[4] = {M.x, M.y, M.z, M.w}, vv[4] = {V.x, V.y, V.z, V.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gj = gg[j] * gs.mul;
        mm[j] = b1 * mm[j] + (1.f - b1) * gj;
        vv[j] = b2 * vv[j] + (1.f - b2) * gj * gj;
        const float mh = mm[j] / bc1, vh = vv[j] / bc2;
        pp[j] -= lr * (mh / (sqrtf(vh) + eps) + wd * pp[j]);
      }
      reinterpret_cast<float4*>(p)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
      reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
      reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
      if (shadow) {
        uint2 o;
        o.x = pack_bf16x2(pp[0], pp[1]);
        o.y = pack_bf16x2(pp[2], pp[3]);
        reinterpret_cast<uint2*>(shadow)[i] = o;
      }
    }
    if (ema) {   // apply_ema runs after the (possibly skipped) update, on whatever the parameters now are
      float4 Em = reinterpret_cast<float4*>(ema)[i];
      Em.x = ema_decay * Em.x + (1.f - ema_decay) * pp[0];
      Em.y = ema_decay * Em.y + (1.f - ema_decay) * pp[1];
      Em.z = ema_decay * Em.z + (1.f - ema_decay) * pp[2];
      Em.w = ema_decay * Em.w + (1.f - ema_decay) * pp[3];
      reinterpret_cast<float4*>(ema)[i] = Em;
    }
  }
}

// segment of element index e: largest s with off[s] <= e (off sorted, off[0] == 0)
__device__ __forceinline__ int seg_of(const long long* __restrict__ off, int nseg, long long e) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void lamb_pass1_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                  float* __restrict__ v, float* __restrict__ u, long long n, float b1, float b2,
                                  float eps, float wd, float bc1, float bc2, float gscale,
                                  const float* __restrict__ gstats, float clip_norm, const float* __restrict__ dyn,
                                  const float* __restrict__ dynscale, const long long* __restrict__ off, int nseg,
                                  float* __restrict__ norms) {
  if (dyn) { bc1 = dyn[1]; bc2 = dyn[2]; }
  const GradScale gs = grad_scale_of(gscale, gstats, clip_norm, dynscale);
  if (gs.skip) return;
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 P = reinterpret_cast<const float4*>(p)[i];
    const float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 M = reinterpret_cast<float4*>(m)[i];
    float4 V = reinterpret_cast<float4*>(v)[i];
    const float pp[4] = {P.x, P.y, P.z, P.w}, gg[4] = {G.x, G.y, G.z, G.w};
    float mm[4] = {M.x, M.y, M.z, M.w}, vv[4] = {V.x, V.y, V.z, V.w}, uu[4];
    float sp = 0.f, su = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = gg[j] * gs.mul;
      mm[j] = b1 * mm[j] + (1.f - b1) * gj;
      vv[j] = b2 * vv[j] + (1.f - b2) * gj * gj;
      uu[j] = (mm[j] / bc1) / (sqrtf(vv[j] / bc2) + eps) + wd * pp[j];
      sp = fmaf(pp[j], pp[j], sp);
      su = fmaf(uu[j], uu[j], su);
    }
    reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    reinterpret_cast<float4*>(u)[i] = make_float4(uu[0], uu[1], uu[2], uu[3]);
    // tensors start at multiples of 64 elements (ParamLayout.ALIGN): a float4 never straddles two;
    // the padding between tensors is zero in p and u and adds nothing
    const int s = seg_of(off, nseg, 4 * i);
    const int s0 = __shfl_sync(__activemask(), s, __ffs(__activemask()) - 1);
    if (__all_sync(__activemask(), s == s0) && __activemask() == 0xffffffffu) {
      sp = warp_sum(sp);
      su = warp_sum(su);
      if ((threadIdx.x & 31) == 0) { atomicAdd(norms + 2 * s, sp); atomicAdd(norms + 2 * s + 1, su); }
    } else {
      atomicAdd(norms + 2 * s, sp);
      atomicAdd(norms + 2 * s + 1, su);
    }
  }
}

__global__ void lamb_pass2_kernel(float* __restrict__ p, const float* __restrict__ u, float* __restrict__ ema,
                                  __nv_bfloat16* __restrict__ shadow, long long n, float lr, float ema_decay,
                                  const float* __restrict__ gstats, const float* __restrict__ dyn,
                                  const float* __restrict__ dynscale, const long long* __restrict__ off, int nseg,
                                  const float* __restrict__ norms) {
  if (dyn) lr = dyn[0];
  const bool skip = dynscale && gstats && gstats[1] > 0.f;
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    if (!skip) {
      const float4 U = reinterpret_cast<const float4*>(u)[i];
      const int s = seg_of(off, nseg, 4 * i);
      // optax.scale_by_trust_ratio: ||p|| / ||u||, 1 where either norm is zero
      const float pn = sqrtf(norms[2 * s]), un = sqrtf(norms[2 * s + 1]);
      const float ratio = (pn == 0.f || un == 0.f) ? 1.f : pn / un;
      const float a = lr * ratio;
      P.x -= a * U.x; P.y -= a * U.y; P.z -= a * U.z; P.w -= a * U.w;
      reinterpret_cast<float4*>(p)[i] = P;
      if (shadow) {
        uint2 o;
        o.x = pack_bf16x2(P.x, P.y);
        o.y = pack_bf16x2(P.z, P.w);
        reinterpret_cast<uint2*>(shadow)[i] = o;
      }
    }
    if (ema) {
      float4 Em = reinterpret_cast<float4*>(ema)[i];
      Em.x = ema_decay * Em.x + (1.f - ema_decay) * P.x;
      Em.y = ema_decay * Em.y + (1.f - ema_decay) * P.y;
      Em.z = ema_decay * Em.z + (1.f - ema_decay) * P.z;
      Em.w = ema_decay * Em.w + (1.f - ema_decay) * P.w;
      reinterpret_cast<float4*>(ema)[i] = Em;
    }
  }
}

__global__ void ema_kernel(float* __restrict__ ema, const float* __restrict__ p, long long n, float decay) {
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 E = reinterpret_cast<float4*>(ema)[i];
    const float4 P = reinterpret_cast<const float4*>(p)[i];
    E.x = decay * E.x + (1.f - decay) * P.x;
    E.y = decay * E.y + (1.f - decay) * P.y;
    E.z = decay * E.z + (1.f - decay) * P.z;
    E.w = decay * E.w + (1.f - decay) * P.w;
    reinterpret_cast<float4*>(ema)[i] = E;
  }
}

// out[0] += sum (g / dynscale[0])^2 (sum g^2 without dynscale), out[1] += number of non-finite elements of g
__global__ void grad_stats_kernel(const float* __restrict__ g, long long n, const float* __restrict__ dynscale,
                                  float* __restrict__ out) {
  const float mul = dynscale ? 1.f / dynscale[0] : 1.f;
  float acc = 0.f, bad = 0.f;
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    const float x = v.x * mul, y = v.y * mul, z = v.z * mul, w = v.w * mul;
    acc += x * x + y * y + z * z + w * w;
    // element by element: finite values whose sum overflows are still finite
    bad += (float)(!isfinite(v.x)) + (float)(!isfinite(v.y)) + (float)(!isfinite(v.z)) + (float)(!isfinite(v.w));
  }
  acc = warp_sum(acc);
  bad = warp_sum(bad);
  __shared__ float sh[2][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { sh[0][wid] = acc; sh[1][wid] = bad; }
  __syncthreads();
  if (wid == 0) {
    float a = lane < (blockDim.x >> 5) ? sh[0][lane] : 0.f;
    float b = lane < (blockDim.x >> 5) ? sh[1][lane] : 0.f;
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) { atomicAdd(out, a); if (b > 0.f) atomicAdd(out + 1, b); }
  }
}

// flax DynamicScale.value_and_grad's scale update: state = {scale, fin_steps, last_is_finite}
__global__ void dynscale_update_kernel(float* __restrict__ st, const float* __restrict__ gstats, float growth,
                                       float backoff, float interval, float min_scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const bool fin = !(gstats[1] > 0.f);
  const float scale = st[0], steps = st[1];
  const bool grow = (steps == interval);
  const float fin_scale = (grow && fin) ? fminf(scale * growth, 3.402823466e38f) : scale;
  const float inf_scale = fmaxf(scale * backoff, min_scale);
  st[0] = fin ? fin_scale : inf_scale;
  st[1] = (grow || !fin) ? 0.f : steps + 1.f;
  st[2] = fin ? 1.f : 0.f;
}

}  // namespace

extern "C" {

int fdx_optimizer_step(const fdx_opt_desc* d, void* stream) {
  FDX_REQUIRE(d && d->p && d->g && d->m && d->v, "optimizer_step: null pointer");
  FDX_REQUIRE(d->n > 0 && d->n % 4 == 0, "optimizer_step: n=%lld must be a multiple of 4 (pad the flat buffer)", d->n);
  FDX_REQUIRE(d->step >= 1, "optimizer_step: step counts from 1");
  FDX_REQUIRE(d->kind == FDX_OPT_ADAM || d->kind == FDX_OPT_LAMB, "optimizer_step: unknown kind %d", d->kind);
  FDX_REQUIRE(!d->dynscale || d->gstats, "optimizer_step: DynamicScale needs the fdx_grad_stats output");
  cudaStream_t st = (cudaStream_t)stream;
  const float bc1 = 1.f - powf(d->b1, (float)d->step), bc2 = 1.f - powf(d->b2, (float)d->step);
  const int grid = stream_grid(d->n / 4, 256);
  if (d->kind == FDX_OPT_ADAM) {
    adam_kernel<<<grid, 256, 0, st>>>(d->p, d->g, d->m, d->v, d->ema, (__nv_bfloat16*)d->shadow_bf16, d->n, d->lr,
                                      d->b1, d->b2, d->eps, d->weight_decay, bc1, bc2, d->ema_decay, d->grad_scale,
                                      d->gstats, d->clip_norm, d->dyn_lr_bc, d->dynscale);
    FDX_LAUNCH_CHECK();
    return FDX_OK;
  }
  FDX_REQUIRE(d->seg_offsets && d->nseg > 0 && d->seg_norms && d->u_ws,
              "optimizer_step: lamb needs the segment table and its workspaces");
  FDX_CUDA(cudaMemsetAsync(d->seg_norms, 0, sizeof(float) * 2 * (size_t)d->nseg, st));
  lamb_pass1_kernel<<<grid, 256, 0, st>>>(d->p, d->g, d->m, d->v, d->u_ws, d->n, d->b1, d->b2, d->eps,
                                          d->weight_decay, bc1, bc2, d->grad_scale, d->gstats, d->clip_norm,
                                          d->dyn_lr_bc, d->dynscale, d->seg_offsets, d->nseg, d->seg_norms);
  FDX_LAUNCH_CHECK();
  lamb_pass2_kernel<<<grid, 256, 0, st>>>(d->p, d->u_ws, d->ema, (__nv_bfloat16*)d->shadow_bf16, d->n, d->lr,
                                          d->ema_decay, d->gstats, d->dyn_lr_bc, d->dynscale, d->seg_offsets,
                                          d->nseg, d->seg_norms);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_adamw_ema_step(float* p, const float* g, float* m, float* v, float* ema, void* shadow_bf16,
                       long long n, float lr, float b1, float b2, float eps, float weight_decay,
                       int step, float ema_decay, float grad_scale, const float* gnorm_sq,
                       float clip_norm, const float* dyn_lr_bc, void* stream) {
  FDX_REQUIRE(ema, "adamw_ema: null ema pointer (use fdx_optimizer_step for an update without EMA)");
  fdx_opt_desc d{};
  d.kind = FDX_OPT_ADAM;
  d.p = p; d.g = g; d.m = m; d.v = v; d.ema = ema; d.shadow_bf16 = shadow_bf16; d.n = n;
  d.lr = lr; d.b1 = b1; d.b2 = b2; d.eps = eps; d.weight_decay = weight_decay; d.step = step;
  d.ema_decay = ema_decay; d.grad_scale = grad_scale; d.gstats = gnorm_sq; d.clip_norm = clip_norm;
  d.dyn_lr_bc = dyn_lr_bc;
  return fdx_optimizer_step(&d, stream);
}

int fdx_ema_update(float* ema, const float* p, long long n, float decay, void* stream) {
  FDX_REQUIRE(ema && p && n > 0 && n % 4 == 0, "ema_update: bad arguments");
  ema_kernel<<<stream_grid(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(ema, p, n, decay);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_grad_stats(const float* g, long long n, const float* dynscale, float* out2, void* stream) {
  FDX_REQUIRE(g && out2 && n > 0 && n % 4 == 0, "grad_stats: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  FDX_CUDA(cudaMemsetAsync(out2, 0, 2 * sizeof(float), st));
  grad_stats_kernel<<<stream_grid(n / 4, 256), 256, 0, st>>>(g, n, dynscale, out2);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_sumsq(const float* g, long long n, float* out, void* stream) {
  // kept for callers that only need the norm: out[0] = sum g^2 (out must hold 2 floats: see fdx_grad_stats)
  return fdx_grad_stats(g, n, nullptr, out, stream);
}

int fdx_dynscale_update(float* state3, const float* gstats, float growth_factor, float backoff_factor,
                        int growth_interval, float minimum_scale, void* stream) {
  FDX_REQUIRE(state3 && gstats, "dynscale_update: null pointer");
  dynscale_update_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(state3, gstats, growth_factor, backoff_factor,
                                                             (float)growth_interval, minimum_scale);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
