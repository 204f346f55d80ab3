/* fdx.h -- C-ABI of libfdx.so, the H100 (sm_90a) kernel library under the
 * flaxdiff_b200 Python surface.
 *
 * The reference (AshishKumar4/FlaxDiff) has no FFI / plugin interface: every device
 * op on its UNet hot path is a flax.linen / jax.numpy call lowered by XLA.  Each entry
 * point below names the reference call site (file:line under /root/reference) whose
 * XLA lowering it replaces.  Conventions:
 *   - plain pointers + sizes, caller-owned DEVICE buffers, no hidden allocation;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it;
 *   - return 0 on success, <0 on error (fdx_last_error() gives the message);
 *   - activations are NHWC bf16 unless stated, described by fdx_act (a pixel stride
 *     larger than c lets producers write straight into channel slots of a concat
 *     buffer: jnp.concatenate at flaxdiff/models/simple_unet.py:145,196 is free);
 *   - conv kernels are HWIO [3][3][Cin][Cout] exactly as flax stores them.
 */
#ifndef FDX_H_
#define FDX_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FDX_OK 0
#define FDX_ERR_INVALID_ARG (-1)
#define FDX_ERR_UNSUPPORTED (-2)
#define FDX_ERR_CUDA (-3)
#define FDX_ERR_NO_DEVICE (-4)

typedef struct fdx_act {
  void* ptr;            /* device pointer to element (n=0,y=0,x=0,c=0) */
  int n, h, w, c;       /* logical dims */
  long long pix_stride; /* elements between consecutive pixels (>= c, multiple of 8) */
} fdx_act;

/* ---- library ---------------------------------------------------------------- */
const char* fdx_last_error(void);
int fdx_version(void);
int fdx_device_sm_count(void);
/* number of libfdx kernels launched (or captured into a CUDA graph) by this process so far */
unsigned long long fdx_launch_count(void);
/* tensor-core kernel family of the most recent launch (-1 = none yet) and its SASS-visible kernel name: lets a
 * profiler attribute a CUDA-event interval around one C-ABI call to the kernel that ran (bench.py roofline). */
#define FDX_KERNEL_TC 0       /* fdx_tc_kernel: pixels-as-M tap-GEMM engine */
#define FDX_KERNEL_TCT 1      /* fdx_tct_kernel: transposed (weights-as-M) engine */
/* 2 and 4: retired kernel families */
#define FDX_KERNEL_WGRAD9 3   /* fdx_wgrad9_kernel: nine-tap weight gradient, ky in M / kx in N */
#define FDX_KERNEL_ATTN_FWD 5 /* fdx_attn_fwd_kernel: fused attention forward */
#define FDX_KERNEL_ATTN_BWD 6 /* fdx_attn_bwd_kernel: fused attention backward */
int fdx_last_kernel_kind(void);
const char* fdx_kernel_kind_name(int kind);

/* ---- tensor-core contractions (wgmma + TMA) ----------------------------------- */
/* flax nn.Conv 3x3 SAME, stride 1 or 2 (models/common.py:166-172, 237-244).
 * y = conv(x, w) + bias + rowvec[n] + res ; bias [Cout] f32, rowvec [N][Cout] f32 (the
 * ResidualBlock's `out + temb` add, common.py:300-308), res = residual add (common.py:334).
 * w_hwio is bf16.  Cin, Cout multiples of 64. */
int fdx_conv3x3_fwd(const fdx_act* x, const void* w_hwio, const float* bias, const float* rowvec,
                    const fdx_act* res, const fdx_act* y, int stride, void* stream);
/* Same convolution, additionally accumulating per (image, output channel) the sum and the sum of
 * squares of the stored bf16 values - the statistics of the GroupNorm that consumes y
 * (models/common.py:273-288), so that norm needs no pass of its own over y.
 * cs->ws = f32 [slots][N][2][ld], zeroed by the caller (the sums are added onto what it holds), pre-offset to
 * y's first channel inside the destination buffer (ld = that buffer's channel count); 1 <= slots <= 64, cs->ws
 * 16-byte aligned and ld a multiple of 4, else FDX_ERR_INVALID_ARG.
 * FDX_ERR_UNSUPPORTED when an image of y has fewer than 128 pixels.  fdx_groupnorm_stats_from_cols turns the
 * sums into fdx_groupnorm_stats' output. */
typedef struct fdx_colstats {
  float* ws;
  int slots;
  int ld;
} fdx_colstats;
int fdx_conv3x3_fwd_stats(const fdx_act* x, const void* w_hwio, const float* bias, const float* rowvec,
                          const fdx_act* res, const fdx_act* y, int stride, const fdx_colstats* cs,
                          void* stream);
int fdx_groupnorm_stats_from_cols(const float* cols, int slots, int N, int ld, int c0, int C, int groups,
                                  float* stats, void* stream);   /* channels [c0, c0+C) of the ld-wide rows */
/* d(loss)/dx of the conv above (jax.value_and_grad, trainer/general_diffusion_trainer.py:321). */
int fdx_conv3x3_dgrad(const fdx_act* dy, const void* w_hwio, const fdx_act* dx, int stride,
                      int accumulate, void* stream);
/* d(loss)/dw, f32 HWIO, ACCUMULATED into dw_hwio (caller zeroes it). */
int fdx_conv3x3_wgrad(const fdx_act* x, const fdx_act* dy, float* dw_hwio, int stride,
                      void* stream);

/* 1x1 convolution in convolution geometry (ResidualBlock.residual_conv, models/common.py:324-333):
 * y = x W + bias + res with W = [Cin][Cout] bf16 (flax (1,1,Cin,Cout) kernel), and its data gradient
 * dx (+)= dy W^T.  Same arithmetic as fdx_gemm on the flattened pixels, but eligible for the transposed
 * engine (few output columns, one or two K chunks: epilogue / bandwidth bound layers). */
int fdx_conv1x1_fwd(const fdx_act* x, const void* w_io, const float* bias, const fdx_act* res, const fdx_act* y,
                    void* stream);
int fdx_conv1x1_dgrad(const fdx_act* dy, const void* w_io, const fdx_act* dx, int accumulate, void* stream);

#define FDX_GEMM_KK 0   /* D[m][n] = sum_k A[m][k] * B[n][k]   (both k-contiguous)   */
#define FDX_GEMM_KMN 1  /* D[m][n] = sum_k A[m][k] * B[k][n]                          */
#define FDX_GEMM_MNMN 2 /* D[m][n] = sum_k A[k][m] * B[k][n]   (weight-gradient type) */
typedef struct {
  int mode;
  int M, N, K;
  int batch1, batch2;      /* two batch dims (e.g. heads, images); 0/1 = none */
  const void* A; long long a_ld, a_s1, a_s2; /* bf16; leading dim and batch strides, elements */
  const void* B; long long b_ld, b_s1, b_s2; /* bf16; b_s1 = b_s2 = 0 -> B shared by the batch */
  void* D; long long d_ld, d_s1, d_s2;
  int d_f32;               /* output dtype: 0 bf16, 1 f32 */
  int d_atomic;            /* f32 atomicAdd into D (split-K allowed) */
  int reduce_batch;        /* MNMN only: also reduce over the batch dims (dense weight grads) */
  float alpha;
  const float* bias;       /* [N] or NULL; added once per output, also under split-K */
  const void* res; long long r_ld, r_s1, r_s2; /* bf16 residual added to D, or NULL */
} fdx_gemm_desc;
/* 1x1 conv (common.py:324-333), nn.DenseGeneral (attention.py:132-154, common.py:300-305),
 * and the QK^T / PV / backward products of nn.dot_product_attention (attention.py:170-174). */
int fdx_gemm(const fdx_gemm_desc* g, void* stream);
/* fdx_gemm with an A operand from two row matrices, as over the concatenation [A0 | A1] along k without writing it:
 * A[m][k] = A0[m][k] (g->A, row stride g->a_ld) for k < K0 and A1[m][k - K0] (row stride a1_ld) for k >= K0.  The
 * product runs fdx_gemm's k-block order and single f32 accumulation, so D is bit for bit fdx_gemm's on the
 * materialised concatenation (same bias, res, output type).  KK and KMN modes, batch 1, 0 < K0 < K with K0 a multiple
 * of 64; A0 and A1 16-byte aligned, row strides multiples of 8.  The skip-connection Dense of SimpleUDiT
 * (simple_vit.py:427-430) and its float32 output projection (as [x | x] x [W_hi; W_lo]). */
int fdx_gemm_cat(const fdx_gemm_desc* g, const void* A1, long long a1_ld, int K0, void* stream);

/* Upsample = jax.image.resize(nearest, x2) + ConvLayer 3x3 (models/common.py:210-226) without materialising
 * the upsampled tensor: four output parities, each a 2x2 convolution of the LOW-resolution input with
 * summed taps (4/9 of the FLOPs).  x / dx are the low-resolution tensors, y / dy the full-resolution ones.
 *   fdx_upconv3x3_pack  : weff bf16 [4 parities][2][2][Cin][Cout] from the f32 HWIO master weights
 *   fdx_upconv3x3_fwd   : y = conv3x3(nearest2x(x)) + bias
 *   fdx_upconv3x3_dgrad : dx (+)= d/dx, one 16-tap launch
 *   fdx_upconv3x3_wgrad : dw_hwio += d/dw; dweff_ws = f32 scratch of 16*Cin*Cout floats */
int fdx_upconv3x3_pack(const float* w_hwio, int cin, int cout, void* weff_bf16, void* stream);
int fdx_upconv3x3_fwd(const fdx_act* x, const void* weff_bf16, const float* bias, const fdx_act* y,
                      void* stream);
int fdx_upconv3x3_fwd_stats(const fdx_act* x, const void* weff_bf16, const float* bias, const fdx_act* y,
                            const fdx_colstats* cs, void* stream);   /* cs as in fdx_conv3x3_fwd_stats */
int fdx_upconv3x3_dgrad(const fdx_act* dy, const void* weff_bf16, const fdx_act* dx, int accumulate,
                        void* stream);
int fdx_upconv3x3_wgrad(const fdx_act* x, const fdx_act* dy, float* dweff_ws, float* dw_hwio,
                        void* stream);

/* ---- normalisation (HBM-bound; warp-shuffle + shared/global atomics reductions) ---- */
/* nn.GroupNorm(groups, eps) statistics (models/common.py:273-281): stats[n][g] = (sum, sumsq), f32. */
int fdx_groupnorm_stats(const fdx_act* x, int groups, float* stats, void* stream);
/* y = act((x-mean)*rstd*gamma+beta) (models/common.py:286-288,310-312; simple_unet.py:209-210).
 * act selects the activation, as in every GroupNorm entry point below: 0 = none, 1 = silu (swish),
 * 2 = mish (z * tanh(softplus(z)), jax.nn.mish); any other value is FDX_ERR_INVALID_ARG. */
int fdx_groupnorm_apply(const fdx_act* x, int groups, const float* stats, const float* gamma,
                        const float* beta, float eps, int act, const fdx_act* y, void* stream);
/* fdx_groupnorm_apply with the statistics taken straight from the producers' epilogue column sums
 * (cols = [slots][N][2][ld] as written by fdx_conv3x3_fwd_stats / fdx_upconv3x3_fwd_stats, channels c0 .. c0+C of
 * the buffer): no fdx_groupnorm_stats_from_cols launch; stats_out[N][groups][2] receives the statistics for the
 * backward. */
int fdx_groupnorm_apply_cols(const fdx_act* x, int groups, const float* cols, int slots, int ld, int c0,
                             const float* gamma, const float* beta, float eps, int act, const fdx_act* y,
                             float* stats_out, void* stream);
/* Backward of the pair above.  ws: f32 scratch of 2*N*groups floats.  dgamma/dbeta ACCUMULATED.
 * csum_img [n][c] / csum_tot [c] (NULL allowed; csum_tot needs csum_img): column sums over pixels of the
 * dx this call produces, written (not accumulated) - the timestep row-vector and conv-bias gradients. */
int fdx_groupnorm_bwd(const fdx_act* x, const fdx_act* dy, int groups, const float* stats,
                      const float* gamma, const float* beta, float eps, int act, float* ws,
                      float* dgamma, float* dbeta, const fdx_act* dx, int accumulate,
                      float* csum_img, float* csum_tot, void* stream);
/* Same, with the result ADDED to another tensor: dx = d/dx + addend (addend may be dx itself = accumulate).  The
 * ResidualBlock's skip gradient (common.py:334-336: out + residual) joins here instead of in a separate pass. */
int fdx_groupnorm_bwd_add(const fdx_act* x, const fdx_act* dy, int groups, const float* stats,
                          const float* gamma, const float* beta, float eps, int act, float* ws,
                          float* dgamma, float* dbeta, const fdx_act* dx, const fdx_act* addend,
                          float* csum_img, float* csum_tot, void* stream);
/* Fused variant of the backward above: the data-gradient convolution that PRODUCES dy applies
 * act'(z) in its epilogue and accumulates the first-pass sums, so x and dy are read once less.
 *   fdx_groupnorm_coeffs : ab[n][0][c] = rstd*gamma_c, ab[n][1][c] = beta_c - mean*rstd*gamma_c
 *   fdx_conv3x3_dgrad_gn : stride-1 3x3 data gradient (as fdx_conv3x3_dgrad) writing
 *                          dz = dgrad * silu'(a x + b) and ws_slots[slot][n][{0,1}][c] += (sum dz, sum dz*x);
 *                          zeroes ws_slots (slots*N*2*C floats) itself; FDX_ERR_UNSUPPORTED when an image
 *                          has fewer than 128 pixels (caller then uses the two-pass path)
 *   fdx_conv3x3_dgrad_gn_act : the same with act'(z), act = 1 (silu; = fdx_conv3x3_dgrad_gn) or 2 (mish).
 *                          Mish runs on the transposed engine only: FDX_ERR_UNSUPPORTED where it does not take
 *                          the layer (Cin not in 64 .. 512, or a multiple of 256; H or W not a multiple of 16),
 *                          and the caller uses fdx_conv3x3_dgrad + fdx_groupnorm_bwd(act = 2)
 *   fdx_groupnorm_bwd_dz : second pass from dz; ws is unused (NULL allowed). */
int fdx_groupnorm_coeffs(const float* stats, const float* gamma, const float* beta, int N, int HW, int C,
                         int groups, float eps, float* ab, void* stream);
int fdx_conv3x3_dgrad_gn(const fdx_act* dy, const void* w_hwio, const fdx_act* dz, const fdx_act* x,
                         const float* ab, float* ws_slots, int slots, void* stream);
int fdx_conv3x3_dgrad_gn_act(const fdx_act* dy, const void* w_hwio, const fdx_act* dz, const fdx_act* x,
                             const float* ab, float* ws_slots, int slots, int act, void* stream);
int fdx_groupnorm_bwd_dz(const fdx_act* x, const fdx_act* dz, int groups, const float* stats,
                         const float* gamma, float eps, const float* ws_slots, int slots, float* ws,
                         float* dgamma, float* dbeta, const fdx_act* dx, int accumulate, float* csum_img,
                         float* csum_tot, void* stream);
/* fdx_groupnorm_bwd_dz with dx = GroupNorm backward + addend (the identity-residual gradient of the
 * ResidualBlock, flaxdiff/models/common.py:334-336), as fdx_groupnorm_bwd_add. */
int fdx_groupnorm_bwd_dz_add(const fdx_act* x, const fdx_act* dz, int groups, const float* stats,
                             const float* gamma, float eps, const float* ws_slots, int slots, float* ws,
                             float* dgamma, float* dbeta, const fdx_act* dx, const fdx_act* addend,
                             float* csum_img, float* csum_tot, void* stream);
/* nn.RMSNorm(eps) over channels (models/attention.py:325-326). C a multiple of 8, <= 1024. */
int fdx_rmsnorm_fwd(const fdx_act* x, const float* scale, float eps, const fdx_act* y,
                    void* stream);
int fdx_rmsnorm_bwd(const fdx_act* x, const fdx_act* dy, const float* scale, float eps,
                    const fdx_act* dx, int accumulate, float* dscale, void* stream);

/* ---- diffusion step streaming kernels ------------------------------------------------ */
/* (x-127.5)/127.5, x_t = alpha*x0 + sigma*eps, target, model input bf16(x_t*c_in)
 * (trainer/general_diffusion_trainer.py:258,285-291; predictors/__init__.py:19-24).
 * target_kind: 0 = x0, 1 = eps, 2 = v.  E = elements per sample. */
int fdx_diffuse_forward(const void* x0, int x0_is_u8, const float* eps, const float* alpha,
                        const float* sigma, const float* c_in, int B, long long E, int normalize,
                        int target_kind, float* x_t, float* target, void* model_in_bf16,
                        void* stream);
/* pred = c_out*F + c_skip*x_t; loss = mean(0.5*(pred-target)^2*w); dF = dloss/dF
 * (general_diffusion_trainer.py:295-302; predictors/__init__.py:84-91). */
int fdx_loss_fwd_bwd(const float* F, const float* x_t, const float* target, const float* c_out,
                     const float* c_skip, const float* weight, int B, long long E,
                     float* loss_sum, float* dF, void* stream);
/* out1 = sum_i coef1[i][b]*in_i ; out2 = sum_i coef2[i][b]*in_i ; out_bf16 = bf16(out1*scale[b]).
 * One pass for x0/eps recovery, CFG mixing (samplers/common.py:93-96) and every sampler update
 * (samplers/euler.py:8-18,39-56; heun_sampler.py:7-27; ddim.py:30-47; ddpm.py:6-15).
 * clip != 0 clamps out1 to [clip_lo, clip_hi] as jnp.clip does: a NaN stays NaN. */
int fdx_affine_combine(int n_in, const float* const* inputs, const float* coef1, const float* coef2,
                       const float* bf16_scale, int B, long long E, float* out1, float* out2,
                       void* out_bf16, int clip, float clip_lo, float clip_hi, void* stream);
/* ---- jax.random's threefry streams (fdx_random.cu) ---------------------------------------------
 * The draws of jax.random.{bits, uniform, normal, randint} for a threefry2x32 key, as JAX 0.4.28 lays them out with
 * jax_threefry_partitionable=False: x_T and the per-step noise of the samplers (samplers/common.py:253-260,
 * euler.py:39-56, ddpm.py:6-37), the trainer's noise, timesteps and unconditional mask
 * (trainer/general_diffusion_trainer.py:266-283).  A draw of any shape is the flat draw of n elements, row-major.
 * The key is (k0, k1), or - when key_dev is non-null - the two words at key_dev in device memory, read by the
 * kernel: a captured graph is replayed with a new key by overwriting those 8 bytes.  0 <= n <= 2^31-1; `out` needs
 * 4-byte alignment only.  split / fold_in stay on the host (two threefry blocks).
 *   bits:    m = ceil(n/2); threefry2x32(key, [0..m), [m..2m)), the two outputs concatenated, first n words.
 *   uniform: f = bitcast((bits >> 9) | 0x3F800000) - 1; max(minval, f*(maxval-minval) + minval), every
 *            operation rounded to f32 on its own.  minval < maxval.
 *   normal:  sqrt(2) * erfinv(uniform(nextafter(-1, 0), 1)) with XLA's f32 erf_inv polynomial (Giles 2010).
 *   randint: k1, k2 = split(key); hi = bits(k1), lo = bits(k2); span = maxval - minval;
 *            mult = (2^16 mod span)^2 mod span; minval + ((hi mod span)*mult + lo mod span) mod span in wrapping
 *            uint32 arithmetic.  minval < maxval. */
int fdx_random_bits(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, uint32_t* out, void* stream);
int fdx_random_uniform(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, float minval, float maxval,
                       float* out, void* stream);
int fdx_random_normal(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, float* out, void* stream);
int fdx_random_randint(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, int minval, int maxval,
                       int32_t* out, void* stream);
/* ---- optimiser / EMA / loss scaling over ONE flat f32 buffer (fdx_optim.cu) -------------------- */
/* optax.adam / adamw / lamb (+ optax.clip_by_global_norm) as flax TrainState.apply_gradients does them
 * (training.py:263-267,594-608; trainer/general_diffusion_trainer.py:311,327), fused with
 * TrainState.apply_ema (trainer/diffusion_trainer.py:31-37) and the refresh of the bf16 weight shadow the
 * tensor-core kernels read.  `ema` NULL = apply_gradients only.  The gradient the update sees is
 *   g * grad_scale [/ dynscale[0]] * min(1, clip_norm / ||.||)    (||.|| = sqrt(gstats[0]) * grad_scale)
 * so with dynscale set, gstats must come from fdx_grad_stats called with the same dynscale: it then holds the
 * squared norm of the gradient with the loss scale removed, which stays finite at any loss scale.
 * and with `dynscale` set the parameter / moment update is SKIPPED when gstats[1] > 0 (non-finite gradients,
 * general_diffusion_trainer.py:313-318) while the EMA still runs on the unchanged parameters.
 * lamb: seg_offsets = the nseg tensor start offsets (elements, ascending, first = 0, multiples of 4),
 * seg_norms = f32 [nseg][2] scratch, u_ws = f32 [n] scratch (optax.scale_by_trust_ratio is per tensor). */
#define FDX_OPT_ADAM 0 /* adam (weight_decay = 0) and adamw */
#define FDX_OPT_LAMB 1
typedef struct fdx_opt_desc {
  int kind;
  float* p; const float* g; float* m; float* v;
  float* ema;               /* or NULL */
  void* shadow_bf16;        /* or NULL */
  long long n;              /* multiple of 4 */
  float lr, b1, b2, eps, weight_decay;
  int step;                 /* optimiser count after this step (>= 1): bias corrections */
  float ema_decay;
  float grad_scale;         /* e.g. 1/world after a sum all-reduce; 1 otherwise */
  const float* gstats;      /* device f32[2] from fdx_grad_stats, or NULL */
  float clip_norm;          /* 0 = no clipping */
  const float* dyn_lr_bc;   /* device {lr, 1-b1^t, 1-b2^t} overriding lr/step (CUDA-graph replay), or NULL */
  const float* dynscale;    /* device DynamicScale state {scale, fin_steps, last_finite}, or NULL */
  const long long* seg_offsets; int nseg; float* seg_norms; float* u_ws;   /* lamb only */
} fdx_opt_desc;
int fdx_optimizer_step(const fdx_opt_desc* d, void* stream);
/* adamw + EMA + shadow, the common case, without the descriptor (gnorm_sq = fdx_grad_stats output). */
int fdx_adamw_ema_step(float* p, const float* g, float* m, float* v, float* ema, void* shadow_bf16,
                       long long n, float lr, float b1, float b2, float eps, float weight_decay,
                       int step, float ema_decay, float grad_scale, const float* gnorm_sq,
                       float clip_norm, const float* dyn_lr_bc /* device {lr,1-b1^t,1-b2^t} or NULL */,
                       void* stream);
/* TrainState.apply_ema on its own: ema = decay*ema + (1-decay)*p (trainer/diffusion_trainer.py:31-37). */
int fdx_ema_update(float* ema, const float* p, long long n, float decay, void* stream);
/* out2[0] = sum (g / dynscale[0])^2, or sum g^2 with dynscale NULL (optax.clip_by_global_norm: the loss scale
 * is removed before squaring, so the sum stays finite at any scale), out2[1] = number of non-finite elements of
 * g, each tested on its own (DynamicScale's is_finite, flax/training/dynamic_scale.py via
 * general_diffusion_trainer.py:308).  fdx_sumsq = fdx_grad_stats(g, n, NULL, out2). */
int fdx_grad_stats(const float* g, long long n, const float* dynscale, float* out2, void* stream);
int fdx_sumsq(const float* g, long long n, float* out2, void* stream);
/* DynamicScale state update after a step: state3 = {scale, fin_steps, last_finite}; finite: after
 * growth_interval finite steps scale *= growth_factor; non-finite: scale = max(scale*backoff, minimum). */
int fdx_dynscale_update(float* state3, const float* gstats, float growth_factor, float backoff_factor,
                        int growth_interval, float minimum_scale, void* stream);

/* ---- data-parallel exchange (fdx_comm.cu): jax.lax.pmean of the gradients and the loss ---------------
 * (trainer/general_diffusion_trainer.py:325,334,340-345).  NCCL is bound at run time (dlopen); one
 * communicator per process, one process per GPU.  fdx_comm_allreduce_avg is asynchronous on `stream` and
 * may be called on sub-ranges ("buckets") of the flat gradient buffer while the backward pass still runs. */
typedef struct fdx_comm fdx_comm;
int fdx_comm_unique_id(void* id128 /* 128 bytes out; rank 0 creates it, every rank passes it to init */);
int fdx_comm_init(fdx_comm** out, int rank, int world, const void* id128);
int fdx_comm_allreduce_avg(fdx_comm* c, float* buf, long long n, void* stream);   /* in place, mean over ranks */
int fdx_comm_world(const fdx_comm* c, int* rank, int* world);
int fdx_comm_nccl_version(void);      /* 0 when NCCL cannot be bound */
int fdx_comm_destroy(fdx_comm* c);
int fdx_cast_f32_bf16(const float* src, void* dst, long long n, void* stream);
/* jax.image.resize(nearest) x2 (models/common.py:214-215) and its adjoint. */
int fdx_upsample2x(const fdx_act* x, const fdx_act* y, void* stream);
int fdx_upsample2x_bwd(const fdx_act* dy, const fdx_act* dx, int accumulate, void* stream);
int fdx_act_add(const fdx_act* a, const fdx_act* b, const fdx_act* out, void* stream);
/* column sums over pixels: out[c] or out[n][c] (bias / timestep-vector gradients). */
int fdx_colsum(const fdx_act* x, float* out, int per_image, void* stream);

/* ---- 3-channel convolutions (CUDA cores) ----------------------------------------------- */
/* conv_in 3->Cout (models/simple_unet.py:47-54): x bf16 [N,H,W,3] dense, w f32 HWIO. */
int fdx_conv_in_fwd(const void* x_bf16, int N, int H, int W, const float* w_hwio,
                    const float* bias, const fdx_act* y, void* stream);
int fdx_conv_in_wgrad(const void* x_bf16, const fdx_act* dy, float* dw_hwio, float* dbias,
                      void* stream);
/* im2col of a 3-channel tensor for the two weight gradients above/below as tensor-core GEMMs:
 * col[p][t*3+k] = src[p + sgn*d(t)][k] (zero outside the image), bf16 [N*H*W][32]; column 27 = 1 if
 * ones_col (bias row).  dW_in = col^T dY ; dW_out = x^T col (via fdx_gemm MNMN). */
int fdx_im2col3x3_c3(const void* src, int src_is_f32, int sgn, int N, int H, int W, int ones_col,
                     void* col_bf16, void* stream);
/* Scatter step of the tensor-core conv_out (models/simple_unet.py:212-221): col f32 [N*H*W][32] holds
 * <x[p], w[t][:][k]> at column t*3+k; y[p][k] = bias[k] + sum_t col[p + d(t)][t*3+k], SAME padding. */
int fdx_col2im3x3_c3(const float* col_f32, const float* bias, int N, int H, int W, float* y_f32,
                     void* stream);
/* conv_out Cin->3 (models/simple_unet.py:212-221): y f32 [N,H,W,3] dense. */
int fdx_conv_out_fwd(const fdx_act* x, const float* w_hwio, const float* bias, float* y_f32,
                     void* stream);
int fdx_conv_out_dgrad(const float* dF, const float* w_hwio, const fdx_act* dx, void* stream);
int fdx_conv_out_wgrad(const fdx_act* x, const float* dF, float* dw_hwio, float* dbias,
                       void* stream);

/* ---- timestep embedding + softmax ------------------------------------------------------ */
/* FourierEmbedding + TimeProjection (models/common.py:97-124), f32; saves four/h1/h2 for bwd. */
int fdx_time_embed_fwd(const float* t, const float* freqs, const float* W1, const float* b1,
                       const float* W2, const float* b2, int B, int D, float* four, float* h1,
                       float* h2, float* emb, void* emb_bf16, void* stream);
int fdx_time_embed_bwd(const float* demb, const float* four, const float* h1, const float* h2,
                       const float* W2, int B, int D, float* dh1_ws, float* dh2_ws, float* dW1,
                       float* db1, float* dW2, float* db2, void* stream);
/* softmax of nn.dot_product_attention (models/attention.py:170-174): S f32 -> P bf16.  Rows hold Lp
 * columns of which the first L are real keys (cross-attention to 77 text tokens is padded to 96). */
int fdx_softmax_fwd(const float* S, long long rows, int L, int Lp, void* P_bf16, void* stream);
int fdx_softmax_bwd(const void* P_bf16, const float* dP, long long rows, int L, int Lp, float scale,
                    void* dS_bf16, void* stream);

/* FlaxGEGLU of the full transformer block (models/attention.py:179-205): u bf16 [rows][2*inner] =
 * [hidden_linear | hidden_gelu] -> g = hidden_linear * gelu_tanh(hidden_gelu) bf16 [rows][inner], and its
 * backward du [rows][2*inner] from dg.  inner a multiple of 8. */
int fdx_geglu_fwd(const void* u_bf16, long long rows, int inner, void* g_bf16, void* stream);
int fdx_geglu_bwd(const void* u_bf16, const void* dg_bf16, long long rows, int inner, void* du_bf16,
                  void* stream);

/* ---- fused attention (fdx_attn.cu) ------------------------------------------------------------------
 * nn.dot_product_attention inside NormalAttention (models/attention.py:156-177): o = softmax(q k^T * scale) v
 * per (image, head), self-attention (Lk = L) or cross-attention to the text context (Lk = 77), and its
 * backward under jax.value_and_grad (trainer/general_diffusion_trainer.py:321).  The logits and probabilities
 * never reach HBM: flash-style wgmma kernels with S in registers and P in shared memory; the backward recomputes
 * them from `lse` (two kernels: dQ per query tile, dK + dV per key block; deterministic, no atomics).
 * Tensors: bf16 [B][rows][heads*dh], `*_ld` = elements between rows, `*_bs` = elements between images.  Every
 * `*_ld` and `*_bs` must be a multiple of 8 and q, k, v, o, d_o, dq, dk, dv 16-byte aligned (TMA boxes and
 * 16-byte vector accesses); otherwise FDX_ERR_INVALID_ARG, naming the field, before anything is launched.
 * dh (as STORED) is 32, 64, 128 or 256 - narrower heads are zero-padded by the caller, `scale` = 1/sqrt(true
 * width).
 * lse: f32 [B][heads][L] (written by fwd, read by bwd); dvec_ws: f32 [B][heads][L] scratch (bwd). */
typedef struct fdx_attn_desc {
  int B, heads, L, Lk, dh;
  float scale;
  const void* q; long long q_ld, q_bs;
  const void* k; long long k_ld, k_bs;
  const void* v; long long v_ld, v_bs;
  void* o; long long o_ld, o_bs;          /* fwd: output; bwd: the saved forward output (input) */
  float* lse;
  /* backward only */
  const void* d_o; long long do_ld, do_bs;
  float* dvec_ws;
  void* dq; long long dq_ld, dq_bs;
  void* dk; long long dk_ld, dk_bs;
  void* dv; long long dv_ld, dv_bs;
} fdx_attn_desc;
int fdx_attention_fwd(const fdx_attn_desc* a, void* stream);
int fdx_attention_bwd(const fdx_attn_desc* a, void* stream);
/* Forward with a key mask, as CLIPTextTransformer's self-attention (transformers' create_causal_mask over
 * `attention_mask`): key j is allowed for query i iff (!causal || j <= i) && key_mask[b][j] != 0.  key_mask is
 * int32 [B][Lk] of 0 / 1, or NULL (every key allowed).  A query row with no allowed key writes zeros (and
 * lse = -inf); the CLIP tokenizer never produces one.  dh 32 or 64 only; dh 128 or 256 gives
 * FDX_ERR_UNSUPPORTED. */
int fdx_attention_fwd_masked(const fdx_attn_desc* a, int causal, const int32_t* key_mask, void* stream);

/* ---- CLIP text tower (fdx_clip.cu): FlaxCLIPTextModel of the text-conditioned trainer ------------------------
 * (flaxdiff/inputs/encoders.py, trainer/general_diffusion_trainer.py:266-275).  Rows are contiguous bf16.
 *   fdx_token_embed   : out[b][t][:] = bf16(tok[ids[b][t]] + pos[t]); ids int32 [B][T], tok f32 [vocab][D],
 *                       pos f32 [>= T][D]; an id outside [0, vocab) gives a NaN row (jnp.take's fill mode) and
 *                       reads nothing.  D a multiple of 8.
 *   fdx_layernorm_fwd : nn.LayerNorm(eps): y = (x - mean) / sqrt(var + eps) * gamma + beta, f32 statistics from
 *                       a two-pass mean / variance.  C a multiple of 8, <= 1280.
 *   fdx_bias_act      : y = act(x + bias) (bias f32 [C] or NULL; x == y allowed).  C a multiple of 8. */
#define FDX_ACT_QUICK_GELU 0 /* z * sigmoid(1.702 z) */
#define FDX_ACT_GELU 1       /* exact erf gelu */
#define FDX_ACT_GELU_TANH 2  /* 0.5 z (1 + tanh(sqrt(2/pi) (z + 0.044715 z^3))): jax.nn.gelu's default (fdx_dit.cu) */
int fdx_token_embed(const int32_t* ids, int B, int T, const float* tok, int vocab, const float* pos, int D,
                    void* out_bf16, void* stream);
int fdx_layernorm_fwd(const void* x_bf16, long long rows, int C, const float* gamma, const float* beta, float eps,
                      void* y_bf16, void* stream);
int fdx_bias_act(const void* x_bf16, long long rows, int C, const float* bias, int act, void* y_bf16, void* stream);

/* ---- CLIP validation metrics (fdx_clip.cu): get_clip_metric / get_clip_score_metric -----------------------------
 * (flaxdiff/metrics/images.py:32-112, training.py:515-525).  The vision tower (transformers modeling_clip.py:640-690)
 * and the text tower run on fdx_gemm, fdx_layernorm_fwd, fdx_attention_fwd[_masked] and fdx_bias_act; these four
 * entry points are the rest.
 *   fdx_clip_image_prep   : images.py:69-70 + AutoProcessor(use_fast=False): x f32 [B][H][W][3] ->
 *                           u8 = ((x + 1) / 2) * 255 in f32, truncated (clamped to [0, 255], NaN -> 0) -> PIL's 8-bit
 *                           two-pass bicubic resize of the crop window only -> lut[c][u8] (x / 255 normalised by the
 *                           processor's mean / std) -> bf16 patches [B*G*G][ld], G = crop / patch, one row per
 *                           patch in the (c, ky, kx) order of the HF conv weight, zero from 3*patch^2 to ld (a
 *                           multiple of 8).  tables: int32 [crop][2 + ksize_y] (output rows) then
 *                           [crop][2 + ksize_x] (output columns), each entry = first source index, tap count, taps
 *                           with 22 fraction bits (PIL's precompute_coeffs + normalize_coeffs_8bpc; a pass PIL skips
 *                           is one tap of 1 << 22).  lut: f32 [3][256].  u8_out: uint8 [B][crop][crop][3] or NULL.
 *   fdx_clip_vision_embed : modeling_clip.py:206-245 + pre_layrnorm: out[b][t] = bf16(LN((t == 0 ? cls :
 *                           patch_f32[b*G2 + t - 1]) + pos[t])) [B][G2 + 1][D], f32 statistics, one rounding.
 *                           D a multiple of 8, <= 1280.
 *   fdx_clip_pool         : out[b] = [LN](x[b][r_b]) bf16 [B][D] from x bf16 [B][T][D]; r_b = 0 when ids is NULL
 *                           (the CLS row, with gamma / beta = post_layernorm), else the first position of the largest
 *                           id of sequence b (FlaxCLIP's argmax(input_ids) EOS rule; ids int32 [B][T]).  gamma / beta
 *                           NULL = no LayerNorm.  D a multiple of 8, <= 1280.
 *   fdx_clip_similarity   : images.py:44-46, 65, 96: cos[b] = <a / (|a| + 1e-6), t / (|t| + 1e-6)> over img / txt f32 [B][P];
 *                           out2 = {mean(1 - cos) (clip_similarity), mean(100 max(cos, 0)) (clip_score)}, f32. */
int fdx_clip_image_prep(const float* x, int B, int H, int W, const int32_t* tables, int ksize_y, int ksize_x,
                        const float* lut, int crop, int patch, int ld, void* patches_bf16, uint8_t* u8_out,
                        void* stream);
int fdx_clip_vision_embed(const float* patch_f32, int B, int G2, int D, const float* cls, const float* pos,
                          const float* gamma, const float* beta, float eps, void* out_bf16, void* stream);
int fdx_clip_pool(const void* x_bf16, int B, int T, int D, const int32_t* ids, const float* gamma, const float* beta,
                  float eps, void* out_bf16, void* stream);
int fdx_clip_similarity(const float* img, const float* txt, int B, int P, float* cos, float* out2, void* stream);

/* ---- SimpleDiT (fdx_dit.cu): flaxdiff/models/simple_dit.py:23-306 ---------------------------------------------------
 * The dense layers run on fdx_gemm and the attention on fdx_attention_fwd / _bwd; these are the streaming passes
 * around them.  Token matrices are bf16 [rows = B * L][C] (row stride C), L tokens per sample; `ada` is the f32
 * [B][ada_ld] output of a block's ada_proj, whose six F-wide chunks a call addresses by column offset.  Column sums run
 * in two ordered stages through ws = f32 [B][nchunk][2][C] (nchunk token chunks per sample): no atomics, the results
 * are reproducible bit for bit.
 *   fdx_dit_adaln_fwd   : y = (xhat * gamma + beta) * (1 + ada[b][scale_off + c]) + ada[b][shift_off + c], xhat the
 *                         LayerNorm of the token (f32 statistics; mean / rstd f32 [rows] written when non-NULL).  A
 *                         NULL ada, gamma or beta drops its term; ada and gamma exclusive.  C a multiple of 8, <= 1536.
 *   fdx_dit_adaln_bwd   : its backward: dx = d/dx (+ addend; dx may alias addend); d0 / d1 (+)= the sums of dy * xhat
 *                         and of dy over each sample's tokens, rows of d0_ld / d1_ld floats (d(scale), d(shift) into
 *                         their chunks of a d_ada buffer) or, reduce_samples, over all rows (d(gamma), d(beta)).
 *   fdx_dit_gate_fwd    : out = x + gate[b][c] * y (the gated residual; gate rows gate_ld floats apart; out may be x).
 *   fdx_dit_gate_bwd    : dy = gate[b][c] * dout and dgate[b][c] = sum over the sample's tokens of dout * y.
 *   fdx_dit_token_mean  : out[b][c] = mean over t of x[b][t][c] (f32 [B][C]); ws as above.
 *   fdx_dit_rope        : RoPE in place on nmat matrices mat_off columns apart in rows of ld elements (q and k of the
 *                         fused QKV output): per dp-wide head, pair (i, i + d/2), i < d/2, rotated by the angle
 *                         (token index in its sample) * 10000^(-2i/d); `inverse` applies the transposed rotation (the
 *                         backward).  Channels [d, dp) of each head are set to zero.  d even.
 *   fdx_bias_act_bwd    : dx = dy * act'(x + bias), act = FDX_ACT_GELU_TANH.
 *   fdx_dit_patchify    : src (B, H, W, C) f32 (src_f32) or bf16 -> dst bf16 [B * (H/p) * (W/p)][ld], row-major
 *                         patches, columns (p1, p2, c), zeros from p*p*C to ld (a multiple of 8).  The patch-embedding
 *                         GEMM's operand, and the transpose of fdx_dit_unpatchify (the final projection's gradient).
 *   fdx_dit_unpatchify  : src f32 [B * L][ld] -> dst f32 (B, H, W, C): 'B (h w) (p1 p2 C) -> B (h p1) (w p2) C'
 *                         (vit_common.py:10-17) over the first p*p*C columns; the transpose of fdx_dit_patchify.
 *   fdx_dit_fourier     : out bf16 [B][2 half] = [sin(t_b 2 pi freqs), cos(t_b 2 pi freqs)] (models/common.py:97-110). */
int fdx_dit_adaln_fwd(const void* x_bf16, long long rows, int L, int C, const float* ada, long long ada_ld,
                      int scale_off, int shift_off, const float* gamma, const float* beta, float eps, void* y_bf16,
                      float* mean, float* rstd, void* stream);
int fdx_dit_adaln_bwd(const void* x_bf16, const void* dy_bf16, long long rows, int L, int C, const float* ada,
                      long long ada_ld, int scale_off, const float* gamma, const float* mean, const float* rstd,
                      const void* addend_bf16, void* dx_bf16, float* ws, int nchunk, float* d0, long long d0_ld,
                      float* d1, long long d1_ld, int reduce_samples, int accumulate, void* stream);
int fdx_dit_gate_fwd(const void* x_bf16, const void* y_bf16, long long rows, int L, int C, const float* gate,
                     long long gate_ld, void* out_bf16, void* stream);
int fdx_dit_gate_bwd(const void* dout_bf16, const void* y_bf16, long long rows, int L, int C, const float* gate,
                     long long gate_ld, void* dy_bf16, float* ws, int nchunk, float* dgate, long long dgate_ld,
                     void* stream);
int fdx_dit_token_mean(const void* x_bf16, int B, int T, int C, float* ws, int nchunk, float* out, void* stream);
int fdx_dit_rope(void* base_bf16, long long rows, int L, long long ld, int heads, int d, int dp, int nmat,
                 long long mat_off, int inverse, void* stream);
int fdx_bias_act_bwd(const void* x_bf16, long long rows, int C, const float* bias, int act, const void* dy_bf16,
                     void* dx_bf16, void* stream);
int fdx_dit_patchify(const void* src, int src_f32, int B, int H, int W, int C, int p, int ld, void* dst_bf16,
                     void* stream);
int fdx_dit_unpatchify(const float* src, int ld, int B, int H, int W, int C, int p, float* dst, void* stream);
int fdx_dit_fourier(const float* t, int B, const float* freqs, int half, void* out_bf16, void* stream);

/* ---- S5 state-space layer (fdx_ssm.cu): flaxdiff/models/ssm_dit.py:58-286, hilbert.py:87-370 -----------------------
 * One S5 layer has ndir (1, or 2 when bidirectional) directions of N complex states over F features.  Its per-token
 * complex values (Bu, the states x, their gradients) are f32 or bf16 rows of 2 * ndir * N columns: direction d owns
 * [2dN, 2dN + 2N), real parts at 2dN + n, imaginary parts at 2dN + N + n.  The dense products run on fdx_gemm.
 *   fdx_ssm_discretize     : ZOH discretisation of one direction (ssm_dit.py:154-169): dt = exp(log_dt),
 *                            A = -exp(log_a_real) + i a_imag, Abar = exp(A dt), Bbar = (Abar - 1) / (A + 1e-8) B.
 *                            Writes wb[f][col0 + n] = Re Bbar[n][f] and wb[f][col0 + N + n] = Im Bbar[n][f] (bf16, rows
 *                            of ldb: both directions' Bu = u Bbar^T as one product), wc = [C_re^T; -C_im^T] bf16 [2N][F]
 *                            (y = Re(C x) = x_cols wc) and adt[col0 + n] = Re(A dt), adt[col0 + N + n] = Im(A dt) / pi.
 *   fdx_ssm_scan           : bu f32 [B * L][2 ndir N] -> states x f32 (x may alias bu), x_k = Abar x_{k-1} + bu_k,
 *                            direction 0 from token 0, direction 1 from token L - 1 (the states sit at their tokens);
 *                            x_bf16 receives a bf16 copy.  x may be NULL: then only the bf16 copy is written (6 instead
 *                            of 10 bytes per state, the inference forward's call, which never runs the adjoint); every
 *                            other pointer is required.  Sequence-parallel over chunks of `chunk` tokens; ws f32
 *                            [B][nchunk][2 ndir N].
 *   fdx_ssm_scan_bwd       : the adjoint lambda_k = dx_k + conj(Abar) lambda_{k+1} (in each direction's step order) from
 *                            dx f32, the saved f32 states x and bu: lambda -> lam_bf16, and per (sample, chunk) partial
 *                            sums of lambda_k conj(x_{k-1}) -> dabar and of lambda_k conj(bu_k) -> dgbar (f32
 *                            [B][nchunk][2 ndir N]).  ws as fdx_ssm_scan's.
 *   fdx_ssm_discretize_bwd : for one direction, from dwb = d(Bbar) f32 rows [col0 + n] (real) / [col0 + N + n] (imag)
 *                            of F, dwc = d(wc) f32 [2N][F] and the nparts rows of dabar / dgbar (ld_part floats apart):
 *                            accumulates (+=) the gradients of log_a_real, a_imag, log_dt, B_re, B_im, C_re and C_im.
 *                            Complex gradients follow d = d/dRe + i d/dIm.  Fixed-order sums, no atomics.
 *   fdx_permute_rows       : dst[b * L + i] = src[b * L + idx[i]] over rows of row_bytes (a multiple of 16): the
 *                            Hilbert / zigzag patch order and its inverse. */
int fdx_ssm_discretize(const float* log_a_real, const float* a_imag, const float* log_dt, const float* b_re,
                       const float* b_im, const float* c_re, const float* c_im, int N, int F, void* wb_bf16, int ldb,
                       int col0, void* wc_bf16, float* adt, void* stream);
int fdx_ssm_discretize_bwd(const float* log_a_real, const float* a_imag, const float* log_dt, const float* b_re,
                           const float* b_im, int N, int F, const float* dwb, int col0, const float* dwc,
                           const float* dabar, const float* dgbar, int nparts, int ld_part, float* g_log_a_real,
                           float* g_a_imag, float* g_log_dt, float* g_b_re, float* g_b_im, float* g_c_re,
                           float* g_c_im, void* stream);
int fdx_ssm_scan(const float* bu, float* x, void* x_bf16, const float* adt, int B, int L, int N, int ndir, int chunk,
                 float* ws, void* stream);
int fdx_ssm_scan_bwd(const float* dx, const float* x, const float* bu, const float* adt, int B, int L, int N, int ndir,
                     int chunk, float* ws, void* lam_bf16, float* dabar, float* dgbar, void* stream);
int fdx_permute_rows(const void* src, void* dst, long long rows, int L, long long row_bytes, const int32_t* idx,
                     void* stream);

/* ---- SimpleMMDiT (flaxdiff/models/simple_mmdit.py:17-331) --------------------------------------------------------
 * The MMDiT block is a parallel block: one LayerNorm of the block input (MMAdaLNZero, :17-90) is modulated twice and
 * both branches are added onto the same residual (MMDiTBlock, :137-158).  Token rows are bf16 [rows = B * L][C],
 * C a multiple of 8, <= 1536 for the LayerNorm pair.  ada is the block's f32 [B][ada_ld] modulation, six C-wide chunks
 * in the reference's split order: scale_mlp 0, shift_mlp 1, gate_mlp 2, scale_attn 3, shift_attn 4, gate_attn 5; the
 * mlp scale and shift enter clipped to [-10, 10], the attention chunks as they are.  d_ada has the same layout.  Column
 * sums run in two ordered stages through ws = f32 [B][nchunk][4][C]: no atomics, reproducible bit for bit.
 *   fdx_mmdit_adaln_fwd : y_attn = xhat (1 + scale_attn) + shift_attn and y_mlp = xhat (1 + clip(scale_mlp)) +
 *                         clip(shift_mlp) from one read of x; mean / rstd f32 [rows] written when non-NULL.
 *   fdx_mmdit_adaln_bwd : dx = d/dx of both (+ addend; dx may alias addend) and the scale_attn, shift_attn,
 *                         scale_mlp, shift_mlp chunks of d_ada (per-sample sums over tokens).  The clip's derivative
 *                         is 1 inside (-10, 10), 0 outside and 1/2 at exactly -10 or 10.
 *   fdx_mmdit_gate_fwd  : out = x + gate_attn y_attn + gate_mlp y_mlp, one rounding (out may be x).
 *   fdx_mmdit_gate_bwd  : dy_attn = gate_attn dout, dy_mlp = gate_mlp dout, and the gate_attn / gate_mlp chunks of
 *                         d_ada = the sample's sums of dout y_attn / dout y_mlp, in one pass over dout. */
int fdx_mmdit_adaln_fwd(const void* x_bf16, long long rows, int L, int C, const float* ada, long long ada_ld,
                        float eps, void* y_attn_bf16, void* y_mlp_bf16, float* mean, float* rstd, void* stream);
int fdx_mmdit_adaln_bwd(const void* x_bf16, const void* dy_attn_bf16, const void* dy_mlp_bf16, long long rows, int L,
                        int C, const float* ada, long long ada_ld, const float* mean, const float* rstd,
                        const void* addend_bf16, void* dx_bf16, float* ws, int nchunk, float* d_ada,
                        long long d_ada_ld, void* stream);
int fdx_mmdit_gate_fwd(const void* x_bf16, const void* y_attn_bf16, const void* y_mlp_bf16, long long rows, int L,
                       int C, const float* ada, long long ada_ld, void* out_bf16, void* stream);
int fdx_mmdit_gate_bwd(const void* dout_bf16, const void* y_attn_bf16, const void* y_mlp_bf16, long long rows, int L,
                       int C, const float* ada, long long ada_ld, void* dy_attn_bf16, void* dy_mlp_bf16, float* ws,
                       int nchunk, float* d_ada, long long d_ada_ld, void* stream);

/* ---- HierarchicalMMDiT (flaxdiff/models/simple_mmdit.py:336-730): affine LayerNorm over rows up to 6144 wide -------
 * A logical row of C columns (C a multiple of 8, <= 6144; f32 statistics, mean / rstd f32 [rows]) is assembled by mode:
 *   0 gather  (PatchMerging, :348-382): row r = coarse patch (b, h, w) of an HPc x WPc grid, columns (p1, p2, c) read
 *             from fine row b (2HPc)(2WPc) + (2h + p1)(2WPc) + 2w + p2 of src0 [.][C/4]; y [rows][C].
 *   1 concat  (the decoder fusion, :693-696): columns [0, C0) from src0 [rows][C0], the rest from src1; y [rows][C].
 *   2 scatter (PatchExpanding, :396-429): src0 [rows][C]; column (p1, p2, c) goes to that fine row of y [.][C/4].
 * The 2x2 modes need C a multiple of 32 and rows a multiple of HPc * WPc.
 *   fdx_layernorm_rows_fwd : y = xhat * gamma + beta.
 *   fdx_layernorm_rows_bwd : dx back through the same assembly into dx0 (gather: the fine rows; concat: the first C0
 *                            columns; scatter: [rows][C]) and, concat, dx1; each destination is overwritten or, with
 *                            its accumulate flag, added to.  dgamma / dbeta (+)= the sums over all rows, formed in
 *                            nchunk row chunks (ws f32 [nchunk][2][C]) and added in chunk order: no atomics. */
int fdx_layernorm_rows_fwd(int mode, const void* src0_bf16, const void* src1_bf16, long long rows, int C, int C0,
                           int HPc, int WPc, const float* gamma, const float* beta, float eps, void* y_bf16,
                           float* mean, float* rstd, void* stream);
int fdx_layernorm_rows_bwd(int mode, const void* src0_bf16, const void* src1_bf16, const void* dy_bf16,
                           long long rows, int C, int C0, int HPc, int WPc, const float* gamma, const float* mean,
                           const float* rstd, void* dx0_bf16, int accumulate0, void* dx1_bf16, int accumulate1,
                           float* ws, int nchunk, float* dgamma, float* dbeta, void* stream);

/* ---- UViT (flaxdiff/models/simple_vit.py:18-250): the sequence assembly and the output head (fdx_uvit.cu) ---------
 * The token stream is bf16 [B * L][F] with L = N + 1 + T (N patches, the time token, T text tokens; F a multiple of 8).
 *   fdx_uvit_assemble_fwd : replaces `x_patches + pos_encoding[:, :N]` and `concat([patches, time, text], 1)`
 *                           (:194-210): row b L + s is bf16(f32(patch[b N + s]) + pos[s]) for s < N (patch bf16
 *                           [B * N][F], pos f32 rows), time[b] for s = N (bf16 [B][F]) and text[b T + s - N - 1]
 *                           (bf16 [B * T][F]; NULL when T = 0).
 *   fdx_uvit_assemble_bwd : splits the stream gradient dx into dpatch (bf16 [B * N][F]), dtime (f32 [B][F]; skipped
 *                           when NULL) and dtext (bf16 [B * T][F]; skipped when NULL), and adds dpos[s] += sum_b dx[b L
 *                           + s] for s < N (f32 [N][F]) in two ordered stages through ws = f32 [nsplit][N][F]: sample
 *                           splits of ceil(B / nsplit), then the partials in split order.  No atomics.
 *   fdx_uvit_head_norm_fwd: final_norm_conv + activation (:240-241): per pixel of x bf16 [pixels][64],
 *                           y = act(LayerNorm(x) gamma + beta), f32 statistics, act 1 = swish, 2 = mish.
 *   fdx_uvit_head_norm_bwd: its backward: dx bf16 and dgamma / dbeta (+)= the sums over pixels, formed in nchunk
 *                           pixel chunks (ws f32 [nchunk][2][64]) and added in chunk order.  No atomics.
 *   fdx_im2col3x3_c6      : final_conv1's operand over concat([src0, src1], -1) (:236-239) without the concat:
 *                           col[p][t*3+k] = bf16(src0[p + d(t)][k]), col[p][32 + t*3+k] = bf16(src1[p + d(t)][k]),
 *                           zero outside the image and in columns 27..31, 59..63; bf16 [N*H*W][64].  Sources are
 *                           dense [N][H][W][3], f32 or bf16 as flagged. */
int fdx_uvit_assemble_fwd(const void* patch_bf16, const float* pos, const void* time_bf16, const void* text_bf16,
                          int B, int N, int T, int F, void* out_bf16, void* stream);
int fdx_uvit_assemble_bwd(const void* dx_bf16, int B, int N, int T, int F, void* dpatch_bf16, float* dtime,
                          void* dtext_bf16, float* ws, int nsplit, float* dpos, void* stream);
int fdx_uvit_head_norm_fwd(const void* x_bf16, long long pixels, const float* gamma, const float* beta, float eps,
                           int act, void* y_bf16, void* stream);
int fdx_uvit_head_norm_bwd(const void* x_bf16, const void* dy_bf16, long long pixels, const float* gamma,
                           const float* beta, float eps, int act, void* dx_bf16, float* ws, int nchunk, float* dgamma,
                           float* dbeta, void* stream);
int fdx_im2col3x3_c6(const void* src0, int src0_is_f32, const void* src1, int src1_is_f32, int N, int H, int W,
                     void* col_bf16, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FDX_H_ */
