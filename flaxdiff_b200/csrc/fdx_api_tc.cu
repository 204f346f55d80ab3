// fdx_api_tc.cu -- C-ABI entry points built on the wgmma tap-GEMM engine:
// conv3x3 (fwd / dgrad / wgrad, stride 1 and 2), conv1x1 / dense / batched GEMM.
//
// Reference interfaces replaced (all lowered by XLA in the reference):
//   flax.linen.Conv via ConvLayer            flaxdiff/models/common.py:166-172
//   Downsample 3x3 stride-2 SAME (pad 0,1)   flaxdiff/models/common.py:237-244
//   residual 1x1 conv                        flaxdiff/models/common.py:324-333
//   nn.DenseGeneral q/k/v/out projections    flaxdiff/models/attention.py:132-154
//   nn.dot_product_attention contractions    flaxdiff/models/attention.py:170-174
#include "fdx_tc.cuh"
#include "../../include/fdx.h"

namespace {

void fill_act_operand(TcOperand& o, const fdx_act* a) {
  o.ptr = a->ptr;
  o.dims[0] = a->c; o.dims[1] = a->w; o.dims[2] = a->h; o.dims[3] = a->n;
  o.strides[0] = 1;
  o.strides[1] = a->pix_stride;
  o.strides[2] = a->pix_stride * a->w;
  o.strides[3] = a->pix_stride * a->w * a->h;
}

int check_act(const fdx_act* a, const char* name) {
  FDX_REQUIRE(a && a->ptr, "%s: null tensor", name);
  FDX_REQUIRE(a->n > 0 && a->h > 0 && a->w > 0 && a->c > 0, "%s: bad dims", name);
  FDX_REQUIRE(a->pix_stride >= a->c && a->pix_stride % 8 == 0,
              "%s: pix_stride=%lld must be >= c and a multiple of 8", name, a->pix_stride);
  return FDX_OK;
}

}  // namespace

extern "C" {

static int conv3x3_fwd_impl(const fdx_act* x, const void* w_hwio, const float* bias, const float* rowvec,
                            const fdx_act* res, const fdx_act* y, int stride, const fdx_colstats* cs,
                            void* stream) {
  int s;
  if ((s = check_act(x, "conv3x3_fwd x")) != FDX_OK) return s;
  if ((s = check_act(y, "conv3x3_fwd y")) != FDX_OK) return s;
  FDX_REQUIRE(stride == 1 || stride == 2, "conv3x3_fwd: stride must be 1 or 2");
  FDX_REQUIRE(x->c % 64 == 0 && y->c % 64 == 0, "conv3x3_fwd: channels must be multiples of 64");
  FDX_REQUIRE(y->n == x->n && y->h == (x->h + stride - 1) / stride &&
                  y->w == (x->w + stride - 1) / stride,
              "conv3x3_fwd: output dims do not match SAME padding");
  TcLaunch L{};
  L.mode = TC_KMN;
  fill_act_operand(L.A, x);
  L.B.ptr = w_hwio;   // HWIO [9*Cin][Cout], Cout contiguous -> MN-major B
  L.B.dims[0] = y->c; L.B.dims[1] = 9ull * x->c; L.B.dims[2] = 1; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = y->c; L.B.strides[2] = 9ull * x->c * y->c;
  L.B.strides[3] = L.B.strides[2];
  L.W = y->w; L.H = y->h; L.N = y->n;
  L.es = stride;
  L.ntaps = 9;
  // jax/flax SAME: stride 1 pads (1,1); stride 2 on even sizes pads (0,1)
  const int pad_lo = (stride == 1) ? 1 : ((x->h % 2 == 0) ? 0 : 1);
  const int pad_lo_w = (stride == 1) ? 1 : ((x->w % 2 == 0) ? 0 : 1);
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      L.tap_dx[t] = kx - pad_lo_w;
      L.tap_dy[t] = ky - pad_lo;
      L.tap_b[t] = t * x->c;
    }
  L.K = x->c;
  L.Ncols = y->c;
  L.out = y->ptr;
  L.os_x = y->pix_stride; L.os_y = y->pix_stride * y->w; L.os_n = y->pix_stride * y->w * y->h;
  L.alpha = 1.f;
  L.bias = bias;
  L.rowvec = rowvec;
  if (res) {
    if ((s = check_act(res, "conv3x3_fwd res")) != FDX_OK) return s;
    FDX_REQUIRE(res->n == y->n && res->h == y->h && res->w == y->w && res->c == y->c,
                "conv3x3_fwd: residual shape mismatch");
    L.res = res->ptr;
    L.rs_x = res->pix_stride; L.rs_y = res->pix_stride * res->w;
    L.rs_n = res->pix_stride * res->w * res->h;
  }
  if (cs) {
    FDX_REQUIRE(cs->ws && cs->slots > 0 && cs->slots <= 64 && cs->ld >= y->c, "conv3x3_fwd_stats: bad workspace");
    L.gn_ws = cs->ws;
    L.gn_slots = cs->slots;
    L.ws_ld = cs->ld;
  }
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

int fdx_conv3x3_fwd(const fdx_act* x, const void* w_hwio, const float* bias, const float* rowvec,
                    const fdx_act* res, const fdx_act* y, int stride, void* stream) {
  return conv3x3_fwd_impl(x, w_hwio, bias, rowvec, res, y, stride, nullptr, stream);
}

int fdx_conv3x3_fwd_stats(const fdx_act* x, const void* w_hwio, const float* bias, const float* rowvec,
                          const fdx_act* res, const fdx_act* y, int stride, const fdx_colstats* cs,
                          void* stream) {
  FDX_REQUIRE(cs, "conv3x3_fwd_stats: null statistics descriptor");
  return conv3x3_fwd_impl(x, w_hwio, bias, rowvec, res, y, stride, cs, stream);
}


int fdx_conv3x3_dgrad(const fdx_act* dy, const void* w_hwio, const fdx_act* dx, int stride,
                      int accumulate, void* stream) {
  int s;
  if ((s = check_act(dy, "conv3x3_dgrad dy")) != FDX_OK) return s;
  if ((s = check_act(dx, "conv3x3_dgrad dx")) != FDX_OK) return s;
  FDX_REQUIRE(stride == 1 || stride == 2, "conv3x3_dgrad: stride must be 1 or 2");
  FDX_REQUIRE(dx->c % 64 == 0 && dy->c % 64 == 0, "conv3x3_dgrad: channels must be multiples of 64");
  const int cin = dx->c, cout = dy->c;
  TcLaunch L{};
  L.mode = TC_KK;
  fill_act_operand(L.A, dy);
  // HWIO viewed as (k = Cout contiguous, n = Cin rows, z1 = tap)
  L.B.ptr = w_hwio;
  L.B.dims[0] = cout; L.B.dims[1] = cin; L.B.dims[2] = 9; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = cout; L.B.strides[2] = (uint64_t)cin * cout;
  L.B.strides[3] = 9ull * cin * cout;
  L.N = dx->n;
  L.es = 1;
  L.K = cout;
  L.Ncols = cin;
  L.alpha = 1.f;
  if (stride == 1) {
    FDX_REQUIRE(dx->n == dy->n && dx->h == dy->h && dx->w == dy->w, "conv3x3_dgrad: dims mismatch");
    L.W = dx->w; L.H = dx->h;
    L.ntaps = 9;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const int t = ky * 3 + kx;
        L.tap_dx[t] = kx - 1;
        L.tap_dy[t] = ky - 1;
        L.tap_b[t] = 8 - t;   // flipped tap
      }
    L.out = dx->ptr;
    L.os_x = dx->pix_stride; L.os_y = dx->pix_stride * dx->w; L.os_n = dx->pix_stride * dx->w * dx->h;
    if (accumulate) { L.res = dx->ptr; L.rs_x = L.os_x; L.rs_y = L.os_y; L.rs_n = L.os_n; }
    return fdx_tc_launch(L, (cudaStream_t)stream);
  }
  // stride 2 (forward: iy = 2*oy + ky, pad (0,1)).  Four output parities; parity p receives
  // taps k == p (mod 2) with source offset (p - k) / 2.
  FDX_REQUIRE(dx->h == 2 * dy->h && dx->w == 2 * dy->w && dx->n == dy->n,
              "conv3x3_dgrad: stride-2 needs even input dims");
  L.W = dy->w; L.H = dy->h;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {
      int nt = 0;
      for (int ky = py; ky < 3; ky += 2)
        for (int kx = px; kx < 3; kx += 2) {
          L.tap_dx[nt] = (px - kx) / 2;
          L.tap_dy[nt] = (py - ky) / 2;
          L.tap_b[nt] = ky * 3 + kx;
          ++nt;
        }
      L.ntaps = nt;
      __nv_bfloat16* base =
          static_cast<__nv_bfloat16*>(dx->ptr) + ((long long)py * dx->w + px) * dx->pix_stride;
      L.out = base;
      L.os_x = 2 * dx->pix_stride; L.os_y = 2 * dx->pix_stride * dx->w;
      L.os_n = dx->pix_stride * dx->w * dx->h;
      if (accumulate) { L.res = base; L.rs_x = L.os_x; L.rs_y = L.os_y; L.rs_n = L.os_n; }
      int r = fdx_tc_launch(L, (cudaStream_t)stream);
      if (r != FDX_OK) return r;
    }
  return FDX_OK;
}

int fdx_conv3x3_dgrad_gn(const fdx_act* dy, const void* w_hwio, const fdx_act* dz, const fdx_act* x,
                         const float* ab, float* ws_slots, int slots, void* stream) {
  return fdx_conv3x3_dgrad_gn_act(dy, w_hwio, dz, x, ab, ws_slots, slots, 1, stream);
}

int fdx_conv3x3_dgrad_gn_act(const fdx_act* dy, const void* w_hwio, const fdx_act* dz, const fdx_act* x,
                             const float* ab, float* ws_slots, int slots, int act, void* stream) {
  int s;
  FDX_REQUIRE(act == 1 || act == 2, "conv3x3_dgrad_gn: act=%d (1 = silu, 2 = mish)", act);
  if ((s = check_act(dy, "conv3x3_dgrad_gn dy")) != FDX_OK) return s;
  if ((s = check_act(dz, "conv3x3_dgrad_gn dz")) != FDX_OK) return s;
  if ((s = check_act(x, "conv3x3_dgrad_gn x")) != FDX_OK) return s;
  FDX_REQUIRE(ab && ws_slots && slots > 0 && slots <= 64, "conv3x3_dgrad_gn: bad workspace");
  FDX_REQUIRE(dz->c % 64 == 0 && dy->c % 64 == 0, "conv3x3_dgrad_gn: channels must be multiples of 64");
  FDX_REQUIRE(dz->n == dy->n && dz->h == dy->h && dz->w == dy->w && x->n == dz->n && x->h == dz->h &&
                  x->w == dz->w && x->c == dz->c,
              "conv3x3_dgrad_gn: dims mismatch");
  if ((long long)dz->h * dz->w < 128) {
    fdx_set_error("conv3x3_dgrad_gn: fewer than 128 pixels per image");
    return FDX_ERR_UNSUPPORTED;
  }
  const int cin = dz->c, cout = dy->c;
  FDX_CUDA(cudaMemsetAsync(ws_slots, 0, sizeof(float) * 2 * (size_t)slots * dz->n * cin, (cudaStream_t)stream));
  TcLaunch L{};
  L.mode = TC_KK;
  fill_act_operand(L.A, dy);
  L.B.ptr = w_hwio;
  L.B.dims[0] = cout; L.B.dims[1] = cin; L.B.dims[2] = 9; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = cout; L.B.strides[2] = (uint64_t)cin * cout;
  L.B.strides[3] = 9ull * cin * cout;
  L.N = dz->n; L.W = dz->w; L.H = dz->h;
  L.es = 1;
  L.K = cout;
  L.Ncols = cin;
  L.alpha = 1.f;
  L.ntaps = 9;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      L.tap_dx[t] = kx - 1;
      L.tap_dy[t] = ky - 1;
      L.tap_b[t] = 8 - t;   // flipped tap
    }
  L.out = dz->ptr;
  L.os_x = dz->pix_stride; L.os_y = dz->pix_stride * dz->w; L.os_n = dz->pix_stride * dz->w * dz->h;
  L.res = x->ptr;
  L.rs_x = x->pix_stride; L.rs_y = x->pix_stride * x->w; L.rs_n = x->pix_stride * x->w * x->h;
  L.gn_ab = ab;
  L.gn_ws = ws_slots;
  L.gn_slots = slots;
  if (act == 1) return fdx_tc_launch(L, (cudaStream_t)stream);
  // mish: the transposed engine's epilogue only (the pixels-as-M engine has no mish variant)
  L.gn_mish = 1;
  s = fdx_tct_launch(L, (cudaStream_t)stream);
  if (s == FDX_ERR_UNSUPPORTED)
    fdx_set_error("conv3x3_dgrad_gn: mish is fused on the transposed engine only (Cin = 64 .. 512 not a multiple "
                  "of 256, images 16-aligned); use fdx_conv3x3_dgrad + fdx_groupnorm_bwd with act = 2");
  return s;
}

int fdx_conv3x3_wgrad(const fdx_act* x, const fdx_act* dy, float* dw_hwio, int stride,
                      void* stream) {
  int s;
  if ((s = check_act(x, "conv3x3_wgrad x")) != FDX_OK) return s;
  if ((s = check_act(dy, "conv3x3_wgrad dy")) != FDX_OK) return s;
  FDX_REQUIRE(stride == 1 || stride == 2, "conv3x3_wgrad: stride must be 1 or 2");
  FDX_REQUIRE(x->c % 64 == 0 && dy->c % 64 == 0, "conv3x3_wgrad: channels must be multiples of 64");
  if (stride == 1) {
    const int r = fdx_wgrad9_launch(x, dy, dw_hwio, (cudaStream_t)stream);
    if (r != FDX_ERR_UNSUPPORTED) return r;
  }
  TcLaunch L{};
  L.mode = TC_MNMN;
  fill_act_operand(L.A, x);
  fill_act_operand(L.B, dy);
  L.W = dy->w; L.H = dy->h; L.N = dy->n;
  L.es = stride;
  L.ntaps = 9;
  const int pad_lo = (stride == 1) ? 1 : ((x->h % 2 == 0) ? 0 : 1);
  const int pad_lo_w = (stride == 1) ? 1 : ((x->w % 2 == 0) ? 0 : 1);
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int t = ky * 3 + kx;
      L.tap_dx[t] = kx - pad_lo_w;
      L.tap_dy[t] = ky - pad_lo;
      L.tap_b[t] = t;
    }
  L.M = x->c;
  L.Ncols = dy->c;
  L.out = dw_hwio;
  L.out_f32 = 1;
  L.out_atomic = 1;
  L.os_tap = (long long)x->c * dy->c;
  L.os_m = dy->c;
  L.alpha = 1.f;
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

// 1x1 convolution (the ResidualBlock's residual_conv, common.py:324-333) in CONVOLUTION geometry - one tap, no
// shift - instead of as a flat GEMM: the launch is then eligible for the transposed engine (fdx_tct.cu, 256
// pixels as N), which matters because these layers have few output columns and only K = Cin (forward) or
// K = Cout (data gradient) = one or two 64-deep chunks, i.e. they are epilogue / bandwidth bound.
int fdx_conv1x1_fwd(const fdx_act* x, const void* w_io, const float* bias, const fdx_act* res, const fdx_act* y,
                    void* stream) {
  int s;
  if ((s = check_act(x, "conv1x1_fwd x")) != FDX_OK) return s;
  if ((s = check_act(y, "conv1x1_fwd y")) != FDX_OK) return s;
  FDX_REQUIRE(x->c % 64 == 0 && y->c % 64 == 0, "conv1x1_fwd: channels must be multiples of 64");
  FDX_REQUIRE(y->n == x->n && y->h == x->h && y->w == x->w, "conv1x1_fwd: dims mismatch");
  TcLaunch L{};
  L.mode = TC_KMN;
  fill_act_operand(L.A, x);
  L.B.ptr = w_io;      // [Cin][Cout], Cout contiguous -> MN-major B
  L.B.dims[0] = y->c; L.B.dims[1] = x->c; L.B.dims[2] = 1; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = y->c; L.B.strides[2] = (uint64_t)x->c * y->c; L.B.strides[3] = L.B.strides[2];
  L.W = y->w; L.H = y->h; L.N = y->n;
  L.es = 1; L.ntaps = 1;
  L.tap_dx[0] = 0; L.tap_dy[0] = 0; L.tap_b[0] = 0;
  L.K = x->c; L.Ncols = y->c;
  L.out = y->ptr;
  L.os_x = y->pix_stride; L.os_y = y->pix_stride * y->w; L.os_n = y->pix_stride * y->w * y->h;
  L.alpha = 1.f; L.bias = bias;
  if (res) {
    if ((s = check_act(res, "conv1x1_fwd res")) != FDX_OK) return s;
    L.res = res->ptr;
    L.rs_x = res->pix_stride; L.rs_y = res->pix_stride * res->w; L.rs_n = res->pix_stride * res->w * res->h;
  }
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

int fdx_conv1x1_dgrad(const fdx_act* dy, const void* w_io, const fdx_act* dx, int accumulate, void* stream) {
  int s;
  if ((s = check_act(dy, "conv1x1_dgrad dy")) != FDX_OK) return s;
  if ((s = check_act(dx, "conv1x1_dgrad dx")) != FDX_OK) return s;
  FDX_REQUIRE(dx->c % 64 == 0 && dy->c % 64 == 0, "conv1x1_dgrad: channels must be multiples of 64");
  FDX_REQUIRE(dx->n == dy->n && dx->h == dy->h && dx->w == dy->w, "conv1x1_dgrad: dims mismatch");
  const int cin = dx->c, cout = dy->c;
  TcLaunch L{};
  L.mode = TC_KK;
  fill_act_operand(L.A, dy);
  L.B.ptr = w_io;      // [Cin][Cout] viewed as (k = Cout contiguous, n = Cin rows)
  L.B.dims[0] = cout; L.B.dims[1] = cin; L.B.dims[2] = 1; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = cout; L.B.strides[2] = (uint64_t)cin * cout; L.B.strides[3] = L.B.strides[2];
  L.W = dx->w; L.H = dx->h; L.N = dx->n;
  L.es = 1; L.ntaps = 1;
  L.tap_dx[0] = 0; L.tap_dy[0] = 0; L.tap_b[0] = 0;
  L.K = cout; L.Ncols = cin;
  L.alpha = 1.f;
  L.out = dx->ptr;
  L.os_x = dx->pix_stride; L.os_y = dx->pix_stride * dx->w; L.os_n = dx->pix_stride * dx->w * dx->h;
  if (accumulate) { L.res = dx->ptr; L.rs_x = L.os_x; L.rs_y = L.os_y; L.rs_n = L.os_n; }
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

// fdx_gemm's launch descriptor for g (checked), shared with fdx_gemm_cat
static int gemm_launch_desc(const fdx_gemm_desc* g, TcLaunch& L) {
  FDX_REQUIRE(g && g->A && g->B && g->D, "gemm: null pointer");
  FDX_REQUIRE(g->mode >= 0 && g->mode <= 2, "gemm: bad mode");
  FDX_REQUIRE(g->M > 0 && g->N > 0 && g->K > 0, "gemm: bad dims");
  FDX_REQUIRE(g->N % 32 == 0, "gemm: N=%d must be a multiple of 32", g->N);
  const int b1 = g->batch1 > 0 ? g->batch1 : 1, b2 = g->batch2 > 0 ? g->batch2 : 1;
  L.mode = g->mode;
  L.gemm_like = 1;
  L.es = 1;
  L.ntaps = 1;
  L.alpha = g->alpha;
  L.bias = g->bias;
  L.out = g->D;
  L.out_f32 = g->d_f32;
  L.out_atomic = g->d_atomic;
  L.Ncols = g->N;
  const bool batched = (b1 * b2) > 1;
  if (g->mode == FDX_GEMM_KK || g->mode == FDX_GEMM_KMN) {
    // A[m][k] (k contiguous)
    L.A.ptr = g->A;
    L.A.dims[0] = g->K; L.A.dims[1] = g->M; L.A.dims[2] = b1; L.A.dims[3] = b2;
    L.A.strides[0] = 1; L.A.strides[1] = g->a_ld;
    L.A.strides[2] = g->a_s1 ? g->a_s1 : (long long)g->a_ld * g->M;
    L.A.strides[3] = g->a_s2 ? g->a_s2 : (long long)L.A.strides[2] * b1;
    L.B.ptr = g->B;
    if (g->mode == FDX_GEMM_KK) {   // B[n][k]
      L.B.dims[0] = g->K; L.B.dims[1] = g->N;
    } else {                        // B[k][n]
      L.B.dims[0] = g->N; L.B.dims[1] = g->K;
    }
    L.B.dims[2] = b1; L.B.dims[3] = b2;
    L.B.strides[0] = 1; L.B.strides[1] = g->b_ld;
    L.B.strides[2] = g->b_s1 ? g->b_s1 : (long long)g->b_ld * L.B.dims[1];
    L.B.strides[3] = g->b_s2 ? g->b_s2 : (long long)L.B.strides[2] * b1;
    L.b_batched = (g->b_s1 != 0 || g->b_s2 != 0) && batched;
    if (!L.b_batched) { L.B.dims[2] = 1; L.B.dims[3] = 1; }
    L.W = g->M; L.H = b1; L.N = b2;
    L.K = g->K;
    L.tap_dx[0] = 0; L.tap_dy[0] = 0; L.tap_b[0] = 0;
    L.os_x = g->d_ld; L.os_y = g->d_s1; L.os_n = g->d_s2;
    if (g->res) { L.res = g->res; L.rs_x = g->r_ld; L.rs_y = g->r_s1; L.rs_n = g->r_s2; }
  } else {
    // A[k][m] (m contiguous), B[k][n] (n contiguous); reduce over k rows
    L.A.ptr = g->A;
    L.A.dims[0] = g->M; L.A.dims[1] = g->K; L.A.dims[2] = b1; L.A.dims[3] = b2;
    L.A.strides[0] = 1; L.A.strides[1] = g->a_ld;
    L.A.strides[2] = g->a_s1 ? g->a_s1 : (long long)g->a_ld * g->K;
    L.A.strides[3] = g->a_s2 ? g->a_s2 : (long long)L.A.strides[2] * b1;
    L.B.ptr = g->B;
    L.B.dims[0] = g->N; L.B.dims[1] = g->K; L.B.dims[2] = b1; L.B.dims[3] = b2;
    L.B.strides[0] = 1; L.B.strides[1] = g->b_ld;
    L.B.strides[2] = g->b_s1 ? g->b_s1 : (long long)g->b_ld * g->K;
    L.B.strides[3] = g->b_s2 ? g->b_s2 : (long long)L.B.strides[2] * b1;
    L.W = g->K; L.H = b1; L.N = b2;
    L.M = g->M;
    L.mn_batched = g->reduce_batch ? 0 : 1;
    L.tap_dx[0] = 0; L.tap_dy[0] = 0; L.tap_b[0] = 0;
    L.os_tap = 0; L.os_m = g->d_ld; L.os_y = g->d_s1; L.os_n = g->d_s2;
    L.splits = (g->reduce_batch && g->d_atomic) ? 0 : 1;
    FDX_REQUIRE(!g->res, "gemm: residual unsupported in MNMN mode");
  }
  return FDX_OK;
}

int fdx_gemm(const fdx_gemm_desc* g, void* stream) {
  TcLaunch L{};
  const int s = gemm_launch_desc(g, L);
  if (s != FDX_OK) return s;
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

int fdx_gemm_cat(const fdx_gemm_desc* g, const void* A1, long long a1_ld, int K0, void* stream) {
  FDX_REQUIRE(g && g->A && A1 && g->B && g->D, "gemm_cat: null pointer");
  FDX_REQUIRE(g->mode == FDX_GEMM_KK || g->mode == FDX_GEMM_KMN,
              "gemm_cat: mode %d: a two-source A exists in the KK and KMN modes only", g->mode);
  FDX_REQUIRE(g->batch1 <= 1 && g->batch2 <= 1, "gemm_cat: batch %d x %d: flat row matrices only (batch 1)",
              g->batch1, g->batch2);
  FDX_REQUIRE(K0 > 0 && K0 < g->K && K0 % 64 == 0,
              "gemm_cat: K0=%d must be a multiple of 64 with 0 < K0 < K=%d", K0, g->K);
  FDX_REQUIRE(reinterpret_cast<uintptr_t>(g->A) % 16 == 0 && reinterpret_cast<uintptr_t>(A1) % 16 == 0,
              "gemm_cat: A0 and A1 must be 16-byte aligned");
  FDX_REQUIRE(g->a_ld >= K0 && g->a_ld % 8 == 0, "gemm_cat: a_ld=%lld must be >= K0 and a multiple of 8", g->a_ld);
  FDX_REQUIRE(a1_ld >= g->K - K0 && a1_ld % 8 == 0, "gemm_cat: a1_ld=%lld must be >= K - K0 and a multiple of 8",
              a1_ld);
  TcLaunch L{};
  const int s = gemm_launch_desc(g, L);
  if (s != FDX_OK) return s;
  L.A.dims[0] = K0;
  L.A1.ptr = A1;
  L.A1.dims[0] = g->K - K0; L.A1.dims[1] = g->M; L.A1.dims[2] = 1; L.A1.dims[3] = 1;
  L.A1.strides[0] = 1; L.A1.strides[1] = a1_ld;
  L.A1.strides[2] = L.A1.strides[3] = (uint64_t)a1_ld * g->M;
  L.cat_k0 = K0;
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

}  // extern "C"
