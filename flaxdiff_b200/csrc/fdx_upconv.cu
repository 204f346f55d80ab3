// fdx_upconv.cu -- Upsample = nearest-neighbour x2 followed by a 3x3 SAME convolution
// (flaxdiff/models/common.py:210-226: jax.image.resize(..., "nearest") + ConvLayer 3x3), computed
// WITHOUT materialising the 4x larger tensor: the sub-pixel (output-parity) decomposition.
//
// Output pixel (2i+py, 2j+px) reads the upsampled rows 2i+py+ky-1, ky = 0..2, i.e. the LOW-resolution
// rows i + floor((py+ky-1)/2):
//     py = 0 : ky=0 -> i-1 ;  ky=1,2 -> i          py = 1 : ky=0,1 -> i ;  ky=2 -> i+1
// so each of the four output parities is a 2x2 convolution of the low-resolution input whose taps are
// sums of the 3x3 taps that land on the same source pixel:
//     W_eff[py][px][a][b] = sum_{ky in S(py,a)} sum_{kx in S(px,b)} W[ky][kx],   source offset (a-1+py, b-1+px)
// 16 tap-GEMMs on a quarter of the pixels instead of 9 on all of them: 4/9 of the FLOPs (these two layers
// are 27 % of the UNet's forward FLOPs), and the upsampled activation never exists in HBM.  Zero padding
// is unchanged: upsampled row -1 / 2H <-> low-resolution row -1 / H, both outside the tensor (TMA fill).
//
// forward : four launches (one per output parity), 4 taps each, output written with pixel stride 2
// dgrad   : ONE launch with 16 taps: dx_low = sum_{parity, tap} dY[parity view, shifted] * W_eff^T
// wgrad   : ONE split-K launch with 16 taps over the low-resolution pixels; the B operand is the
//           stride-2 parity view of dY; the 16 slabs are then folded back onto the nine 3x3 taps.
#include "fdx_tc.cuh"
#include "../../include/fdx.h"

namespace {

__host__ __device__ inline int up_slot(int parity, int k) {   // which of the two source rows tap k hits
  return parity == 0 ? (k >= 1 ? 1 : 0) : (k == 2 ? 1 : 0);
}

// weff[(py*2+px)*4 + a*2+b][ci][co] (bf16)  <-  w[ky*3+kx][ci][co] (f32 master weights)
__global__ void __launch_bounds__(256)
upconv_pack_kernel(const float* __restrict__ w, long long slab, __nv_bfloat16* __restrict__ weff) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < slab;
       i += (long long)gridDim.x * blockDim.x) {
    float t[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) t[k] = w[k * slab + i];
#pragma unroll
    for (int ph = 0; ph < 4; ++ph) {
      const int py = ph >> 1, px = ph & 1;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) acc[up_slot(py, ky) * 2 + up_slot(px, kx)] += t[ky * 3 + kx];
#pragma unroll
      for (int ab = 0; ab < 4; ++ab) weff[(ph * 4 + ab) * slab + i] = __float2bfloat16(acc[ab]);
    }
  }
}

// dw[ky*3+kx][ci][co] += sum_{py,px} dweff[(py*2+px)*4 + slot(py,ky)*2 + slot(px,kx)][ci][co]
__global__ void __launch_bounds__(256)
upconv_fold_kernel(const float* __restrict__ dweff, long long slab, float* __restrict__ dw) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < slab;
       i += (long long)gridDim.x * blockDim.x) {
    float t[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) t[k] = dweff[k * slab + i];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        float acc = 0.f;
#pragma unroll
        for (int ph = 0; ph < 4; ++ph)
          acc += t[ph * 4 + up_slot(ph >> 1, ky) * 2 + up_slot(ph & 1, kx)];
        dw[(ky * 3 + kx) * slab + i] += acc;
      }
  }
}

void fill_act(TcOperand& o, const fdx_act* a) {
  o.ptr = a->ptr;
  o.dims[0] = a->c; o.dims[1] = a->w; o.dims[2] = a->h; o.dims[3] = a->n;
  o.strides[0] = 1;
  o.strides[1] = a->pix_stride;
  o.strides[2] = a->pix_stride * a->w;
  o.strides[3] = a->pix_stride * a->w * a->h;
}

int check_pair(const fdx_act* lo, const fdx_act* hi, const char* what) {
  FDX_REQUIRE(lo && lo->ptr && hi && hi->ptr, "%s: null tensor", what);
  FDX_REQUIRE(hi->n == lo->n && hi->h == 2 * lo->h && hi->w == 2 * lo->w,
              "%s: the full-resolution tensor must be exactly twice the low-resolution one", what);
  FDX_REQUIRE(lo->c % 64 == 0 && hi->c % 64 == 0, "%s: channels must be multiples of 64", what);
  FDX_REQUIRE(lo->pix_stride >= lo->c && lo->pix_stride % 8 == 0 && hi->pix_stride >= hi->c &&
                  hi->pix_stride % 8 == 0,
              "%s: pix_stride must be >= c and a multiple of 8", what);
  return FDX_OK;
}

}  // namespace

extern "C" {

int fdx_upconv3x3_pack(const float* w_hwio, int cin, int cout, void* weff_bf16, void* stream) {
  FDX_REQUIRE(w_hwio && weff_bf16 && cin > 0 && cout > 0, "upconv3x3_pack: bad arguments");
  const long long slab = (long long)cin * cout;
  long long grid = (slab + 255) / 256;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  upconv_pack_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(w_hwio, slab, (__nv_bfloat16*)weff_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

static int upconv_fwd_impl(const fdx_act* x, const void* weff_bf16, const float* bias, const fdx_act* y,
                           const fdx_colstats* cs, void* stream) {
  int s = check_pair(x, y, "upconv3x3_fwd");
  if (s != FDX_OK) return s;
  FDX_REQUIRE(weff_bf16, "upconv3x3_fwd: null weights");
  if (cs) {
    FDX_REQUIRE(cs->ws && cs->slots > 0 && cs->slots <= 64 && cs->ld >= y->c, "upconv3x3_fwd_stats: bad workspace");
    // the pixels-as-M epilogue adds its sums with 16-byte vector reductions
    FDX_REQUIRE(reinterpret_cast<uintptr_t>(cs->ws) % 16 == 0 && cs->ld % 4 == 0,
                "upconv3x3_fwd_stats: the workspace must be 16-byte aligned and ld=%d a multiple of 4", cs->ld);
    if ((long long)y->h * y->w < 128) {
      fdx_set_error("upconv3x3_fwd_stats: fewer than 128 pixels per image of y (%dx%d)", y->w, y->h);
      return FDX_ERR_UNSUPPORTED;
    }
  }
  const int cin = x->c, cout = y->c;
  for (int ph = 0; ph < 4; ++ph) {
    const int py = ph >> 1, px = ph & 1;
    TcLaunch L{};
    L.mode = TC_KMN;
    fill_act(L.A, x);
    // this parity's four slabs as one MN-major matrix [4*Cin][Cout]
    L.B.ptr = static_cast<const __nv_bfloat16*>(weff_bf16) + (long long)ph * 4 * cin * cout;
    L.B.dims[0] = cout; L.B.dims[1] = 4ull * cin; L.B.dims[2] = 1; L.B.dims[3] = 1;
    L.B.strides[0] = 1; L.B.strides[1] = cout; L.B.strides[2] = 4ull * cin * cout;
    L.B.strides[3] = L.B.strides[2];
    L.W = x->w; L.H = x->h; L.N = x->n;
    L.es = 1;
    L.ntaps = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int t = a * 2 + b;
        L.tap_dx[t] = b - 1 + px;
        L.tap_dy[t] = a - 1 + py;
        L.tap_b[t] = t * cin;
      }
    L.K = cin;
    L.Ncols = cout;
    L.out = static_cast<__nv_bfloat16*>(y->ptr) + ((long long)py * y->w + px) * y->pix_stride;
    L.os_x = 2 * y->pix_stride; L.os_y = 2 * y->pix_stride * y->w; L.os_n = y->pix_stride * y->w * y->h;
    L.alpha = 1.f;
    L.bias = bias;
    if (cs) {   // the four parities add their quarter of the pixels to the same sums
      L.gn_ws = cs->ws;
      L.gn_slots = cs->slots;
      L.ws_ld = cs->ld;
    }
    s = fdx_tc_launch(L, (cudaStream_t)stream);
    if (s != FDX_OK) return s;
  }
  return FDX_OK;
}

int fdx_upconv3x3_fwd(const fdx_act* x, const void* weff_bf16, const float* bias, const fdx_act* y,
                      void* stream) {
  return upconv_fwd_impl(x, weff_bf16, bias, y, nullptr, stream);
}

int fdx_upconv3x3_fwd_stats(const fdx_act* x, const void* weff_bf16, const float* bias, const fdx_act* y,
                            const fdx_colstats* cs, void* stream) {
  FDX_REQUIRE(cs, "upconv3x3_fwd_stats: null statistics descriptor");
  return upconv_fwd_impl(x, weff_bf16, bias, y, cs, stream);
}

int fdx_upconv3x3_dgrad(const fdx_act* dy, const void* weff_bf16, const fdx_act* dx, int accumulate,
                        void* stream) {
  int s = check_pair(dx, dy, "upconv3x3_dgrad");
  if (s != FDX_OK) return s;
  FDX_REQUIRE(weff_bf16, "upconv3x3_dgrad: null weights");
  const int cin = dx->c, cout = dy->c;
  TcLaunch L{};
  L.mode = TC_KK;
  fill_act(L.A, dy);
  // W_eff viewed as (k = Cout contiguous, n = Cin rows, z1 = 16 slabs)
  L.B.ptr = weff_bf16;
  L.B.dims[0] = cout; L.B.dims[1] = cin; L.B.dims[2] = 16; L.B.dims[3] = 1;
  L.B.strides[0] = 1; L.B.strides[1] = cout; L.B.strides[2] = (uint64_t)cin * cout;
  L.B.strides[3] = 16ull * cin * cout;
  L.W = dx->w; L.H = dx->h; L.N = dx->n;
  L.es = 2;                                   // A (dY) is read at every other pixel
  L.ntaps = 16;
  // forward: y[2i+py][2j+px] += x[i+oy][j+ox] W_eff[ph][a][b], (oy, ox) = (a-1+py, b-1+px)
  // => dx[i][j] += dY[2(i-oy)+py][2(j-ox)+px] W_eff[ph][a][b]^T : A offset = parity - 2*offset
  for (int ph = 0; ph < 4; ++ph)
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int py = ph >> 1, px = ph & 1, t = ph * 4 + a * 2 + b;
        L.tap_dx[t] = px - 2 * (b - 1 + px);
        L.tap_dy[t] = py - 2 * (a - 1 + py);
        L.tap_b[t] = t;
      }
  L.K = cout;
  L.Ncols = cin;
  L.alpha = 1.f;
  L.out = dx->ptr;
  L.os_x = dx->pix_stride; L.os_y = dx->pix_stride * dx->w; L.os_n = dx->pix_stride * dx->w * dx->h;
  if (accumulate) { L.res = dx->ptr; L.rs_x = L.os_x; L.rs_y = L.os_y; L.rs_n = L.os_n; }
  return fdx_tc_launch(L, (cudaStream_t)stream);
}

int fdx_upconv3x3_wgrad(const fdx_act* x, const fdx_act* dy, float* dweff_ws, float* dw_hwio,
                        void* stream) {
  int s = check_pair(x, dy, "upconv3x3_wgrad");
  if (s != FDX_OK) return s;
  FDX_REQUIRE(dweff_ws && dw_hwio, "upconv3x3_wgrad: null pointer");
  const int cin = x->c, cout = dy->c;
  cudaStream_t st = (cudaStream_t)stream;
  const long long slab = (long long)cin * cout;
  FDX_CUDA(cudaMemsetAsync(dweff_ws, 0, sizeof(float) * 16 * slab, st));
  TcLaunch L{};
  L.mode = TC_MNMN;
  fill_act(L.A, x);
  fill_act(L.B, dy);
  L.W = x->w; L.H = x->h; L.N = x->n;        // reduction runs over the LOW-resolution pixels
  L.es = 1;
  L.es_b = 2;
  L.ntaps = 16;
  for (int ph = 0; ph < 4; ++ph)
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int py = ph >> 1, px = ph & 1, t = ph * 4 + a * 2 + b;
        L.tap_dx[t] = b - 1 + px;
        L.tap_dy[t] = a - 1 + py;
        L.tap_bdx[t] = px;
        L.tap_bdy[t] = py;
        L.tap_b[t] = t;
      }
  L.M = cin;
  L.Ncols = cout;
  L.out = dweff_ws;
  L.out_f32 = 1;
  L.out_atomic = 1;
  L.os_tap = slab;
  L.os_m = cout;
  L.alpha = 1.f;
  s = fdx_tc_launch(L, st);
  if (s != FDX_OK) return s;
  long long grid = (slab + 255) / 256;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  upconv_fold_kernel<<<(int)grid, 256, 0, st>>>(dweff_ws, slab, dw_hwio);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
