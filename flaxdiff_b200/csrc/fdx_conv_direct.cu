// fdx_conv_direct.cu -- the two 3-channel 3x3 convolutions of the UNet on CUDA cores.
//
//   conv_in   Cin=3  -> 64   flaxdiff/models/simple_unet.py:47-54   (K = 27: too thin for an MMA tile)
//   conv_out  64 -> Cout=3   flaxdiff/models/simple_unet.py:212-221 (N = 3)
// Both are HBM-bound (0.23 GFLOP/img at 256^2 against 17 MB/img of activation traffic), so
// they run as direct convolutions: weights in shared memory, one 16-byte channel vector
// per thread, f32 accumulation. Forward and all gradients.
#include "fdx_common.cuh"
#include "../../include/fdx.h"

namespace {

// ---- conv_in forward: x bf16 [N,H,W,3] dense, w f32 [9][3][Cout], y bf16 act ------------
__global__ void __launch_bounds__(256)
cin3_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                const float* __restrict__ bias, int N, int H, int W, int Cout,
                __nv_bfloat16* __restrict__ y, long long yps) {
  extern __shared__ float sw[];   // [27][Cout] + [Cout]
  for (int i = threadIdx.x; i < 27 * Cout; i += blockDim.x) sw[i] = w[i];
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sw[27 * Cout + i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int vpp = Cout >> 3;
  const long long total = (long long)N * H * W * vpp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vpp);
    long long p = i / vpp;
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    const int n = (int)(p / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = sw[27 * Cout + cv * 8 + j];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = py + ky - 1;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = px + kx - 1;
        if (ix < 0 || ix >= W) continue;
        const __nv_bfloat16* xp = x + ((long long)(n * H + iy) * W + ix) * 3;
        const float v0 = __bfloat162float(xp[0]), v1 = __bfloat162float(xp[1]),
                    v2 = __bfloat162float(xp[2]);
        const float* wp = sw + ((ky * 3 + kx) * 3) * Cout + cv * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          acc[j] += v0 * wp[j] + v1 * wp[Cout + j] + v2 * wp[2 * Cout + j];
      }
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(y + p * yps + cv * 8) = o;
  }
}

// ---- shared weight-gradient kernel of the two 3-channel convolutions ----------------------
// out[j][c] += sum_p small_j(p) * wide[p][c],  j = (tap t, k in 0..2), c in 0..63, where
//   small_j(p) = S[p + SGN*d(t)][k]  (zero outside the image).
//   conv_in :  wide = dY (bf16, 64 ch), S = x_in (bf16, 3 ch), SGN=+1, out = dW[(t*3+k)*64 + c]
//   conv_out:  wide = x  (bf16, 64 ch), S = dF   (f32, 3 ch),  SGN=-1, out = dW[(t*64+c)*3 + k]
// Block = 4 pixel lanes x 64 channels; every thread keeps 27 accumulators; wide is read once,
// fully coalesced; the 27 scalars are warp-broadcast loads that hit L1.
template <bool SMALL_F32, int SGN>
__global__ void __launch_bounds__(256)
rank27_wgrad_kernel(const __nv_bfloat16* __restrict__ wide, long long wps,
                    const void* __restrict__ small_, int N, int H, int W,
                    float* __restrict__ dw, float* __restrict__ db) {
  const int c = threadIdx.x & 63, q = threadIdx.x >> 6;
  const long long npix = (long long)N * H * W;
  const long long per = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = blockIdx.x * per, p1 = (p0 + per < npix) ? p0 + per : npix;
  float acc[27];
#pragma unroll
  for (int j = 0; j < 27; ++j) acc[j] = 0.f;
  float accb = 0.f;
  for (long long p = p0 + q; p < p1; p += 4) {
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    const float v = __bfloat162float(wide[p * wps + c]);
    if (!SMALL_F32) accb += v;                       // conv_in bias: sum of dY
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = py + SGN * (ky - 1);
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = px + SGN * (kx - 1);
        if (sx < 0 || sx >= W) continue;
        const long long sp = p + (long long)SGN * ((ky - 1) * W + (kx - 1));
        float s0, s1, s2;
        if (SMALL_F32) {
          const float* sm = static_cast<const float*>(small_) + sp * 3;
          s0 = sm[0]; s1 = sm[1]; s2 = sm[2];
        } else {
          const __nv_bfloat16* sm = static_cast<const __nv_bfloat16*>(small_) + sp * 3;
          s0 = __bfloat162float(sm[0]); s1 = __bfloat162float(sm[1]); s2 = __bfloat162float(sm[2]);
        }
        const int t = ky * 3 + kx;
        acc[t * 3 + 0] += s0 * v; acc[t * 3 + 1] += s1 * v; acc[t * 3 + 2] += s2 * v;
      }
    }
    if (SMALL_F32 && c < 3) accb += static_cast<const float*>(small_)[p * 3 + c];   // conv_out bias
  }
  __shared__ float sh[4][28][64];
#pragma unroll
  for (int j = 0; j < 27; ++j) sh[q][j][c] = acc[j];
  sh[q][27][c] = accb;
  __syncthreads();
  for (int i = threadIdx.x; i < 28 * 64; i += 256) {
    const int j = i >> 6, cc = i & 63;
    const float v = sh[0][j][cc] + sh[1][j][cc] + sh[2][j][cc] + sh[3][j][cc];
    if (j < 27) {
      const int t = j / 3, k = j % 3;
      const int idx = SMALL_F32 ? (t * 64 + cc) * 3 + k : (t * 3 + k) * 64 + cc;
      atomicAdd(&dw[idx], v);
    } else if (db) {
      if (!SMALL_F32) atomicAdd(&db[cc], v);
      else if (cc < 3) atomicAdd(&db[cc], v);
    }
  }
}

// ---- conv_out forward: x bf16 act [.,Cin], w f32 [9][Cin][3], y f32 [N,H,W,3] -----------
__global__ void __launch_bounds__(128)
cout3_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long xps, const float* __restrict__ w,
                 const float* __restrict__ bias, int N, int H, int W, int Cin,
                 float* __restrict__ y) {
  extern __shared__ float sw[];   // [9][Cin][3]
  for (int i = threadIdx.x; i < 27 * Cin; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long long npix = (long long)N * H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix;
       p += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    float a0 = bias ? bias[0] : 0.f, a1 = bias ? bias[1] : 0.f, a2 = bias ? bias[2] : 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = py + ky - 1;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = px + kx - 1;
        if (ix < 0 || ix >= W) continue;
        const __nv_bfloat16* xp = x + (p + (long long)(ky - 1) * W + (kx - 1)) * xps;
        const float* wp = sw + (ky * 3 + kx) * Cin * 3;
        for (int c8 = 0; c8 < Cin; c8 += 8) {
          const uint4 u = *reinterpret_cast<const uint4*>(xp + c8);
          const float2 q0 = unpack_bf16x2(u.x), q1 = unpack_bf16x2(u.y), q2 = unpack_bf16x2(u.z),
                       q3 = unpack_bf16x2(u.w);
          const float v[8] = {q0.x, q0.y, q1.x, q1.y, q2.x, q2.y, q3.x, q3.y};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float* ww = wp + (c8 + j) * 3;
            a0 += v[j] * ww[0]; a1 += v[j] * ww[1]; a2 += v[j] * ww[2];
          }
        }
      }
    }
    y[p * 3 + 0] = a0; y[p * 3 + 1] = a1; y[p * 3 + 2] = a2;
  }
}

// ---- conv_out dgrad: dx[p][ci] = sum_{t,co} dF[p - d(t)][co] * w[t][ci][co] ---------------
__global__ void __launch_bounds__(256)
cout3_dgrad_kernel(const float* __restrict__ dF, const float* __restrict__ w, int N, int H, int W,
                   int Cin, __nv_bfloat16* __restrict__ dx, long long dxps) {
  extern __shared__ float sw[];   // [9][Cin][3]
  for (int i = threadIdx.x; i < 27 * Cin; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int vpp = Cin >> 3;
  const long long total = (long long)N * H * W * vpp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % vpp);
    const long long p = i / vpp;
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int oy = py - ky + 1;
      if (oy < 0 || oy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ox = px - kx + 1;
        if (ox < 0 || ox >= W) continue;
        const float* g = dF + (p + (long long)(1 - ky) * W + (1 - kx)) * 3;
        const float g0 = g[0], g1 = g[1], g2 = g[2];
        const float* wp = sw + ((ky * 3 + kx) * Cin + cv * 8) * 3;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += g0 * wp[j * 3] + g1 * wp[j * 3 + 1] + g2 * wp[j * 3 + 2];
      }
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(dx + p * dxps + cv * 8) = o;
  }
}

// ---- im2col of a 3-channel tensor: col[p][t*3+k] = S[p + sgn*d(t)][k] (0 outside), bf16 [P][32];
//      column 27 optionally = 1 (bias row), columns 28..31 = 0.  Feeds the wgmma engine so the two
//      3-channel weight gradients are (pixels x 32)^T (pixels x 64) GEMMs instead of CUDA-core loops.
template <bool SMALL_F32>
__global__ void __launch_bounds__(256)
im2col3_kernel(const void* __restrict__ src_, int sgn, int N, int H, int W, int ones_col,
               __nv_bfloat16* __restrict__ col) {
  const long long npix = (long long)N * H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix;
       p += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = py + sgn * (ky - 1);
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = px + sgn * (kx - 1);
        if (sx < 0 || sx >= W) continue;
        const long long sp = p + (long long)sgn * ((ky - 1) * W + (kx - 1));
        const int t = ky * 3 + kx;
        if (SMALL_F32) {
          const float* sm = static_cast<const float*>(src_) + sp * 3;
          v[t * 3] = sm[0]; v[t * 3 + 1] = sm[1]; v[t * 3 + 2] = sm[2];
        } else {
          const __nv_bfloat16* sm = static_cast<const __nv_bfloat16*>(src_) + sp * 3;
          v[t * 3] = __bfloat162float(sm[0]); v[t * 3 + 1] = __bfloat162float(sm[1]);
          v[t * 3 + 2] = __bfloat162float(sm[2]);
        }
      }
    }
    if (ones_col) v[27] = 1.f;
    uint4* o = reinterpret_cast<uint4*>(col + p * 32);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 u;
      u.x = pack_bf16x2(v[8 * j], v[8 * j + 1]); u.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
      u.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]); u.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
      o[j] = u;
    }
  }
}

// ---- col2im for conv_out: the Cin->3 convolution is a (pixels x Cin)(Cin x 27) tensor-core GEMM whose
//      f32 result col[p][t*3+k] = <x[p], w[t][:][k]> is scattered back here:
//      y[p][k] = bias[k] + sum_t col[p + d(t)][t*3+k]   (taps outside the image contribute 0 = SAME padding)
__global__ void __launch_bounds__(256)
col2im3_kernel(const float* __restrict__ col, const float* __restrict__ bias, int N, int H, int W,
               float* __restrict__ y) {
  const long long npix = (long long)N * H * W;
  const float b0 = bias ? bias[0] : 0.f, b1 = bias ? bias[1] : 0.f, b2 = bias ? bias[2] : 0.f;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix;
       p += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(p % W);
    const int py = (int)((p / W) % H);
    float a0 = b0, a1 = b1, a2 = b2;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = py + ky - 1;
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = px + kx - 1;
        if (sx < 0 || sx >= W) continue;
        const float* c = col + (p + (long long)(ky - 1) * W + (kx - 1)) * 32 + (ky * 3 + kx) * 3;
        a0 += c[0]; a1 += c[1]; a2 += c[2];
      }
    }
    y[p * 3 + 0] = a0; y[p * 3 + 1] = a1; y[p * 3 + 2] = a2;
  }
}

}  // namespace

extern "C" {

int fdx_im2col3x3_c3(const void* src, int src_is_f32, int sgn, int N, int H, int W, int ones_col,
                     void* col_bf16, void* stream) {
  FDX_REQUIRE(src && col_bf16, "im2col3x3_c3: null pointer");
  FDX_REQUIRE(sgn == 1 || sgn == -1, "im2col3x3_c3: sgn must be +1 or -1");
  const long long npix = (long long)N * H * W;
  long long grid = (npix + 255) / 256;
  if (grid > fdx_num_sms() * 16) grid = fdx_num_sms() * 16;
  if (src_is_f32)
    im2col3_kernel<true><<<(int)grid, 256, 0, (cudaStream_t)stream>>>(src, sgn, N, H, W, ones_col,
                                                                      (__nv_bfloat16*)col_bf16);
  else
    im2col3_kernel<false><<<(int)grid, 256, 0, (cudaStream_t)stream>>>(src, sgn, N, H, W, ones_col,
                                                                       (__nv_bfloat16*)col_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_conv_in_fwd(const void* x_bf16, int N, int H, int W, const float* w_hwio,
                    const float* bias, const fdx_act* y, void* stream) {
  FDX_REQUIRE(x_bf16 && w_hwio && y && y->ptr, "conv_in_fwd: null pointer");
  FDX_REQUIRE(y->n == N && y->h == H && y->w == W && y->c % 8 == 0 && y->c <= 256,
              "conv_in_fwd: bad output shape");
  const long long total = (long long)N * H * W * (y->c / 8);
  long long grid = (total + 255) / 256;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  cin3_fwd_kernel<<<(int)grid, 256, sizeof(float) * 28 * y->c, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x_bf16, w_hwio, bias, N, H, W, y->c, (__nv_bfloat16*)y->ptr,
      y->pix_stride);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_conv_in_wgrad(const void* x_bf16, const fdx_act* dy, float* dw_hwio, float* dbias,
                      void* stream) {
  FDX_REQUIRE(x_bf16 && dy && dy->ptr && dw_hwio, "conv_in_wgrad: null pointer");
  FDX_REQUIRE(dy->c == 64, "conv_in_wgrad: Cout must be 64 (got %d)", dy->c);
  rank27_wgrad_kernel<false, +1><<<fdx_num_sms() * 4, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)dy->ptr, dy->pix_stride, x_bf16, dy->n, dy->h, dy->w, dw_hwio, dbias);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_col2im3x3_c3(const float* col_f32, const float* bias, int N, int H, int W, float* y_f32,
                     void* stream) {
  FDX_REQUIRE(col_f32 && y_f32 && N > 0 && H > 0 && W > 0, "col2im3x3_c3: bad arguments");
  const long long npix = (long long)N * H * W;
  long long grid = (npix + 255) / 256;
  if (grid > fdx_num_sms() * 16) grid = fdx_num_sms() * 16;
  col2im3_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(col_f32, bias, N, H, W, y_f32);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_conv_out_fwd(const fdx_act* x, const float* w_hwio, const float* bias, float* y_f32,
                     void* stream) {
  FDX_REQUIRE(x && x->ptr && w_hwio && y_f32, "conv_out_fwd: null pointer");
  FDX_REQUIRE(x->c % 8 == 0 && x->c <= 256, "conv_out_fwd: bad Cin %d", x->c);
  const long long npix = (long long)x->n * x->h * x->w;
  long long grid = (npix + 127) / 128;
  if (grid > fdx_num_sms() * 16) grid = fdx_num_sms() * 16;
  cout3_fwd_kernel<<<(int)grid, 128, sizeof(float) * 27 * x->c, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x->ptr, x->pix_stride, w_hwio, bias, x->n, x->h, x->w, x->c, y_f32);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_conv_out_dgrad(const float* dF, const float* w_hwio, const fdx_act* dx, void* stream) {
  FDX_REQUIRE(dF && w_hwio && dx && dx->ptr, "conv_out_dgrad: null pointer");
  FDX_REQUIRE(dx->c % 8 == 0 && dx->c <= 256, "conv_out_dgrad: bad Cin %d", dx->c);
  const long long total = (long long)dx->n * dx->h * dx->w * (dx->c / 8);
  long long grid = (total + 255) / 256;
  if (grid > fdx_num_sms() * 8) grid = fdx_num_sms() * 8;
  cout3_dgrad_kernel<<<(int)grid, 256, sizeof(float) * 27 * dx->c, (cudaStream_t)stream>>>(
      dF, w_hwio, dx->n, dx->h, dx->w, dx->c, (__nv_bfloat16*)dx->ptr, dx->pix_stride);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_conv_out_wgrad(const fdx_act* x, const float* dF, float* dw_hwio, float* dbias,
                       void* stream) {
  FDX_REQUIRE(x && x->ptr && dF && dw_hwio, "conv_out_wgrad: null pointer");
  FDX_REQUIRE(x->c == 64, "conv_out_wgrad: Cin must be 64 (got %d)", x->c);
  rank27_wgrad_kernel<true, -1><<<fdx_num_sms() * 4, 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)x->ptr, x->pix_stride, dF, x->n, x->h, x->w, dw_hwio, dbias);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
