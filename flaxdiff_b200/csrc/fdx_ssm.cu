// fdx_ssm.cu -- the S5 layer of the hybrid SSM-attention DiT (flaxdiff/models/ssm_dit.py:58-286) around the GEMM
// engine: the ZOH discretisation and its backward, the diagonal complex linear recurrence x_k = Abar x_{k-1} + Bu_k
// (forward direction from token 0, backward direction from token L-1) and its adjoint, and the row permutation of the
// Hilbert / zigzag patch orders (hilbert.py:87-370).
//
// Complex state columns: a layer with `ndir` directions of N states keeps its per-token complex values in rows of
// 2 * ndir * N floats; direction d owns columns [2dN, 2dN + 2N), real parts first (2dN + n), then imaginary parts
// (2dN + N + n).  The dense products (Bu = u Bbar^T, y = Re(C x), their gradients) are fdx_gemm calls on these rows.
//
// The scans are parallel over the sequence: each sample's L steps are cut into chunks of `chunk` steps.  A first pass
// scans every chunk from zero and keeps its end value; the second pass carries the preceding chunks' end values into
// the chunk (Horner over the chunks with Abar^chunk = exp(chunk * A dt), never a product of `chunk` factors) and
// rescans it.  The state and the adjoint are f32 throughout.  Every reduction runs in a fixed order without atomics.
#include "fdx_common.cuh"
#include "../../include/fdx.h"
#include <math.h>

namespace {

constexpr int kScanBlock = 128;     // complex states per scan block
constexpr int kScanUnroll = 8;      // steps whose loads are issued together
constexpr int kDiscBlock = 256;

struct cf { float x, y; };
__device__ __forceinline__ cf cmul(cf a, cf b) { return {a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
__device__ __forceinline__ cf cmulc(cf a, cf b) { return {a.x * b.x + a.y * b.y, a.x * b.y - a.y * b.x}; }  // conj(a) b
__device__ __forceinline__ cf cfma(cf a, cf b, cf c) {   // a b + c
  return {fmaf(a.x, b.x, fmaf(-a.y, b.y, c.x)), fmaf(a.x, b.y, fmaf(a.y, b.x, c.y))};
}
__device__ __forceinline__ cf cfmac(cf a, cf b, cf c) {  // conj(a) b + c
  return {fmaf(a.x, b.x, fmaf(a.y, b.y, c.x)), fmaf(a.x, b.y, fmaf(-a.y, b.x, c.y))};
}
__device__ __forceinline__ cf cdiv(cf a, cf b) {
  const float d = 1.f / fmaf(b.x, b.x, b.y * b.y);
  return {(a.x * b.x + a.y * b.y) * d, (a.y * b.x - a.x * b.y) * d};
}
// exp(s * (re + i im)).  sincospif reduces its argument exactly, so no slow-path reduction (and no local array)
// is compiled in; the phase is therefore passed in half-turns.
__device__ __forceinline__ cf cexp_scaled(float s, float re, float im_over_pi) {
  float sn, cs;
  sincospif(s * im_over_pi, &sn, &cs);
  const float m = expf(s * re);
  return {m * cs, m * sn};
}

inline int stream_grid(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = (long long)fdx_num_sms() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// ---- discretisation (ssm_dit.py:154-172) --------------------------------------------------------------------------
// dt = exp(log_dt), A = -exp(log_A_real) + i A_imag, Abar = exp(A dt), g = (Abar - 1) / (A + 1e-8), Bbar = g B.
// Writes the bf16 operands wb[f][col0 + n] = Re Bbar[n][f], wb[f][col0 + N + n] = Im Bbar[n][f] (rows of ldb) and
// wc[n][f] = C_re[f][n], wc[N + n][f] = -C_im[f][n], and adt[col0 + n] = Re(A dt), adt[col0 + N + n] = Im(A dt) / pi.
constexpr float kInvPi = 0.3183098861837907f;

// adt = (Re(A dt), Im(A dt) / pi): the scans' exponent, from which they form Abar and Abar^chunk
__device__ __forceinline__ void ssm_state(const float* log_a_real, const float* a_imag, const float* log_dt, int n,
                                          float& dt, cf& A, cf& adt, cf& Ab, cf& g) {
  dt = expf(log_dt[n]);
  A = {-expf(log_a_real[n]), a_imag[n]};
  adt = {A.x * dt, dt * (A.y * kInvPi)};
  // Abar - 1 without the cancellation of a slow state (|Abar| -> 1): expm1(r) cos(t) - 2 sin^2(t / 2) + i e^r sin(t)
  float sn, cs, sh, ch;
  sincospif(adt.y, &sn, &cs);
  sincospif(0.5f * adt.y, &sh, &ch);
  const float em = expm1f(adt.x);
  Ab = {(em + 1.f) * cs, (em + 1.f) * sn};
  g = cdiv({fmaf(em, cs, -2.f * sh * sh), Ab.y}, {A.x + 1e-8f, A.y});
}

__global__ void ssm_discretize_kernel(const float* __restrict__ log_a_real, const float* __restrict__ a_imag,
                                      const float* __restrict__ log_dt, const float* __restrict__ b_re,
                                      const float* __restrict__ b_im, const float* __restrict__ c_re,
                                      const float* __restrict__ c_im, int N, int F, __nv_bfloat16* __restrict__ wb,
                                      int ldb, int col0, __nv_bfloat16* __restrict__ wc, float* __restrict__ adt) {
  const long long total = (long long)N * F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / F), f = (int)(i % F);
    float dt;
    cf A, adt_n, Ab, g;
    ssm_state(log_a_real, a_imag, log_dt, n, dt, A, adt_n, Ab, g);
    const cf bb = cmul(g, {b_re[i], b_im[i]});
    wb[(long long)f * ldb + col0 + n] = __float2bfloat16(bb.x);
    wb[(long long)f * ldb + col0 + N + n] = __float2bfloat16(bb.y);
    wc[i] = __float2bfloat16(c_re[(long long)f * N + n]);
    wc[(long long)N * F + i] = __float2bfloat16(-c_im[(long long)f * N + n]);
    if (f == 0) {
      adt[col0 + n] = adt_n.x;
      adt[col0 + N + n] = adt_n.y;
    }
  }
}

// Backward of the discretisation for one direction: one block per state n.  dwb rows col0 + n / col0 + N + n are
// d(Re Bbar[n]) / d(Im Bbar[n]) over f, dwc rows n / N + n are the gradients of wc; dab[p][col0 + n] / [col0 + N + n]
// and dgb[p][...] (p < nparts) are the adjoint scan's partial sums of sum_k lambda_k conj(x_{k-1}) = d(Abar) and of
// sum_k lambda_k conj(Bu_k) (the conjugate-linear convention: d = dRe + i dIm).  Since Bu = g (u B^T),
// d(g) = sum_k lambda_k conj(Bu_k) / conj(g): taken from the f32 scan rather than from the bf16 product behind dwb, it
// keeps the two paths from A into the output, through Abar and through g, in the same precision (for a slow state
// they nearly cancel).  Every output is accumulated (+=).  Sums over f and over p run in a fixed order.
__global__ void __launch_bounds__(kDiscBlock)
ssm_discretize_bwd_kernel(const float* __restrict__ log_a_real, const float* __restrict__ a_imag,
                          const float* __restrict__ log_dt, const float* __restrict__ b_re,
                          const float* __restrict__ b_im, int N, int F, const float* __restrict__ dwb, int col0,
                          const float* __restrict__ dwc, const float* __restrict__ dab,
                          const float* __restrict__ dgb, int nparts, int ld_part,
                          float* g_log_a_real, float* g_a_imag, float* g_log_dt, float* g_b_re, float* g_b_im,
                          float* g_c_re, float* g_c_im) {
  __shared__ float red[4][kDiscBlock];
  const int n = blockIdx.x, tid = threadIdx.x;
  float dt;
  cf A, adt, Ab, g;
  ssm_state(log_a_real, a_imag, log_dt, n, dt, A, adt, Ab, g);
  cf dg = {0.f, 0.f}, dA_scan = {0.f, 0.f};
  const float* dre = dwb + (long long)(col0 + n) * F;
  const float* dim = dwb + (long long)(col0 + N + n) * F;
  for (int f = tid; f < F; f += kDiscBlock) {
    const long long i = (long long)n * F + f;
    const cf db = {dre[f], dim[f]};
    const cf gb = cmulc(g, db);
    g_b_re[i] += gb.x;
    g_b_im[i] += gb.y;
    g_c_re[(long long)f * N + n] += dwc[i];
    g_c_im[(long long)f * N + n] -= dwc[(long long)N * F + i];
  }
  for (int p = tid; p < nparts; p += kDiscBlock) {
    dA_scan.x += dab[(long long)p * ld_part + col0 + n];
    dA_scan.y += dab[(long long)p * ld_part + col0 + N + n];
    dg.x += dgb[(long long)p * ld_part + col0 + n];
    dg.y += dgb[(long long)p * ld_part + col0 + N + n];
  }
  red[0][tid] = dg.x; red[1][tid] = dg.y; red[2][tid] = dA_scan.x; red[3][tid] = dA_scan.y;
  __syncthreads();
  for (int s = kDiscBlock / 2; s > 0; s >>= 1) {
    if (tid < s) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red[j][tid] += red[j][tid + s];
    }
    __syncthreads();
  }
  if (tid == 0) {
    dg = cdiv({red[0][0], red[1][0]}, {g.x, -g.y});
    const cf Ap = {A.x + 1e-8f, A.y};
    const cf inv = cdiv({1.f, 0.f}, Ap);
    const cf dAb = cfmac(inv, dg, {red[2][0], red[3][0]});        // + conj(1 / A') dg
    const cf gA = cmul(g, inv);
    const cf dAp = cmulc(gA, dg);                                 // -conj(g / A') dg, negated below
    const cf dz = cmulc(Ab, dAb);                                  // z = A dt, Abar = exp(z)
    const cf dA = {fmaf(dt, dz.x, -dAp.x), fmaf(dt, dz.y, -dAp.y)};
    const float ddt = A.x * dz.x + A.y * dz.y;                     // Re(conj(A) dz)
    g_log_a_real[n] += dA.x * A.x;
    g_a_imag[n] += dA.y;
    g_log_dt[n] += ddt * dt;
  }
}

// ---- the scan ----------------------------------------------------------------------------------------------------
// Thread (state s, chunk c, sample b).  Step i of a direction is token i (forward) or L - 1 - i (backward direction).
struct ScanPos {
  int s_ok, cre, cim, rev;
  cf a;          // Abar
  float re, im;  // A dt (imaginary part in half-turns)
};

__device__ __forceinline__ ScanPos scan_pos(const float* adt, int N, int ndir) {
  ScanPos p;
  const int S = N * ndir;
  const int s = blockIdx.x * kScanBlock + threadIdx.x;
  p.s_ok = s < S;
  const int d = p.s_ok ? s / N : 0, n = p.s_ok ? s % N : 0;
  p.cre = 2 * d * N + n;
  p.cim = p.cre + N;
  p.rev = d == 1;
  p.re = adt[p.cre];
  p.im = adt[p.cim];
  p.a = cexp_scaled(1.f, p.re, p.im);
  return p;
}

__device__ __forceinline__ long long scan_row(int b, int L, int i, int rev) {
  return (long long)b * L + (rev ? L - 1 - i : i);
}

// Pass 1: every chunk scanned from zero; its last state goes to ws[b][c][col].
__global__ void __launch_bounds__(kScanBlock)
ssm_scan_chunk_kernel(const float* __restrict__ bu, const float* __restrict__ adt, int L, int N, int ndir, int chunk,
                      float* __restrict__ ws) {
  const ScanPos p = scan_pos(adt, N, ndir);
  if (!p.s_ok) return;
  const int c = blockIdx.y, b = blockIdx.z, nch = gridDim.y, ld = 2 * N * ndir;
  const int i0 = c * chunk, i1 = min(L, i0 + chunk);
  cf h = {0.f, 0.f};
  for (int i = i0; i < i1; i += kScanUnroll) {
    cf v[kScanUnroll];
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i + j < i1) {
        const long long r = scan_row(b, L, i + j, p.rev) * ld;
        v[j] = {bu[r + p.cre], bu[r + p.cim]};
      }
    }
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j)
      if (i + j < i1) h = cfma(p.a, h, v[j]);
  }
  float* w = ws + ((long long)b * nch + c) * ld;
  w[p.cre] = h.x;
  w[p.cim] = h.y;
}

// Pass 2: carry = the state before the chunk's first step, from the end values of chunks 0..c-1 (all `chunk` long);
// rescan the chunk from it.  x (f32) may alias bu; x16 receives the bf16 copy.
__global__ void __launch_bounds__(kScanBlock)
ssm_scan_kernel(const float* bu, const float* __restrict__ adt, int L, int N, int ndir, int chunk,
                const float* __restrict__ ws, float* x, __nv_bfloat16* __restrict__ x16) {
  const ScanPos p = scan_pos(adt, N, ndir);
  if (!p.s_ok) return;
  const int c = blockIdx.y, b = blockIdx.z, nch = gridDim.y, ld = 2 * N * ndir;
  const cf pw = cexp_scaled((float)chunk, p.re, p.im);           // Abar^chunk
  cf h = {0.f, 0.f};
  const float* w = ws + (long long)b * nch * ld;
  for (int k = 0; k < c; ++k) h = cfma(pw, h, {w[(long long)k * ld + p.cre], w[(long long)k * ld + p.cim]});
  const int i0 = c * chunk, i1 = min(L, i0 + chunk);
  for (int i = i0; i < i1; i += kScanUnroll) {
    cf v[kScanUnroll];
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i + j < i1) {
        const long long r = scan_row(b, L, i + j, p.rev) * ld;
        v[j] = {bu[r + p.cre], bu[r + p.cim]};
      }
    }
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i + j < i1) {
        h = cfma(p.a, h, v[j]);
        const long long r = scan_row(b, L, i + j, p.rev) * ld;
        x[r + p.cre] = h.x;
        x[r + p.cim] = h.y;
        x16[r + p.cre] = __float2bfloat16(h.x);
        x16[r + p.cim] = __float2bfloat16(h.y);
      }
    }
  }
}

// ---- the adjoint scan: lambda_i = dx_i + conj(Abar) lambda_{i+1} (in step order) ----------------------------------
// Pass 1: every chunk's adjoint from zero past its end; the value at its first step goes to ws[b][c][col].
__global__ void __launch_bounds__(kScanBlock)
ssm_scan_bwd_chunk_kernel(const float* __restrict__ dx, const float* __restrict__ adt, int L, int N, int ndir,
                          int chunk, float* __restrict__ ws) {
  const ScanPos p = scan_pos(adt, N, ndir);
  if (!p.s_ok) return;
  const int c = blockIdx.y, b = blockIdx.z, nch = gridDim.y, ld = 2 * N * ndir;
  const int i0 = c * chunk, i1 = min(L, i0 + chunk);
  cf lam = {0.f, 0.f};
  for (int i = i1 - 1; i >= i0; i -= kScanUnroll) {
    cf v[kScanUnroll];
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i - j >= i0) {
        const long long r = scan_row(b, L, i - j, p.rev) * ld;
        v[j] = {dx[r + p.cre], dx[r + p.cim]};
      }
    }
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j)
      if (i - j >= i0) lam = cfmac(p.a, lam, v[j]);
  }
  float* w = ws + ((long long)b * nch + c) * ld;
  w[p.cre] = lam.x;
  w[p.cim] = lam.y;
}

// Pass 2: carry = the adjoint at the next chunk's first step (Horner from the last chunk down; every chunk but the
// last is `chunk` long); rescan the chunk, writing lambda (bf16) and this chunk's sums of lambda_i conj(x_{i-1}) to
// dab[b][c][col] (x_{-1} = 0) and of lambda_i conj(bu_i) to dgb[b][c][col].
__global__ void __launch_bounds__(kScanBlock)
ssm_scan_bwd_kernel(const float* __restrict__ dx, const float* __restrict__ x, const float* __restrict__ bu,
                    const float* __restrict__ adt, int L, int N, int ndir, int chunk, const float* __restrict__ ws,
                    __nv_bfloat16* __restrict__ lam16, float* __restrict__ dab, float* __restrict__ dgb) {
  const ScanPos p = scan_pos(adt, N, ndir);
  if (!p.s_ok) return;
  const int c = blockIdx.y, b = blockIdx.z, nch = gridDim.y, ld = 2 * N * ndir;
  const cf pw = cexp_scaled((float)chunk, p.re, p.im);
  cf lam = {0.f, 0.f};
  const float* w = ws + (long long)b * nch * ld;
  for (int k = nch - 1; k > c; --k) lam = cfmac(pw, lam, {w[(long long)k * ld + p.cre], w[(long long)k * ld + p.cim]});
  const int i0 = c * chunk, i1 = min(L, i0 + chunk);
  cf da = {0.f, 0.f}, dg = {0.f, 0.f};
  for (int i = i1 - 1; i >= i0; i -= kScanUnroll) {
    cf v[kScanUnroll], xp[kScanUnroll], bv[kScanUnroll];
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i - j >= i0) {
        const long long r = scan_row(b, L, i - j, p.rev) * ld;
        v[j] = {dx[r + p.cre], dx[r + p.cim]};
        bv[j] = {bu[r + p.cre], bu[r + p.cim]};
        xp[j] = {0.f, 0.f};
        if (i - j > 0) {
          const long long rp = scan_row(b, L, i - j - 1, p.rev) * ld;
          xp[j] = {x[rp + p.cre], x[rp + p.cim]};
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kScanUnroll; ++j) {
      if (i - j >= i0) {
        lam = cfmac(p.a, lam, v[j]);
        const long long r = scan_row(b, L, i - j, p.rev) * ld;
        lam16[r + p.cre] = __float2bfloat16(lam.x);
        lam16[r + p.cim] = __float2bfloat16(lam.y);
        da = cfmac(xp[j], lam, da);                                // conj(x_{i-1}) lambda_i
        dg = cfmac(bv[j], lam, dg);                                // conj(bu_i) lambda_i
      }
    }
  }
  const long long o = ((long long)b * nch + c) * ld;
  dab[o + p.cre] = da.x;
  dab[o + p.cim] = da.y;
  dgb[o + p.cre] = dg.x;
  dgb[o + p.cim] = dg.y;
}

// ---- row permutation: dst[b * L + i] = src[b * L + idx[i]], 16-byte vectors -----------------------------------------
__global__ void permute_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long rows, int L,
                                    int vecs, const int32_t* __restrict__ idx) {
  const long long total = rows * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vecs;
    const int v = (int)(i % vecs);
    const long long b = r / L;
    dst[i] = src[(b * L + idx[r % L]) * vecs + v];
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int scan_check(int B, int L, int N, int ndir, int chunk, const char* what) {
  FDX_REQUIRE(B > 0 && B <= 65535 && L > 0 && N > 0 && (ndir == 1 || ndir == 2) && chunk > 0,
              "%s: bad sizes (B=%d, L=%d, N=%d, ndir=%d, chunk=%d)", what, B, L, N, ndir, chunk);
  FDX_REQUIRE((L + chunk - 1) / chunk <= 65535, "%s: more than 65535 chunks (L=%d, chunk=%d)", what, L, chunk);
  return FDX_OK;
}

}  // namespace

extern "C" {

int fdx_ssm_discretize(const float* log_a_real, const float* a_imag, const float* log_dt, const float* b_re,
                       const float* b_im, const float* c_re, const float* c_im, int N, int F, void* wb_bf16, int ldb,
                       int col0, void* wc_bf16, float* adt, void* stream) {
  FDX_REQUIRE(log_a_real && a_imag && log_dt && b_re && b_im && c_re && c_im && wb_bf16 && wc_bf16 && adt,
              "ssm_discretize: null pointer");
  FDX_REQUIRE(N > 0 && F > 0 && col0 >= 0 && ldb >= col0 + 2 * N, "ssm_discretize: bad sizes (N=%d, F=%d, ldb=%d, "
              "col0=%d)", N, F, ldb, col0);
  ssm_discretize_kernel<<<stream_grid((long long)N * F, 256), 256, 0, (cudaStream_t)stream>>>(
      log_a_real, a_imag, log_dt, b_re, b_im, c_re, c_im, N, F, (__nv_bfloat16*)wb_bf16, ldb, col0,
      (__nv_bfloat16*)wc_bf16, adt);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_ssm_discretize_bwd(const float* log_a_real, const float* a_imag, const float* log_dt, const float* b_re,
                           const float* b_im, int N, int F, const float* dwb, int col0, const float* dwc,
                           const float* dabar, const float* dgbar, int nparts, int ld_part, float* g_log_a_real,
                           float* g_a_imag, float* g_log_dt, float* g_b_re, float* g_b_im, float* g_c_re,
                           float* g_c_im, void* stream) {
  FDX_REQUIRE(log_a_real && a_imag && log_dt && b_re && b_im && dwb && dwc && dabar && dgbar && g_log_a_real &&
                  g_a_imag &&
                  g_log_dt && g_b_re && g_b_im && g_c_re && g_c_im,
              "ssm_discretize_bwd: null pointer");
  FDX_REQUIRE(N > 0 && F > 0 && nparts > 0 && col0 >= 0 && ld_part >= col0 + 2 * N,
              "ssm_discretize_bwd: bad sizes (N=%d, F=%d, nparts=%d, ld_part=%d, col0=%d)", N, F, nparts, ld_part,
              col0);
  ssm_discretize_bwd_kernel<<<N, kDiscBlock, 0, (cudaStream_t)stream>>>(
      log_a_real, a_imag, log_dt, b_re, b_im, N, F, dwb, col0, dwc, dabar, dgbar, nparts, ld_part, g_log_a_real,
      g_a_imag, g_log_dt, g_b_re, g_b_im, g_c_re, g_c_im);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_ssm_scan(const float* bu, float* x, void* x_bf16, const float* adt, int B, int L, int N, int ndir, int chunk,
                 float* ws, void* stream) {
  FDX_REQUIRE(bu && x && x_bf16 && adt && ws, "ssm_scan: null pointer");
  const int s = scan_check(B, L, N, ndir, chunk, "ssm_scan");
  if (s != FDX_OK) return s;
  const dim3 grid((N * ndir + kScanBlock - 1) / kScanBlock, (L + chunk - 1) / chunk, B);
  cudaStream_t st = (cudaStream_t)stream;
  ssm_scan_chunk_kernel<<<grid, kScanBlock, 0, st>>>(bu, adt, L, N, ndir, chunk, ws);
  FDX_LAUNCH_CHECK();
  ssm_scan_kernel<<<grid, kScanBlock, 0, st>>>(bu, adt, L, N, ndir, chunk, ws, x, (__nv_bfloat16*)x_bf16);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_ssm_scan_bwd(const float* dx, const float* x, const float* bu, const float* adt, int B, int L, int N, int ndir,
                     int chunk, float* ws, void* lam_bf16, float* dabar, float* dgbar, void* stream) {
  FDX_REQUIRE(dx && x && bu && adt && ws && lam_bf16 && dabar && dgbar, "ssm_scan_bwd: null pointer");
  const int s = scan_check(B, L, N, ndir, chunk, "ssm_scan_bwd");
  if (s != FDX_OK) return s;
  const dim3 grid((N * ndir + kScanBlock - 1) / kScanBlock, (L + chunk - 1) / chunk, B);
  cudaStream_t st = (cudaStream_t)stream;
  ssm_scan_bwd_chunk_kernel<<<grid, kScanBlock, 0, st>>>(dx, adt, L, N, ndir, chunk, ws);
  FDX_LAUNCH_CHECK();
  ssm_scan_bwd_kernel<<<grid, kScanBlock, 0, st>>>(dx, x, bu, adt, L, N, ndir, chunk, ws, (__nv_bfloat16*)lam_bf16,
                                                   dabar, dgbar);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

int fdx_permute_rows(const void* src, void* dst, long long rows, int L, long long row_bytes, const int32_t* idx,
                     void* stream) {
  FDX_REQUIRE(src && dst && idx && src != dst, "permute_rows: null or aliased pointer");
  FDX_REQUIRE(rows > 0 && L > 0 && rows % L == 0 && row_bytes > 0 && row_bytes % 16 == 0 && aligned16(src) &&
                  aligned16(dst),
              "permute_rows: rows a multiple of L, rows of a multiple of 16 bytes, 16-byte aligned tensors");
  const int vecs = (int)(row_bytes / 16);
  permute_rows_kernel<<<stream_grid(rows * vecs, 256), 256, 0, (cudaStream_t)stream>>>(
      (const uint4*)src, (uint4*)dst, rows, L, vecs, idx);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // extern "C"
