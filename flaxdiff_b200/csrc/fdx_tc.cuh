// fdx_tc.cuh -- launch descriptor of the wgmma "tap-GEMM" engine (fdx_tc.cu).
//
// One persistent, warp-specialised kernel computes
//     D[m, n] = alpha * sum_{tap t} sum_{k} A_t[m, k] * B_t[n, k]   (+ epilogue)
// where the A operand is a 4-D NHWC (or strided 2-D / batched) bf16 tensor read
// through TMA with a per-tap spatial shift (zero fill outside the image = SAME
// padding), and B is either K-major ([n][k], k contiguous) or MN-major
// ([k][n], n contiguous).  This single engine is the 3x3 conv forward, dgrad,
// wgrad, 1x1 conv, dense layer and the attention contractions.
#pragma once
#include "fdx_common.cuh"
#include "../../include/fdx.h"

struct TcOperand {
  const void* ptr;        // bf16
  uint64_t dims[4];       // innermost first: (c, x, y, n)
  uint64_t strides[4];    // in ELEMENTS; strides[0] must be 1
};

enum TcMode {
  TC_KK = 0,     // A K-major (rows = pixels, k = channels), B K-major
  TC_KMN = 1,    // A K-major, B MN-major (n contiguous, k = rows)
  TC_MNMN = 2,   // A MN-major (m = channels, k = pixels), B MN-major  (wgrad-type)
};

constexpr int kTcMaxTaps = 16;   // 9 for a 3x3 conv, 16 = 4 phases x 2x2 taps of the sub-pixel upsample conv

struct TcLaunch {
  int mode;
  TcOperand A, B;
  // logical output pixel space (x, y, n) for TC_KK/TC_KMN; reduction pixel space for TC_MNMN
  int W, H, N;
  int es;                 // element stride of the A read (1, or 2 for stride-2 conv)
  int ntaps;              // 1..kTcMaxTaps
  int tap_dx[kTcMaxTaps], tap_dy[kTcMaxTaps];   // A spatial offset of tap t (already includes -pad)
  int tap_b[kTcMaxTaps];  // TC_KK: B z1 coordinate of tap t; TC_KMN: B row offset of tap t (elements of k);
                          // TC_MNMN: output slab index of tap t
  // TC_MNMN only: the B operand may be a strided, shifted view of its tensor (element stride es_b,
  // per-tap offset) - the output-parity view of dY in the sub-pixel upsample weight gradient
  int es_b;               // 0/1 = dense, 2 = every other pixel
  int tap_bdx[kTcMaxTaps], tap_bdy[kTcMaxTaps];
  int K;                  // channels per tap (TC_KK/TC_KMN); ignored for TC_MNMN
  int M;                  // TC_MNMN only: valid rows (channels of A)
  int Ncols;              // total output columns
  int b_batched;          // B z1/z2 coordinates follow the tile's (y, n) block (batched GEMM)
  int mn_batched;         // TC_MNMN: reduce over x only; (y, n) index the batch (os_y/os_n used)
  int gemm_like;          // rows along x only (no 2-D pixel patch)
  // epilogue
  void* out;              // bf16 or f32
  int out_f32;
  int out_atomic;         // f32 atomicAdd (TC_MNMN split-K)
  long long os_x, os_y, os_n;   // output element offsets per pixel coordinate (TC_KK/TC_KMN)
  long long os_tap, os_m;       // TC_MNMN: out[tap_b*os_tap + m*os_m + n]
  float alpha;
  const float* bias;      // [Ncols] or null
  const float* rowvec;    // [N][Ncols] per-image vector (timestep embedding add) or null
  const void* res;        // bf16 residual / accumulate source or null
  long long rs_x, rs_y, rs_n;
  int splits;             // TC_MNMN: split-K factor (0 = auto)
  // Fused first pass of GroupNorm(+SiLU) backward (TC_KK only): res = the norm's input x,
  // gn_ab = [N][2][Ncols] (a, b), gn_ws = [gn_slots][N][2][Ncols] zeroed sums; out receives dz.
  const float* gn_ab;
  float* gn_ws;
  int gn_slots;
  int gn_mish;            // with gn_ab: dz = dy * mish'(z) instead of silu'(z); transposed engine only
  // gn_ws without gn_ab (TC_KMN only): per-(image, output channel) sum / sum of squares of the stored
  // values, gn_ws = [gn_slots][N][2][ws_ld] already offset to this launch's first channel.
  int ws_ld;
  // Two-source A (one-tap K-major GEMMs): k < cat_k0 reads A, k >= cat_k0 reads A1 at k - cat_k0.  cat_k0 is a
  // multiple of 64, so every 64-deep k chunk comes from one source.  A1.ptr == nullptr = one source.
  TcOperand A1;
  int cat_k0;
};

int fdx_tc_launch(const TcLaunch& L, cudaStream_t stream);

// All-nine-taps weight-gradient kernel (fdx_wgrad9.cu); FDX_ERR_UNSUPPORTED = shape not covered.
int fdx_wgrad9_launch(const fdx_act* x, const fdx_act* dy, float* dw, cudaStream_t stream);

// Transposed formulation (weights as A, 256 pixels as N) for Ncols = 64 / 128 (fdx_tct.cu);
// FDX_ERR_UNSUPPORTED = geometry not covered.
int fdx_tct_launch(const TcLaunch& L, cudaStream_t stream);
