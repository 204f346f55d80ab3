// fdx_random.cu -- jax.random's threefry streams on the device (JAX 0.4.28, jax_threefry_partitionable=False).
//
// Reference call sites replaced (jax.random calls lowered by XLA):
//   jax.random.normal       x_T and the per-step noise of the ancestral samplers   samplers/common.py:253-260,
//                           samplers/euler.py:39-56, ddpm.py:6-37; the training noise  general_diffusion_trainer.py:283
//   jax.random.randint / uniform     timesteps                                      schedulers/discrete.py:60-63, common.py
//   jax.random.bernoulli             unconditional mask (= uniform < p)             general_diffusion_trainer.py:266-275
//
// threefry_random_bits for 32-bit words: m = ceil(n/2) blocks, block i encrypts the counter pair (i, i + m); word 0
// of block i is element i, word 1 is element i + m (for odd n the last word 1 is dropped).  One thread computes one
// block, so its two words land m elements apart.  A CTA stages a tile of blocks in shared memory and writes both
// halves from there with 16-byte stores on 16-byte-aligned addresses; the ragged head and tail of each half (m and
// the output pointer need not be multiples of four words) go out as 4-byte stores.
//
// The key comes by value or, when key_dev is non-null, from two words of device memory: a captured graph is replayed
// with a new key by overwriting those 8 bytes.
#include "fdx_common.cuh"
#include "../../include/fdx.h"

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;
constexpr int kTile = kThreads * kPerThread;   // blocks (= words per half) staged per CTA iteration

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return __funnelshift_l(x, x, r); }

// Threefry-2x32, 20 rounds (Salmon et al., Random123), as jax/_src/prng.py threefry2x32
__device__ __forceinline__ void threefry2x32(uint32_t k0, uint32_t k1, uint32_t& x0, uint32_t& x1) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  x0 += ks[0];
  x1 += ks[1];
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if (i % 2 == 0) {
      x0 += x1; x1 = rotl32(x1, 13) ^ x0;  x0 += x1; x1 = rotl32(x1, 15) ^ x0;
      x0 += x1; x1 = rotl32(x1, 26) ^ x0;  x0 += x1; x1 = rotl32(x1, 6) ^ x0;
    } else {
      x0 += x1; x1 = rotl32(x1, 17) ^ x0;  x0 += x1; x1 = rotl32(x1, 29) ^ x0;
      x0 += x1; x1 = rotl32(x1, 16) ^ x0;  x0 += x1; x1 = rotl32(x1, 24) ^ x0;
    }
    x0 += ks[(i + 1) % 3];
    x1 += ks[(i + 2) % 3] + (uint32_t)(i + 1);
  }
}

// jax.random.uniform: 23 random mantissa bits under exponent 0 give [1, 2); every operation rounds to f32 on its
// own (no FMA contraction), in JAX's order.
__device__ __forceinline__ float bits_to_uniform(uint32_t bits, float minval, float span) {
  const float f = __fsub_rn(__uint_as_float((bits >> 9) | 0x3F800000u), 1.0f);
  return fmaxf(minval, __fadd_rn(__fmul_rn(f, span), minval));
}

// XLA's single-precision erf_inv (Giles 2010, "Approximating the erfinv function"), one rounding per operation.
// |u| < 1 by construction of the uniform that feeds it, so the +-inf edge case of XLA's version cannot occur.
__device__ __forceinline__ float erfinv_f32(float u) {
  float w = -log1pf(__fmul_rn(-u, u));
  float p;
  if (w < 5.0f) {
    w = __fsub_rn(w, 2.5f);
    p = 2.81022636e-08f;
    p = __fadd_rn(3.43273939e-07f, __fmul_rn(p, w));
    p = __fadd_rn(-3.5233877e-06f, __fmul_rn(p, w));
    p = __fadd_rn(-4.39150654e-06f, __fmul_rn(p, w));
    p = __fadd_rn(0.00021858087f, __fmul_rn(p, w));
    p = __fadd_rn(-0.00125372503f, __fmul_rn(p, w));
    p = __fadd_rn(-0.00417768164f, __fmul_rn(p, w));
    p = __fadd_rn(0.246640727f, __fmul_rn(p, w));
    p = __fadd_rn(1.50140941f, __fmul_rn(p, w));
  } else {
    w = __fsub_rn(__fsqrt_rn(w), 3.0f);
    p = -0.000200214257f;
    p = __fadd_rn(0.000100950558f, __fmul_rn(p, w));
    p = __fadd_rn(0.00134934322f, __fmul_rn(p, w));
    p = __fadd_rn(-0.00367342844f, __fmul_rn(p, w));
    p = __fadd_rn(0.00573950773f, __fmul_rn(p, w));
    p = __fadd_rn(-0.0076224613f, __fmul_rn(p, w));
    p = __fadd_rn(0.00943887047f, __fmul_rn(p, w));
    p = __fadd_rn(1.00167406f, __fmul_rn(p, w));
    p = __fadd_rn(2.83297682f, __fmul_rn(p, w));
  }
  return __fmul_rn(p, u);
}

enum Kind { kBits = 0, kUniform = 1, kNormal = 2, kRandint = 3 };

struct RandomArgs {
  uint32_t k0, k1;
  const uint32_t* key_dev;
  long long n;
  float minval, maxval;   // uniform
  int imin, imax;         // randint
  uint32_t* out;
};

template <int KIND>
__global__ void __launch_bounds__(kThreads) fdx_random_kernel(const RandomArgs a) {
  __shared__ uint32_t sh[2][kTile];
  uint32_t k0 = a.k0, k1 = a.k1;
  if (a.key_dev) { k0 = a.key_dev[0]; k1 = a.key_dev[1]; }
  const long long n = a.n, m = (n + 1) / 2;

  // per-kind constants
  float fmin = 0.f, fspan = 0.f;
  uint32_t j0 = 0, j1 = 0, span = 1, mult = 0;
  if (KIND == kUniform) { fmin = a.minval; fspan = __fsub_rn(a.maxval, a.minval); }
  if (KIND == kNormal) { fmin = -0.99999994f; fspan = __fsub_rn(1.0f, fmin); }   // nextafter(-1, 0)
  if (KIND == kRandint) {
    // split(key): random_bits(key, 4).reshape(2, 2) -> the blocks (0, 2) and (1, 3) give (a0, b0), (a1, b1);
    // the higher bits are drawn from (a0, a1), the lower bits from (b0, b1)
    uint32_t a0 = 0, b0 = 2, a1 = 1, b1 = 3;
    threefry2x32(k0, k1, a0, b0);
    threefry2x32(k0, k1, a1, b1);
    k0 = a0; k1 = a1; j0 = b0; j1 = b1;
    span = (uint32_t)a.imax - (uint32_t)a.imin;
    mult = 65536u % span;
    mult = (mult * mult) % span;
  }

  const long long off = (long long)((reinterpret_cast<uintptr_t>(a.out) >> 2) & 3);
  for (long long T = (long long)blockIdx.x * kTile; T < m; T += (long long)gridDim.x * kTile) {
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) {
      const int s = threadIdx.x + j * kThreads;
      const long long i = T + s;
      if (i < m) {
        uint32_t w0 = (uint32_t)i, w1 = (uint32_t)(i + m);
        threefry2x32(k0, k1, w0, w1);
        if (KIND == kUniform) {
          w0 = __float_as_uint(bits_to_uniform(w0, fmin, fspan));
          w1 = __float_as_uint(bits_to_uniform(w1, fmin, fspan));
        } else if (KIND == kNormal) {
          w0 = __float_as_uint(__fmul_rn(1.41421354f, erfinv_f32(bits_to_uniform(w0, fmin, fspan))));
          w1 = __float_as_uint(__fmul_rn(1.41421354f, erfinv_f32(bits_to_uniform(w1, fmin, fspan))));
        } else if (KIND == kRandint) {
          uint32_t l0 = (uint32_t)i, l1 = (uint32_t)(i + m);
          threefry2x32(j0, j1, l0, l1);
          w0 = (uint32_t)a.imin + ((w0 % span) * mult + (l0 % span)) % span;
          w1 = (uint32_t)a.imin + ((w1 % span) * mult + (l1 % span)) % span;
        }
        sh[0][s] = w0;
        sh[1][s] = w1;
      }
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // this tile's words of half h are the elements [lo, hi) of the output
      const long long lo = (h ? m : 0) + T;
      long long hi = lo + kTile;
      const long long end = h ? n : m;
      if (hi > end) hi = end;
      // groups of four elements whose first address is 16-byte aligned; the first group may start before lo
      const long long g0 = ((lo + off) & ~3LL) - off;
      for (long long g = g0 + 4LL * threadIdx.x; g < hi; g += 4LL * kThreads) {
        if (g >= lo && g + 4 <= hi) {
          const uint32_t* s = &sh[h][g - lo];
          *reinterpret_cast<uint4*>(a.out + g) = make_uint4(s[0], s[1], s[2], s[3]);
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (g + e >= lo && g + e < hi) a.out[g + e] = sh[h][g + e - lo];
        }
      }
    }
    __syncthreads();
  }
}

template <int KIND>
int launch_random(RandomArgs a, void* stream) {
  if (a.n == 0) return FDX_OK;
  const long long tiles = ((a.n + 1) / 2 + kTile - 1) / kTile;
  long long grid = (long long)fdx_num_sms() * 8;
  if (grid > tiles) grid = tiles;
  fdx_random_kernel<KIND><<<(int)grid, kThreads, 0, (cudaStream_t)stream>>>(a);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

}  // namespace

#define FDX_RANDOM_CHECK(who)                                                                         \
  FDX_REQUIRE(n >= 0 && n <= 2147483647LL, who ": n=%lld must be in [0, 2^31-1]", n);                 \
  FDX_REQUIRE(n == 0 || out, who ": null output");                                                    \
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(out) & 3) == 0, who ": out must be 4-byte aligned");       \
  FDX_REQUIRE((reinterpret_cast<uintptr_t>(key_dev) & 3) == 0, who ": key_dev must be 4-byte aligned")

extern "C" {

int fdx_random_bits(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, uint32_t* out, void* stream) {
  FDX_RANDOM_CHECK("random_bits");
  RandomArgs a{k0, k1, key_dev, n, 0.f, 0.f, 0, 0, out};
  return launch_random<kBits>(a, stream);
}

int fdx_random_uniform(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, float minval, float maxval,
                       float* out, void* stream) {
  FDX_RANDOM_CHECK("random_uniform");
  FDX_REQUIRE(minval < maxval, "random_uniform: minval=%g must be below maxval=%g", (double)minval, (double)maxval);
  RandomArgs a{k0, k1, key_dev, n, minval, maxval, 0, 0, reinterpret_cast<uint32_t*>(out)};
  return launch_random<kUniform>(a, stream);
}

int fdx_random_normal(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, float* out, void* stream) {
  FDX_RANDOM_CHECK("random_normal");
  RandomArgs a{k0, k1, key_dev, n, 0.f, 0.f, 0, 0, reinterpret_cast<uint32_t*>(out)};
  return launch_random<kNormal>(a, stream);
}

int fdx_random_randint(uint32_t k0, uint32_t k1, const uint32_t* key_dev, long long n, int minval, int maxval,
                       int32_t* out, void* stream) {
  FDX_RANDOM_CHECK("random_randint");
  FDX_REQUIRE(minval < maxval, "random_randint: minval=%d must be below maxval=%d", minval, maxval);
  RandomArgs a{k0, k1, key_dev, n, 0.f, 0.f, minval, maxval, reinterpret_cast<uint32_t*>(out)};
  return launch_random<kRandint>(a, stream);
}

}  // extern "C"
