// fdx_epilogue.cuh -- coalesced bf16 epilogue for the wgmma kernels.
//
// WgAcc::row32 hands every thread of a consumer warp one accumulator ROW (one output pixel).  Storing
// straight from that layout makes each 16-byte store instruction of a warp touch 32 different cache
// lines.  Here each warp stages its 32 rows x 64 channels (4 KB, XOR-swizzled 16-byte pieces, conflict free)
// in shared memory and moves it to / from global memory with 8 lanes per pixel: four complete
// 128-byte lines per instruction, for the store and for the fused side-input read alike.  Each 64-column
// chunk loads its own side input (residual, or the GroupNorm input below) just before its accumulator
// exchange; the caller requests those lines into L2 before the main loop, so the load is an L2 hit.  Holding
// the next chunk's side input in registers instead would not fit beside a 128 x 128 accumulator.
//
// EPI = EPI_COLSTATS additionally accumulates, per (image, output channel), the sum and the sum of
// squares of the bf16 values it stores: the statistics pass of the GroupNorm that consumes this tensor
// (flaxdiff/models/common.py:273-288) then never reads it (2 B/element saved; two fused multiply-adds
// per element in the coalesced store phase).
//
// EPI = EPI_GN_BWD fuses the first pass of GroupNorm(+SiLU) backward (flaxdiff/models/common.py:286-288,
// 310-312 under jax.grad) into the data-gradient convolution that produces its input: with
// z = a_c x + b_c (a_c = rstd*gamma_c, b_c = beta_c - mean*a_c, per image) the kernel writes
// dz = dy * silu'(z) instead of dy and accumulates the two per-(image, channel) sums the backward
// needs, S0 = sum dz and S1 = sum dz*x, so that no separate statistics pass reads x and dy again.
#pragma once
#include "fdx_common.cuh"

struct EpiArgs {
  void* out;               // bf16
  const float* bias;       // [Ncols] or null
  const float* rowvec;     // [N][Ncols] or null
  const void* res;         // bf16 or null (GN: the GroupNorm input x)
  int Ncols;
  float alpha;
  // ---- EPI_GN_BWD / EPI_COLSTATS only ----
  const float* gn_ab;      // EPI_GN_BWD: [N][2][Ncols]: a then b
  float* gn_ws;            // [slots][N][2][ws_ld] f32 atomics: (sum dz, sum dz*x) or (sum y, sum y*y)
  int gn_N;                // images
  int ws_ld;               // channels per row of gn_ws (the destination BUFFER's channel count)
};

enum { EPI_PLAIN = 0, EPI_GN_BWD = 1, EPI_COLSTATS = 2 };

__device__ __forceinline__ uint32_t epi_swz(int row, int piece) {   // byte offset inside a warp's 4 KB tile
  return (uint32_t)(row * 128 + ((piece ^ (row & 7)) << 4));
}

__device__ __forceinline__ float epi_silu_grad_times(float dy, float z) {
  const float sg = sigmoid_fast(z);
  return dy * sg * (1.f + z * (1.f - sg));
}

// One warp of a consumer warpgroup, its 32 accumulator rows, the warpgroup's WN columns of the tile.
//   stage   : this warp's 4 KB staging tile (shared memory, 128-byte aligned)
//   acc, xs, xbar : the warpgroup's accumulator, its exchange tile and named barrier (see WgAcc::row32)
//   col_base: first global output column of the warpgroup's columns
//   valid / obase / rbase / img : this LANE's row: in range?, element offsets into out / res, image index
//   mainloop: called once to compute the accumulator
//   GN only : par = running chunk parity (kept by the caller across tiles), slot = workspace slot of
//             this tile; all rows of the tile belong to image `img` of lane 0.
// Row offsets are kept as 32-bit distances from lane 0's row (the host checks that a tile's rows span less than
// 2^31 elements).  The chunk loop is unrolled, so every WgAcc::row32 reads fixed registers and a chunk's
// accumulator registers are free once it is written: the accumulator never leaves the register file, and ptxas
// does not serialise the main loop's wgmma.
template <int WN, int EPI, class Acc, class MainFn>
__device__ __forceinline__ void epilogue_bf16_coalesced(const EpiArgs& e, uint8_t* stage, const Acc& acc, float* xs,
                                                       int xbar, int lane, int col_base, bool valid, long long obase,
                                                       long long rbase, int img, MainFn mainloop, int* par = nullptr,
                                                       int slot = 0) {
  constexpr bool GN = (EPI == EPI_GN_BWD);
  constexpr bool SUMS = (EPI != EPI_PLAIN);
  const uint32_t sbase = smem_u32(stage);
  const int sub = lane >> 3, piece = lane & 7;       // coalesced phase: 4 rows x 8 pieces per instruction
  const bool side = (e.res != nullptr);
  const long long rbase0 = __shfl_sync(0xffffffffu, rbase, 0), obase0 = __shfl_sync(0xffffffffu, obase, 0);
  const __nv_bfloat16* resp = side ? static_cast<const __nv_bfloat16*>(e.res) + rbase0 : nullptr;
  __nv_bfloat16* outp = static_cast<__nv_bfloat16*>(e.out) + obase0;

  // per-lane coalesced coordinates: rows 4k + sub, k = 0..7
  int rb_k[8], ob_k[8];
  uint32_t ok_mask = 0;
  {
    const int rd = (int)(rbase - rbase0), od = (int)(obase - obase0);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int r = 4 * k + sub;
      rb_k[k] = __shfl_sync(0xffffffffu, rd, r);
      ob_k[k] = __shfl_sync(0xffffffffu, od, r);
      if (__shfl_sync(0xffffffffu, (int)valid, r)) ok_mask |= 1u << k;
    }
  }
  const int img0 = __shfl_sync(0xffffffffu, img, 0);

  mainloop();

#pragma unroll
  for (int c0 = 0; c0 < WN; c0 += 64) {
    const int col0 = col_base + c0;
    if (col0 >= e.Ncols) break;                      // uniform over the CTA
    const bool half2 = (col0 + 32) < e.Ncols;        // second 32-column half present (Ncols % 32 == 0)
    // ---- side input of this chunk: global -> registers -> shared (coalesced layout) -----------------
    // Loaded before the accumulator exchange so that its latency overlaps it; the lines were requested
    // into L2 before the main loop.
    uint4 xr[8];
    if (side) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        xr[k] = make_uint4(0, 0, 0, 0);
        if (((ok_mask >> k) & 1u) && (piece < 4 || half2))
          xr[k] = *reinterpret_cast<const uint4*>(resp + rb_k[k] + col0 + piece * 8);
      }
#pragma unroll
      for (int k = 0; k < 8; ++k)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + epi_swz(4 * k + sub, piece)),
                     "r"(xr[k].x), "r"(xr[k].y), "r"(xr[k].z), "r"(xr[k].w)
                     : "memory");
      __syncwarp();
    }
    // ---- accumulator rows -> bf16 in shared -----------------------------------------------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !half2) break;
      float f[32];
      acc.row32(xs, xbar, c0 + h * 32, f);
#pragma unroll
      for (int j = 0; j < 32; ++j) f[j] *= e.alpha;
      if (e.bias) {
        const float4* b4 = reinterpret_cast<const float4*>(e.bias + col0 + h * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 b = __ldg(b4 + j);
          f[4 * j] += b.x; f[4 * j + 1] += b.y; f[4 * j + 2] += b.z; f[4 * j + 3] += b.w;
        }
      }
      if (e.rowvec) {
        // rows outside the tensor (tile padding) must not index the per-image vector
        const float4* r4 =
            reinterpret_cast<const float4*>(e.rowvec + (long long)(valid ? img : 0) * e.Ncols + col0 + h * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 b = __ldg(r4 + j);
          f[4 * j] += b.x; f[4 * j + 1] += b.y; f[4 * j + 2] += b.z; f[4 * j + 3] += b.w;
        }
      }
      const float4* ga4 = nullptr;
      const float4* gb4 = nullptr;
      if constexpr (GN) {
        const float* ab = e.gn_ab + (long long)img0 * 2 * e.Ncols + col0 + h * 32;
        ga4 = reinterpret_cast<const float4*>(ab);
        gb4 = reinterpret_cast<const float4*>(ab + e.Ncols);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t addr = sbase + epi_swz(lane, h * 4 + j);
        if (side) {
          uint4 u;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                       : "r"(addr)
                       : "memory");
          const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z),
                       d = unpack_bf16x2(u.w);
          const float xv[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
          if constexpr (GN) {
            const float4 a0 = __ldg(ga4 + 2 * j), a1 = __ldg(ga4 + 2 * j + 1);
            const float4 b0 = __ldg(gb4 + 2 * j), b1 = __ldg(gb4 + 2 * j + 1);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
              f[8 * j + i] = epi_silu_grad_times(f[8 * j + i], fmaf(xv[i], av[i], bv[i]));
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) f[8 * j + i] += xv[i];
          }
        }
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr),
                     "r"(pack_bf16x2(f[8 * j + 0], f[8 * j + 1])), "r"(pack_bf16x2(f[8 * j + 2], f[8 * j + 3])),
                     "r"(pack_bf16x2(f[8 * j + 4], f[8 * j + 5])), "r"(pack_bf16x2(f[8 * j + 6], f[8 * j + 7]))
                     : "memory");
      }
    }
    __syncwarp();
    // ---- shared -> global, coalesced (GN: plus the column sums of dz and dz*x) ---------------------
    float s0[8], s1[8];
    if constexpr (SUMS) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { s0[i] = 0.f; s1[i] = 0.f; }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      uint4 u;
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                   : "r"(sbase + epi_swz(4 * k + sub, piece))
                   : "memory");
      const bool live = ((ok_mask >> k) & 1u) && (piece < 4 || half2);
      if (live) *reinterpret_cast<uint4*>(outp + ob_k[k] + col0 + piece * 8) = u;
      if constexpr (SUMS) {
        if (live) {
          const float2 d0 = unpack_bf16x2(u.x), d1 = unpack_bf16x2(u.y), d2 = unpack_bf16x2(u.z),
                       d3 = unpack_bf16x2(u.w);
          // second factor: the GroupNorm input x (EPI_GN_BWD; read again, an L1 hit, rather than held in
          // registers through the accumulator exchange) or the stored value itself (EPI_COLSTATS)
          const uint4 xq = GN ? *reinterpret_cast<const uint4*>(resp + rb_k[k] + col0 + piece * 8) : u;
          const float2 x0 = unpack_bf16x2(xq.x), x1 = unpack_bf16x2(xq.y), x2 = unpack_bf16x2(xq.z),
                       x3 = unpack_bf16x2(xq.w);
          s0[0] += d0.x; s0[1] += d0.y; s0[2] += d1.x; s0[3] += d1.y;
          s0[4] += d2.x; s0[5] += d2.y; s0[6] += d3.x; s0[7] += d3.y;
          s1[0] = fmaf(d0.x, x0.x, s1[0]); s1[1] = fmaf(d0.y, x0.y, s1[1]);
          s1[2] = fmaf(d1.x, x1.x, s1[2]); s1[3] = fmaf(d1.y, x1.y, s1[3]);
          s1[4] = fmaf(d2.x, x2.x, s1[4]); s1[5] = fmaf(d2.y, x2.y, s1[5]);
          s1[6] = fmaf(d3.x, x3.x, s1[6]); s1[7] = fmaf(d3.y, x3.y, s1[7]);
        }
      }
    }
    if constexpr (SUMS) {
      // rows of this warp: combine the four `sub` lane groups; lanes 0..7 then own 8 channels each
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s0[i] += __shfl_xor_sync(0xffffffffu, s0[i], 8);
        s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], 8);
        s0[i] += __shfl_xor_sync(0xffffffffu, s0[i], 16);
        s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], 16);
      }
      // each warp adds its own 32-row partial (lanes 0..7 own 8 channels each) with 16-byte reductions
      if (lane < 8 && (piece < 4 || half2)) {
        float* d0 = e.gn_ws + (((long long)slot * e.gn_N + img0) * 2) * e.ws_ld + col0 + piece * 8;
        float* d1 = d0 + e.ws_ld;
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d0), "f"(s0[0]), "f"(s0[1]), "f"(s0[2]),
                     "f"(s0[3]) : "memory");
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d0 + 4), "f"(s0[4]), "f"(s0[5]),
                     "f"(s0[6]), "f"(s0[7]) : "memory");
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d1), "f"(s1[0]), "f"(s1[1]), "f"(s1[2]),
                     "f"(s1[3]) : "memory");
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d1 + 4), "f"(s1[4]), "f"(s1[5]),
                     "f"(s1[6]), "f"(s1[7]) : "memory");
      }
      *par ^= 1;
    }
    __syncwarp();
  }
}
