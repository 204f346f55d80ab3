// fdx_tct.cu -- the TRANSPOSED formulation of the 3x3 convolution (forward and data gradient) for
// layers with few output channels (Cout = 64 / 128 forward, Cin = 64 .. 384 in the data gradient).
//
// fdx_tc.cu puts the pixels in the M dimension, so a Cout = 64 layer can only issue N = 64 MMAs, whose
// shared-memory operand traffic per FLOP is twice that of N = 128.  Here the roles are swapped,
//     D^T[co, px] = sum_tap sum_ci  W_tap[ci, co]  *  X[px + tap, ci]
// A = the weight tile (64 output channels x 64 k; MN-major straight from HWIO in the forward, K-major from the
// (Cout, Cin, tap) view in the data gradient), B = 256 pixels (a 16 x 16 block, 64 channels, K-major).  The
// accumulator is D^T: row = output channel, column = pixel, one m64 n256 k16 wgmma per K step.  A tile is one
// 64-channel column block of one 16 x 16 pixel block; a layer with more columns has one tile per 64-column
// block, and tiles that differ only in their column block are adjacent in tile order, so they run at about
// the same time on neighbouring CTAs and the second block's pixel loads hit L2.
//
// Ping-pong: warps 8..11 = producer (one thread issues TMA into one ring, in tile order), warps 0..7 = two
// consumer warpgroups that take alternate tiles of the CTA's persistent tile sequence.  Each owns its whole
// tile (128 accumulator registers per thread), so warpgroup 0 runs the main loop of tile 2i while warpgroup 1
// runs the epilogue of tile 2i - 1: output stores and side-input loads overlap the other tile's MMAs.
// The epilogue moves its HBM traffic by TMA as well: each warpgroup's leader requests the side input (residual,
// accumulate source, or x of the fused GroupNorm backward) of a tile's first 32-pixel chunks when the tile's main
// loop starts, into a ring of 4 KB chunk buffers, and stores each finished chunk from the same buffer with one
// bulk tensor store, so neither direction waits on per-thread global round trips.
// Geometry: stride 1, W and H multiples of 16; output and side input 16-byte aligned with 16-byte strides (TMA).
#include "fdx_tc.cuh"
#include "fdx_epilogue.cuh"

namespace {

constexpr int kThreads = 3 * 128;            // two consumer warpgroups + the producer warpgroup
constexpr int kWBytes = 64 * 128;            // weight tile: 64 channels x 64 k bf16
constexpr int kPixBytes = 2 * 128 * 128;     // two boxes of 128 pixels x 64 channels bf16
constexpr int kHaloBytes = 18 * 16 * 128;    // 16 x 18 pixel box
constexpr int kChunkBytes = 32 * 128;        // one epilogue chunk: 32 pixels x 64 channels bf16 (one TMA box)
// Chunk buffers per consumer warpgroup: the side input of a tile's first num_cbufs chunks is requested before
// its main loop and each later chunk's num_cbufs - 1 chunks ahead, so more buffers hide more of the HBM latency.
// The halo rings leave room for five; the five-stage per-tap ring for three.
__host__ __device__ constexpr int num_cbufs(bool halo) { return halo ? 5 : 3; }
__host__ __device__ constexpr int epi_bytes(bool halo) { return 2 * num_cbufs(halo) * kChunkBytes; }
static_assert((2 * 5 + 1 + 2 * 3) * 8 <= 256 && (2 * 3 + 1 + 2 * 5) * 8 <= 256, "tct: barrier area");

// RES (halo at K = 64 only): the nine weight tiles stay resident after the ring, so a stage is the pixel box alone
__host__ __device__ constexpr int stage_bytes(bool halo, bool res) {
  return halo ? (res ? 0 : 3 * kWBytes) + kHaloBytes : kWBytes + kPixBytes;
}
// halo: a fourth 60 KB (or, with RES, 36 KB) stage does not fit beside the chunk buffers
__host__ __device__ constexpr int num_stages(bool halo) { return halo ? 3 : 5; }
__host__ __device__ constexpr int wres_bytes(bool res) { return res ? 9 * kWBytes : 0; }
__host__ __device__ constexpr int ring_bytes(bool halo, bool res) {
  return num_stages(halo) * stage_bytes(halo, res) + wres_bytes(res);
}
// ring (+ resident weights), chunk buffers, barriers; 1024 = alignment slack of the dynamic base
__host__ __device__ constexpr int smem_bytes(bool halo, bool res) {
  return ring_bytes(halo, res) + epi_bytes(halo) + 1024 + 256;
}
// halo and RES: 180 + 40 + 1.25 = 221.25 KB; per-tap: 200 + 24 + 1.25 = 225.25 KB
static_assert(smem_bytes(true, false) <= 227 * 1024 && smem_bytes(true, true) <= 227 * 1024 &&
              smem_bytes(false, false) <= 227 * 1024, "tct: shared memory");
static_assert((num_stages(true) * stage_bytes(true, true)) % 1024 == 0, "tct: resident weights need 1024-byte alignment");
static_assert(ring_bytes(true, false) % 1024 == 0 && ring_bytes(true, true) % 1024 == 0 &&
              ring_bytes(false, false) % 1024 == 0, "tct: 128-byte-swizzled chunk buffers need 1024-byte alignment");

struct TctDev {
  int nxb, nyb, nimg, W, H;
  int ntaps, tap_dx[kTcMaxTaps], tap_dy[kTcMaxTaps], tap_b[kTcMaxTaps];
  int kchunks, K, Ncols, cblks, ntiles;
  float alpha;
  const float* bias;
  const float* rowvec;
  int has_res;             // a side input (mapR) is added, or is x of the fused GroupNorm backward
  float* cs_ws;            // fused per-(image, channel) sums or null
  int cs_slots, cs_ld;
  const float* gn_ab;      // GNB kernels: [N][2][Ncols] GroupNorm coefficients a, b of the tensor `res` (= x)
};

// Tile t = (pixel block t / cblks, column block t % cblks).  CTA b runs tiles b, b + grid, b + 2 grid, ...; with
// RES the grid is a multiple of cblks, so the column block (and the resident weights) of a CTA never changes.
struct TileCoord { int cb, nb, x0, y0; };

__device__ __forceinline__ TileCoord tile_coord(const TctDev& p, int tile) {
  const int mt = tile / p.cblks;
  return {tile % p.cblks, mt / (p.nxb * p.nyb), (mt % p.nxb) * 16, ((mt / p.nxb) % p.nyb) * 16};
}

// HALO = true (3x3 stride-1 only): with per-tap loads every (tap, K chunk) re-loads its 256 pixels, 40 KB of TMA
// per 2.1 MFLOP = 52 FLOP per byte, so the layers are L2 -> shared-memory bandwidth bound.  ONE tall box of
// 16 x 18 pixels (rows y0-1 .. y0+16) is loaded per (kx, K chunk); the three ky taps are 2048-byte row offsets
// into it (swizzle-aligned views, exactly as in the nine-tap weight gradient), so a stage carries three weight
// tiles + 36 KB of pixels and feeds twelve MMAs: 96 -> 36 KB of pixel traffic per three taps.
// GNB = true (HALO data gradient only): the first pass of the GroupNorm(+SiLU) backward in the epilogue - with x = the
// GroupNorm input (side input `res`) and z = a_c x + b_c the kernel stores dz = dy * silu'(z) instead of dy and
// accumulates S0 = sum dz, S1 = sum dz * x per (image, channel) into the column-sum workspace, exactly as the
// pixels-as-M engine's EPI_GN_BWD (fdx_epilogue.cuh).
// RES = true (HALO with one K chunk, K = 64): all nine 8 KB weight tiles of the CTA's column block are loaded
// once per CTA, on their own mbarrier, into 72 KB after the ring; a stage then carries only the 36 KB pixel box.
// Otherwise every tile re-fetched the same 72 KB of weights, 40 % of its 180 KB of L2 -> shared-memory traffic.
// The MMAs and their order (kx, ky, k16) are those of the plain HALO path, so the outputs are bit-identical.
template <bool A_MN, bool HALO, bool GNB, bool RES>
__global__ void __launch_bounds__(kThreads, 1)
fdx_tct_kernel(const __grid_constant__ CUtensorMap mapW, const __grid_constant__ CUtensorMap mapX,
               const __grid_constant__ CUtensorMap mapR, const __grid_constant__ CUtensorMap mapO,
               const __grid_constant__ TctDev p) {
  static_assert(HALO || !RES, "tct: resident weights need the halo stage");
  constexpr int kStageBytes = stage_bytes(HALO, RES);
  constexpr int S = num_stages(HALO);
  constexpr int kRingBytes = ring_bytes(HALO, RES);                // the ring, then the resident weights
  constexpr int kCBufs = num_cbufs(HALO);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* wres = smem + S * kStageBytes;                          // RES: tap t at t * kWBytes
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kRingBytes + epi_bytes(HALO));
  uint64_t* full = bars;
  uint64_t* empty = bars + S;
  uint64_t* wfull = bars + 2 * S;                                  // RES: the resident weights have landed
  uint64_t* cfull = bars + 2 * S + 1;                              // [2][kCBufs]: a chunk's side input has landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapW);
    tma_prefetch_desc(&mapX);
    tma_prefetch_desc(&mapO);
    if (p.has_res) tma_prefetch_desc(&mapR);
    for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 1); }
    if constexpr (RES) mbar_init(wfull, 1);
    for (int i = 0; i < 2 * kCBufs; ++i) mbar_init(&cfull[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  // stages per tile: HALO (kx, K chunk), taps t = ky * 3 + kx (fdx_conv3x3_fwd / dgrad fill order); else (tap, K chunk)
  const int nst = (HALO ? 3 : p.ntaps) * p.kchunks;

  // setmaxnreg sits inside each role's branch: issued before code both roles run, ptxas ignores it (C7507)
  if (warp >= 8) {
    producer_regs();
    if (warp == 8 && lane == 0) {
      // A_MN: HWIO rows = (tap, ci), co contiguous: box (64 co, 64 k rows); else (k = Cout contiguous,
      // rows = Cin, z1 = tap): box (64 k, 64 rows)
      auto load_w = [&](uint8_t* dst, uint64_t* bar, int cb, int t, int kc) {
        if constexpr (A_MN) tma_load_4d(dst, &mapW, bar, cb * 64, p.tap_b[t] + kc * 64, 0, 0);
        else tma_load_4d(dst, &mapW, bar, kc * 64, cb * 64, p.tap_b[t], 0);
      };
      if constexpr (RES) {
        mbar_arrive_expect_tx(wfull, 9 * kWBytes);
#pragma unroll
        for (int t = 0; t < 9; ++t) load_w(wres + t * kWBytes, wfull, tile_coord(p, blockIdx.x).cb, t, 0);
      }
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(p, tile);
        for (int q = 0; q < nst; ++q) {
          const int qt = q / p.kchunks, kc = q % p.kchunks;     // qt = kx (HALO) or the tap
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sw = smem + stage * kStageBytes;
          mbar_arrive_expect_tx(&full[stage], kStageBytes);
          if constexpr (HALO) {
            if constexpr (!RES) {
#pragma unroll
              for (int ky = 0; ky < 3; ++ky) load_w(sw + ky * kWBytes, &full[stage], tc.cb, ky * 3 + qt, kc);
            }
            tma_load_4d(sw + (RES ? 0 : 3 * kWBytes), &mapX, &full[stage], kc * 64, tc.x0 + qt - 1, tc.y0 - 1, tc.nb);
          } else {
            load_w(sw, &full[stage], tc.cb, qt, kc);
            uint8_t* sx = sw + kWBytes;
            tma_load_4d(sx, &mapX, &full[stage], kc * 64, tc.x0 + p.tap_dx[qt], tc.y0 + p.tap_dy[qt], tc.nb);
            tma_load_4d(sx + 16384, &mapX, &full[stage], kc * 64, tc.x0 + p.tap_dx[qt], tc.y0 + 8 + p.tap_dy[qt],
                        tc.nb);
          }
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    consumer_regs();
    // ============ consumers: warpgroup wg owns the CTA's local tiles wg, wg + 2, ... =========================
    // The epilogue works in the accumulator's own layout: lane l of warp q holds channel rows 16 q + l / 4 and
    // 16 q + l / 4 + 8 of the tile's 64, and pixel pairs 8 j + 2 (l % 4).  A lane always owns the same two
    // channels, so bias, timestep row and the fused GroupNorm sums are per-lane registers, reduced once per tile.
    const int q = warp & 3;
    const int wg = warp >> 2;
    const int t128 = threadIdx.x & 127;
    const bool wg_leader = t128 == 0;
    const int xbar = 1 + wg;                             // named barrier of this warpgroup's chunk buffers
    // MMA hand-off: a warpgroup waits on barrier 3 + wg before its main loop and, after issuing it, arrives on
    // the other's, so the two main loops never interleave on the tensor cores.  It is also what makes the ring's
    // parity waits sound: a warpgroup starts on its tile's stages only after the other has waited on all earlier
    // ones, so no full[] barrier is ever waited on more than one phase ahead (a parity wait one phase early
    // would pass at once, on a stage not yet loaded).
    const int my_turn = 3 + wg, their_turn = 4 - wg;
    const int crow = q * 16 + (lane >> 2);               // this lane's first channel row; the second is crow + 8
    float acc[128];
    // Side input and output move by TMA through the warpgroup's kCBufs chunk buffers.  Chunk c of a tile is
    // pixel rows 2 c, 2 c + 1 of its 16 x 16 block, 64 channels: one {64, 16, 2, 1} box, 128-byte swizzled, so
    // the eight 16-byte rows of one 8 x 8 ldmatrix / stmatrix matrix (8 pixels, one channel piece) fall in 8
    // different bank groups.  The warpgroup's n-th chunk (8 per tile) uses buffer n % kCBufs and barrier phase
    // n / kCBufs.  The side input arrives in the buffer, each warp reads its 16 channels of it into accumulator
    // layout (ldmatrix.trans), overwrites them with its output (stmatrix.trans), and one store sends the buffer
    // back.  The leader thread issues all of it: bulk async-groups are per thread, so only the
    // thread that committed a buffer's store can tell when its buffer may be refilled.  Side input and output
    // are touched once and carry the evict-first L2 policy, so they do not push out the pixel boxes that
    // neighbouring tiles still read.
    uint8_t* cbuf = smem + kRingBytes + wg * kCBufs * kChunkBytes;
    uint64_t* wg_cfull = cfull + wg * kCBufs;
    auto load_chunk = [&](const TileCoord& c, int ci, int n) {
      uint64_t* bar = &wg_cfull[n % kCBufs];
      mbar_arrive_expect_tx(bar, kChunkBytes);
      tma_load_4d_hint(cbuf + (n % kCBufs) * kChunkBytes, &mapR, bar, c.cb * 64, c.x0, c.y0 + 2 * ci, c.nb,
                       l2_evict_first_policy());
    };
    auto store_chunk = [&](const TileCoord& c, int ci, int n) {
      tma_store_4d_hint(&mapO, cbuf + (n % kCBufs) * kChunkBytes, c.cb * 64, c.x0, c.y0 + 2 * ci, c.nb,
                        l2_evict_first_policy());
      bulk_commit_group();
    };
    // every CTA has at least one tile, so the producer always issues the resident weights' loads
    if constexpr (RES) mbar_wait(wfull, 0);
    const uint32_t wres_u32 = smem_u32(wres);
    for (int i = wg, tile = blockIdx.x + wg * gridDim.x; tile < p.ntiles; i += 2, tile += 2 * gridDim.x) {
      const TileCoord tc = tile_coord(p, tile);
      const int nb = tc.nb;
      const int n0 = (i >> 1) * 8;                         // the warpgroup's chunk count before this tile
      // the side input of the first kCBufs chunks, requested before the main loop so that it has the main
      // loop (and the wait for the tensor cores) to arrive from HBM; their buffers are free once the previous
      // tile's stores have read them
      if (p.has_res && wg_leader) {
        bulk_wait_group_read<0>();
#pragma unroll
        for (int c = 0; c < kCBufs; ++c) load_chunk(tc, c, n0 + c);
      }
      const int ch = tc.cb * 64 + crow;                    // this lane's channels: ch and ch + 8
      float add[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        add[h] = 0.f;
        if constexpr (!GNB) {   // GNB launches have neither (fdx_tct_launch): the zeros then hold no registers
          if (p.bias) add[h] += __ldg(p.bias + ch + 8 * h);
          if (p.rowvec) add[h] += __ldg(p.rowvec + (long long)nb * p.Ncols + ch + 8 * h);
        }
      }
      float ga[2], gb[2];
      if constexpr (GNB) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          ga[h] = __ldg(p.gn_ab + (long long)nb * 2 * p.Ncols + ch + 8 * h);
          gb[h] = __ldg(p.gn_ab + ((long long)nb * 2 + 1) * p.Ncols + ch + 8 * h);
        }
      }
      // ---- main loop: the ring holds the CTA's tiles in order; this tile's stages start at i * nst ----
      int stage = (i * nst) % S;
      uint32_t phase = ((i * nst) / S) & 1;
#pragma unroll
      for (int j = 0; j < 128; ++j) acc[j] = 0.f;
      if (i > 0) named_bar_sync(my_turn, 256);
      int prev = -1;
      for (int kq = 0; kq < nst; ++kq) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint32_t sw = smem_u32(smem + stage * kStageBytes);
        // HALO: the 16 x 18 box; per-tap: two 16 x 8 boxes
        const uint32_t sx = sw + (HALO ? (RES ? 0 : 3) : 1) * kWBytes;
        // weight tile of (ky, this stage): RES, tap ky * 3 + kx of the resident set (kq = kx); else ky of the stage
        const uint32_t wb = RES ? wres_u32 + kq * kWBytes : sw;
#pragma unroll
        for (int ky = 0; ky < (HALO ? 3 : 1); ++ky) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t wt = wb + ky * (RES ? 3 : 1) * kWBytes;
            const uint32_t aw = A_MN ? wt + k * 2048 : wt + k * 32;
            const uint64_t db = gmma_desc_sw128(sx + ky * 2048 + k * 32, 16, 1024);   // HALO: rows ky .. ky+15
            const uint64_t da = A_MN ? gmma_desc_sw128(aw, 8192, 1024) : gmma_desc_sw128(aw, 16, 1024);
            wgmma_m64n256k16<A_MN ? 1 : 0, 0>(acc, da, db);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && wg_leader) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      if (tile + gridDim.x < p.ntiles) named_bar_arrive(their_turn, 256);   // the other warpgroup's next tile
      wgmma_wait<0>();
      if (wg_leader) mbar_arrive(&empty[prev]);

      // the tile's coordinates again: kept in registers across the main loop, they make the GroupNorm-backward
      // variants spill
      const TileCoord ec = tile_coord(p, tile);
      float s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f};
      // ldmatrix / stmatrix address of this lane: row l % 8 of matrix l / 8 = (8-pixel group 2 hp + l / 16,
      // channel half (l / 8) % 2), i.e. box row 8 (l / 16) + l % 8 of the half chunk hp and the 16-byte unit of
      // channels 16 q + 8 ((l / 8) % 2) .. + 7, under the 128-byte swizzle (unit u -> u ^ (row % 8))
      const uint32_t lane_off =
          ((lane >> 4) * 8 + (lane & 7)) * 128 + (((2 * q + ((lane >> 3) & 1)) ^ (lane & 7)) << 4);
      // Unrolled: the chunk index is a compile-time register index, and the 16 accumulator registers of a
      // chunk die once it is written out.
#pragma unroll
      for (int ci = 0; ci < 8; ++ci) {
        const int n = n0 + ci;
        const uint32_t cb = smem_u32(cbuf + (n % kCBufs) * kChunkBytes);
        if (ci > 0) {
          named_bar_sync(xbar, 128);                     // every warp has written and fenced chunk ci - 1
          if (wg_leader) store_chunk(ec, ci - 1, n - 1);
        }
        if (p.has_res) mbar_wait(&wg_cfull[n % kCBufs], (n / kCBufs) & 1);
        // columns 32 ci .. 32 ci + 31 = pixel rows 2 ci, 2 ci + 1; half hp = 8-pixel groups 2 hp, 2 hp + 1
#pragma unroll
        for (int hp = 0; hp < 2; ++hp) {
          const uint32_t addr = cb + hp * 16 * 128 + lane_off;
          uint32_t r[4];
          if (p.has_res) ldmatrix_x4_trans(addr, r);
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const int h = m & 1;                           // channel row crow + 8 h
            const float* d = &acc[(ci * 4 + 2 * hp + (m >> 1)) * 4 + 2 * h];
            float f[2] = {d[0] * p.alpha + add[h], d[1] * p.alpha + add[h]};
            float xv[2];
            if (p.has_res) {
              const float2 x2 = unpack_bf16x2(r[m]);
              xv[0] = x2.x; xv[1] = x2.y;
              if constexpr (GNB) {
#pragma unroll
                for (int e = 0; e < 2; ++e) f[e] = epi_silu_grad_times(f[e], fmaf(xv[e], ga[h], gb[h]));
              } else {
#pragma unroll
                for (int e = 0; e < 2; ++e) f[e] += xv[e];
              }
            }
            r[m] = pack_bf16x2(f[0], f[1]);
            if (p.cs_ws) {
              const float2 hv = unpack_bf16x2(r[m]);
              // second factor: the GroupNorm input x (GNB) or the stored value itself (forward column statistics)
              s0[h] += hv.x; s1[h] = fmaf(hv.x, GNB ? xv[0] : hv.x, s1[h]);
              s0[h] += hv.y; s1[h] = fmaf(hv.y, GNB ? xv[1] : hv.y, s1[h]);
            }
          }
          stmatrix_x4_trans(addr, r);                      // the rows ldmatrix read: each warp owns its channels
        }
        fence_proxy_async_smem();                        // the buffer's new contents, visible to the TMA store
        if (wg_leader) {
          if (p.has_res) {
            // refill the buffer of chunk ci - 1, whose store was issued at the top of this chunk: the side input
            // of chunk ci + kCBufs - 1, kCBufs - 1 chunks before it is needed
            if (ci > 0 && ci + kCBufs - 1 < 8) {
              bulk_wait_group_read<0>();
              load_chunk(ec, ci + kCBufs - 1, n + kCBufs - 1);
            }
          } else {
            bulk_wait_group_read<kCBufs - 2>();          // chunk n + 1's buffer has been read by its last store
          }
        }
      }
      named_bar_sync(xbar, 128);
      if (wg_leader) store_chunk(ec, 7, n0 + 7);
      if (p.cs_ws) {
        // the four lanes of a quad hold the same two channels: combine them
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int o = 1; o < 4; o <<= 1) {
            s0[h] += __shfl_xor_sync(0xffffffffu, s0[h], o);
            s1[h] += __shfl_xor_sync(0xffffffffu, s1[h], o);
          }
        }
        if ((lane & 3) == 0) {
          float* w = p.cs_ws + (((long long)(tile % p.cs_slots) * p.nimg + ec.nb) * 2) * p.cs_ld + ec.cb * 64 + crow;
#pragma unroll
          for (int h = 0; h < 2; ++h) { atomicAdd(w + 8 * h, s0[h]); atomicAdd(w + p.cs_ld + 8 * h, s1[h]); }
        }
      }
    }
    if (wg_leader) bulk_wait_group<0>();                 // every output store has completed
  }
}

// weights, pixels (the A operand), side input (unset without one) and output
struct TctMaps { CUtensorMap w, x, r, o; };

template <bool A_MN, bool HALO, bool GNB, bool RES>
int launch_tct_grid(const TctMaps& m, const TctDev& d, cudaStream_t stream) {
  constexpr int smem = smem_bytes(HALO, RES);
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(fdx_tct_kernel<A_MN, HALO, GNB, RES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  smem));
    attr_set = true;
  }
  int grid = fdx_num_sms();
  if (grid <= 0) return FDX_ERR_NO_DEVICE;
  // RES: a whole number of column-block groups, so each CTA keeps one column block (tile_coord); ntiles is a
  // multiple of cblks, so the clamp below keeps that.
  if (RES) grid = (grid >= d.cblks ? grid / d.cblks : 1) * d.cblks;
  if (d.ntiles < grid) grid = d.ntiles;
  fdx_tct_kernel<A_MN, HALO, GNB, RES><<<grid, kThreads, smem, stream>>>(m.w, m.x, m.r, m.o, d);
  fdx_note_kernel(FDX_KERNEL_TCT);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

// Halo launches with one K chunk keep their weights resident (RES); at K >= 128 the nine taps (147 KB and more)
// do not fit beside the ring.  RES needs a grid of whole column-block groups; where that would leave SMs idle
// (cblks = 5 on 132 SMs: 130 CTAs) the plain halo launch is the faster one, by about 1 % on an H100 SXM.
template <bool A_MN, bool HALO, bool GNB = false>
int launch_tct(const TctMaps& m, const TctDev& d, cudaStream_t stream) {
  if constexpr (HALO) {
    const int sms = fdx_num_sms();
    if (d.kchunks == 1 && std::min(d.ntiles, sms / d.cblks * d.cblks) == std::min(d.ntiles, sms))
      return launch_tct_grid<A_MN, true, GNB, true>(m, d, stream);
  }
  return launch_tct_grid<A_MN, HALO, GNB, false>(m, d, stream);
}

// TMA needs a 16-byte-aligned base and strides that are multiples of 16 bytes
bool tma_view_ok(const void* base, long long sx, long long sy, long long sn) {
  return reinterpret_cast<uintptr_t>(base) % 16 == 0 && sx % 8 == 0 && sy % 8 == 0 && sn % 8 == 0;
}

// the epilogue's TMA view of the output or side input: (channel, x, y, image), one chunk box {64, 16, 2, 1}
int make_chunk_map(CUtensorMap* map, const void* base, const TcLaunch& L, long long sx, long long sy,
                   long long sn) {
  const uint64_t dims[4] = {(uint64_t)L.Ncols, (uint64_t)L.W, (uint64_t)L.H, (uint64_t)L.N};
  const uint64_t str[3] = {(uint64_t)sx * 2, (uint64_t)sy * 2, (uint64_t)sn * 2};
  const uint32_t box[4] = {64, 16, 2, 1};
  const uint32_t est[4] = {1, 1, 1, 1};
  return fdx_make_tmap_bf16(map, base, 4, dims, str, box, est, 1);
}

}  // namespace

// FDX_ERR_UNSUPPORTED (no error text) = geometry not covered; the caller uses the generic engine.
int fdx_tct_launch(const TcLaunch& L, cudaStream_t stream) {
  if (L.mode == TC_MNMN || L.gemm_like || L.es != 1 || L.out_f32 || L.out_atomic || L.b_batched)
    return FDX_ERR_UNSUPPORTED;
  // halo-sharing variant: standard 3x3 stride-1 tap set in (ky, kx) order
  bool halo = L.ntaps == 9;
  for (int t = 0; t < 9 && halo; ++t) halo = (L.tap_dx[t] == t % 3 - 1) && (L.tap_dy[t] == t / 3 - 1);
  // fused GroupNorm-backward first pass: halo data gradient with x as the side input and the sums workspace
  if (L.gn_ab && (!halo || L.mode != TC_KK || !L.res || !L.gn_ws || L.bias || L.rowvec)) return FDX_ERR_UNSUPPORTED;
  // column counts the generic engine would have to cover with N < 256 tiles (64, 128, 192, 320, 384, ...)
  if (L.Ncols % 64 != 0 || L.Ncols % 256 == 0 || L.Ncols > 512) return FDX_ERR_UNSUPPORTED;
  if (L.W % 16 != 0 || L.H % 16 != 0 || L.K % 64 != 0) return FDX_ERR_UNSUPPORTED;
  // the epilogue moves output and side input by TMA
  if (!tma_view_ok(L.out, L.os_x, L.os_y, L.os_n) || (L.res && !tma_view_ok(L.res, L.rs_x, L.rs_y, L.rs_n)))
    return FDX_ERR_UNSUPPORTED;
  TctDev d{};
  d.W = L.W; d.H = L.H; d.nimg = L.N;
  d.nxb = L.W / 16; d.nyb = L.H / 16;
  d.ntaps = L.ntaps;
  for (int i = 0; i < kTcMaxTaps; ++i) { d.tap_dx[i] = L.tap_dx[i]; d.tap_dy[i] = L.tap_dy[i]; d.tap_b[i] = L.tap_b[i]; }
  d.K = L.K; d.kchunks = L.K / 64; d.Ncols = L.Ncols;
  d.cblks = L.Ncols / 64;
  d.ntiles = d.cblks * d.nxb * d.nyb * d.nimg;
  d.alpha = L.alpha; d.bias = L.bias; d.rowvec = L.rowvec;
  d.has_res = L.res != nullptr;
  d.cs_ws = L.gn_ws; d.cs_slots = L.gn_slots > 0 ? L.gn_slots : 1; d.cs_ld = L.ws_ld > 0 ? L.ws_ld : L.Ncols;
  d.gn_ab = L.gn_ab;

  TctMaps m{};
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.A.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.A.strides[i] * 2;
    uint32_t box[4] = {64, 16, (uint32_t)(halo ? 18 : 8), 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&m.x, L.A.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.B.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.B.strides[i] * 2;
    uint32_t box[4] = {64, 64, 1, 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&m.w, L.B.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  int s = make_chunk_map(&m.o, L.out, L, L.os_x, L.os_y, L.os_n);
  if (s != FDX_OK) return s;
  if (L.res && (s = make_chunk_map(&m.r, L.res, L, L.rs_x, L.rs_y, L.rs_n)) != FDX_OK) return s;
  if (L.mode == TC_KMN) return halo ? launch_tct<true, true>(m, d, stream) : launch_tct<true, false>(m, d, stream);
  if (L.gn_ab) return launch_tct<false, true, true>(m, d, stream);   // fused GroupNorm backward
  return halo ? launch_tct<false, true>(m, d, stream) : launch_tct<false, false>(m, d, stream);
}
