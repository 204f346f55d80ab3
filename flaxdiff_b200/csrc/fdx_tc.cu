// fdx_tc.cu -- the wgmma / TMA "tap-GEMM" engine for sm_90a.
//
// Replaces what the reference delegates to XLA for every dense contraction on the
// UNet hot path: flax nn.Conv 3x3 / 1x1 (flaxdiff/models/common.py:166-172,
// 237-244, 324-333), nn.DenseGeneral projections (models/attention.py:132-154)
// and the QK^T / PV products of nn.dot_product_attention (attention.py:170-174),
// forward and backward.
//
// Design (one CTA per SM, persistent over 128 x BN output tiles):
//   last WG     TMA producer (one thread): per K-chunk one 128B-swizzled A box (64 channels x
//               128 pixels, shifted by the tap offset; out-of-image = zero fill
//               = SAME padding) and the matching B box, into a ring of stages.
//   warpgroups  consumers (one per 128 output columns): wgmma m64 x {64,128} x 16
//               (bf16 -> f32 registers) over all 128 rows, release each stage once
//               its MMAs retire, then run the epilogue on their own columns: fuse
//               bias + per-image timestep vector + residual, store bf16/f32 (or f32
//               atomics for the split-K weight gradient).
#include "fdx_tc_kernel.cuh"

namespace {

template <int BN, int MODE, int EPI>
int launch_cfg(const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d, cudaStream_t stream) {
  using Cfg = TcCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(fdx_tc_kernel<BN, MODE, EPI>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  int grid = fdx_num_sms();
  if (grid <= 0) return FDX_ERR_NO_DEVICE;
  if (d.ntiles < grid) grid = d.ntiles;
  fdx_tc_kernel<BN, MODE, EPI><<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mA, mB, d);
  fdx_note_kernel(FDX_KERNEL_TC);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

template <int BN, int MODE>
int launch_gn(const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d, cudaStream_t stream) {
  if constexpr (MODE == TC_KK) {
    if (d.gn_ab) return launch_cfg<BN, MODE, EPI_GN_BWD>(mA, mB, d, stream);
  }
  if constexpr (MODE == TC_KMN) {
    if (d.gn_ws && !d.gn_ab) return launch_cfg<BN, MODE, EPI_COLSTATS>(mA, mB, d, stream);
  }
  return launch_cfg<BN, MODE, EPI_PLAIN>(mA, mB, d, stream);
}

template <int MODE>
int launch_mode(int BN, const CUtensorMap& mA, const CUtensorMap& mB, const TcDev& d,
                cudaStream_t stream) {
  switch (BN) {
    case 64: return launch_gn<64, MODE>(mA, mB, d, stream);
    case 128: return launch_gn<128, MODE>(mA, mB, d, stream);
    case 256: return launch_gn<256, MODE>(mA, mB, d, stream);
  }
  fdx_set_error("tc: unsupported BN %d", BN);
  return FDX_ERR_UNSUPPORTED;
}

int pow2_floor(int v) {
  int p = 1;
  while (p * 2 <= v) p *= 2;
  return p;
}

}  // namespace

int fdx_tc_launch(const TcLaunch& L, cudaStream_t stream) {
  FDX_REQUIRE(L.mode >= TC_KK && L.mode <= TC_MNMN, "tc: bad mode %d", L.mode);
  FDX_REQUIRE(L.ntaps >= 1 && L.ntaps <= kTcMaxTaps, "tc: bad ntaps %d", L.ntaps);
  FDX_REQUIRE(L.es == 1 || L.es == 2, "tc: bad element stride %d", L.es);
  FDX_REQUIRE(L.Ncols > 0 && L.Ncols % 32 == 0, "tc: Ncols=%d must be a multiple of 32", L.Ncols);
  FDX_REQUIRE(L.A.strides[0] == 1 && L.B.strides[0] == 1, "tc: innermost strides must be 1");
  const bool cat = L.A1.ptr != nullptr;
  FDX_REQUIRE(!cat || (L.gemm_like && L.mode != TC_MNMN && L.ntaps == 1 && L.cat_k0 > 0 && L.cat_k0 % kBK == 0 &&
                       L.cat_k0 < L.K && L.A1.strides[0] == 1 && !L.gn_ab && !L.gn_ws),
              "tc: a two-source A needs a one-tap K-major GEMM with 0 < K0 < K, K0 a multiple of %d", kBK);

  // Few output columns (Ncols = 64 / 128): the transposed formulation (fdx_tct.cu) issues M x 256 x 16 MMAs
  // instead of 128 x Ncols x 16 ones; faster on every such layer (profiles/layers_r01_tct.txt).
  if (L.mode != TC_MNMN) {
    const int rt = fdx_tct_launch(L, stream);
    if (rt != FDX_ERR_UNSUPPORTED) return rt;
  }
  TcDev d{};
  d.mode = L.mode;
  d.W = L.W; d.H = L.H; d.N = L.N; d.es = L.es; d.ntaps = L.ntaps;
  d.es_b = L.es_b > 1 ? L.es_b : 1;
  FDX_REQUIRE(d.es_b <= 2, "tc: bad B element stride %d", L.es_b);
  bool b_view = d.es_b != 1;
  for (int i = 0; i < kTcMaxTaps; ++i) {
    d.tap_dx[i] = L.tap_dx[i]; d.tap_dy[i] = L.tap_dy[i]; d.tap_b[i] = L.tap_b[i];
    d.tap_bdx[i] = L.tap_bdx[i]; d.tap_bdy[i] = L.tap_bdy[i];
    b_view = b_view || L.tap_bdx[i] != 0 || L.tap_bdy[i] != 0;
  }
  FDX_REQUIRE(!b_view || L.mode == TC_MNMN, "tc: strided / shifted B views exist only in TC_MNMN");
  d.K = L.K; d.M = L.M; d.Ncols = L.Ncols; d.b_batched = L.b_batched; d.mn_batched = L.mn_batched;
  d.out = L.out; d.out_f32 = L.out_f32; d.out_atomic = L.out_atomic;
  d.os_x = L.os_x; d.os_y = L.os_y; d.os_n = L.os_n; d.os_tap = L.os_tap; d.os_m = L.os_m;
  d.alpha = L.alpha; d.bias = L.bias; d.rowvec = L.rowvec; d.res = L.res;
  d.rs_x = L.rs_x; d.rs_y = L.rs_y; d.rs_n = L.rs_n;
  d.gn_ab = L.gn_ab; d.gn_ws = L.gn_ws; d.gn_slots = L.gn_slots > 0 ? L.gn_slots : 1;
  d.ws_ld = L.ws_ld > 0 ? L.ws_ld : L.Ncols;
  d.cat_kc = L.cat_k0 / kBK;
  if (L.out_f32) {
    // float4 stores and 16-byte vector reductions
    FDX_REQUIRE(reinterpret_cast<uintptr_t>(L.out) % 16 == 0 && L.os_x % 4 == 0 && L.os_y % 4 == 0 &&
                    L.os_n % 4 == 0 && L.os_tap % 4 == 0 && L.os_m % 4 == 0,
                "tc: f32 output must be 16-byte aligned with strides that are multiples of 4");
  }
  if (L.gn_ws && !L.gn_ab) {
    FDX_REQUIRE(L.mode == TC_KMN && !L.gemm_like && !L.out_f32 && !L.out_atomic,
                "tc: output column statistics need a bf16 convolution-forward launch");
  }
  if (L.gn_ab) {
    FDX_REQUIRE(L.mode == TC_KK && !L.gemm_like && L.res && L.gn_ws && !L.out_f32 && !L.out_atomic &&
                    !L.bias && !L.rowvec,
                "tc: GroupNorm-backward fusion needs a plain bf16 data-gradient launch");
  }

  // ---- column tile --------------------------------------------------------
  // cost model per row tile: ntiles * (BN + 64)  (MMA columns incl. padding + A re-read per tile)
  int BN = 64;
  {
    long long best = -1;
    const int cands[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
      const int bn = cands[i];
      const long long nt = (L.Ncols + bn - 1) / bn;
      const long long cost = nt * (bn + 64);
      if (best < 0 || cost < best) { best = cost; BN = bn; }
    }
  }
  const int rows_per_tile = (L.mode == TC_MNMN) ? 64 : 128;
  // ---- pixel box ----------------------------------------------------------
  int TW, TH, TN;
  if (!L.gemm_like) {
    // conv: a 16 x 8 (or 16 x 4) pixel patch; small images pack several per tile.  Not under per-image column
    // sums, whose epilogue adds all rows of a tile into one image's sums: there the box is one image deep
    // (TN = 1) and as tall as it takes, its rows below the image zero-filled by TMA and invalid in the epilogue.
    // Where the packed box already has TN = 1 both rules give the same box.
    TW = pow2_floor(L.W < 16 ? L.W : 16);
    int rem = rows_per_tile / TW;
    TH = L.gn_ws ? rem : pow2_floor(L.H < rem ? L.H : rem);
    TN = rem / TH;
  } else {
    // GEMM: rows along x only; (y, n) are batch coordinates. A box taller than the
    // matrix is fine: TMA zero-fills and the epilogue predicates on x < W.
    TW = rows_per_tile;
    TH = 1;
    TN = 1;
  }
  d.TW = TW; d.TH = TH; d.TN = TN;
  if (L.mode != TC_MNMN && !L.out_f32 && !L.out_atomic) {
    // the bf16 epilogue holds each row's offsets as 32-bit distances from the tile's first row
    auto span = [&](long long sx, long long sy, long long sn) {
      return (TW - 1) * llabs(sx) + (TH - 1) * llabs(sy) + (TN - 1) * llabs(sn);
    };
    FDX_REQUIRE(span(L.os_x, L.os_y, L.os_n) < (1LL << 31) && span(L.rs_x, L.rs_y, L.rs_n) < (1LL << 31),
                "tc: the rows of one output tile span 2^31 elements or more");
  }
  d.nxb = (L.W + TW - 1) / TW;
  d.nyb = (L.H + TH - 1) / TH;
  d.nnb = (L.N + TN - 1) / TN;
  const long long pix_blocks = (long long)d.nxb * d.nyb * d.nnb;

  if (L.mode != TC_MNMN) {
    d.nblks = (L.Ncols + BN - 1) / BN;
    d.kchunks = (L.K + kBK - 1) / kBK;
    d.ntiles = (int)(pix_blocks * d.nblks);
    d.splits = 1;
    d.mblks = 1;
    d.tpp = 1;
    d.ntp = L.ntaps;
    FDX_REQUIRE(!L.res || !L.out_atomic, "tc: residual with atomic output unsupported");
  } else {
    d.nblks = (L.Ncols + BN - 1) / BN;
    d.tpp = (L.M <= 64 && L.ntaps > 1 && !b_view) ? 2 : 1;
    d.ntp = (L.ntaps + d.tpp - 1) / d.tpp;
    d.mblks = (L.M + 127) / 128;
    d.kchunks = 0;
    long long base_tiles = (long long)d.ntp * d.mblks * d.nblks;
    const long long kblocks = L.mn_batched ? d.nxb : pix_blocks;
    const long long nbz = L.mn_batched ? (long long)d.nyb * d.nnb : 1;
    int splits = L.splits;
    if (splits <= 0) {
      // wave-aware split-K: pick the split count whose tile total fills w waves of the machine
      // best (w = 1..4); more waves only when they raise the fill by > 3 %.
      const int sms = fdx_num_sms();
      const long long bt = base_tiles * nbz;
      double best_eff = -1.0;
      splits = 1;
      for (int w = 1; w <= 4; ++w) {
        long long sp = ((long long)sms * w) / bt;
        if (sp < 1) sp = 1;
        if (sp > kblocks) sp = kblocks;
        const long long tiles = bt * sp;
        const long long waves = (tiles + sms - 1) / sms;
        const double eff = (double)tiles / (double)(waves * sms);
        if (eff > best_eff + 0.03) { best_eff = eff; splits = (int)sp; }
      }
    }
    if (splits > kblocks) splits = (int)kblocks;
    FDX_REQUIRE(splits == 1 || L.out_atomic, "tc: split-K needs atomic output");
    d.splits = splits;
    d.ntiles = (int)(base_tiles * splits * nbz);
  }

  // ---- tensor maps ----------------------------------------------------------
  CUtensorMap mA, mB;
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.A.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.A.strides[i] * 2;
    uint32_t box[4] = {64, (uint32_t)(TW * L.es), (uint32_t)(TH * L.es), (uint32_t)TN};
    uint32_t est[4] = {1, (uint32_t)L.es, (uint32_t)L.es, 1};
    int s = fdx_make_tmap_bf16(&mA, L.A.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }
  {
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.B.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.B.strides[i] * 2;
    uint32_t box[4];
    uint32_t est[4] = {1, 1, 1, 1};
    if (L.mode == TC_KK) {
      box[0] = 64; box[1] = (uint32_t)BN; box[2] = 1; box[3] = 1;
    } else if (L.mode == TC_KMN) {
      box[0] = 64; box[1] = 64; box[2] = 1; box[3] = 1;
    } else {
      box[0] = 64; box[1] = (uint32_t)(TW * d.es_b); box[2] = (uint32_t)(TH * d.es_b); box[3] = (uint32_t)TN;
      est[1] = est[2] = (uint32_t)d.es_b;
    }
    int s = fdx_make_tmap_bf16(&mB, L.B.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
  }

  if (cat) {
    CUtensorMap mA1;
    uint64_t dims[4], str[3];
    for (int i = 0; i < 4; ++i) dims[i] = L.A1.dims[i];
    for (int i = 1; i < 4; ++i) str[i - 1] = L.A1.strides[i] * 2;
    uint32_t box[4] = {64, (uint32_t)TW, 1, 1};
    uint32_t est[4] = {1, 1, 1, 1};
    int s = fdx_make_tmap_bf16(&mA1, L.A1.ptr, 4, dims, str, box, est, 1);
    if (s != FDX_OK) return s;
    return fdx_tc_cat_launch(BN, L.mode, mA, mB, mA1, d, stream);
  }
  switch (L.mode) {
    case TC_KK: return launch_mode<TC_KK>(BN, mA, mB, d, stream);
    case TC_KMN: return launch_mode<TC_KMN>(BN, mA, mB, d, stream);
    default: return launch_mode<TC_MNMN>(BN, mA, mB, d, stream);
  }
}
