"""The convolutions' fused GroupNorm column sums compared element by element with float64: fdx_conv3x3_fwd_stats and
fdx_upconv3x3_fwd_stats, through every route they take, and the GroupNorm kernels that read those sums
(fdx_groupnorm_stats_from_cols, fdx_groupnorm_apply_cols), at the UNet's own layers (C2's 256-image batch, C3's
256 x 256 level), on images whose tiles are partial, and on the 12- to 15-pixel-wide images that need a one-image
pixel box.

The reference of the sums is the per-(image, channel) sum and sum of squares of the bf16 output the kernel stored,
read back: it does not depend on how the convolution rounds.  Every case runs twice:
  * dense: random operands; the sums are checked against gamma(D) times their sum of |terms|, D the chain of f32
    additions of elementwise_ref.colstats_depth (the worst |err| / bound is printed as `WORST <case> <ratio>`);
  * exact: integer operands with weights sparse enough that every sum of |terms| stays below 2^24, which the case
    asserts.  Then every summation order is exact and the workspace must equal the float64 sums bit for bit: this
    is what sees a dropped or doubled tile among 10^6 pixels.
The workspace starts from a random prior that the sums add onto (the upsample's four parity launches rely on that),
has one slot more than its descriptor names and channels on both sides of the output's slot; all of that must come
back unchanged.  The output is a channel slot of a wider buffer, NaN-prefilled, and must be bit-identical to the same
convolution without sums.  Each case id names its route, restated from the launch code, and the case asserts the
kind of the kernel that ran last."""
import math

import pytest
import torch

import elementwise_ref as R
import mish_ref as M
from flaxdiff_b200 import _lib, ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
SENTINEL = -1234.0                                   # exactly representable in bf16
KIND = {"tc": 0, "tct": 1}                           # FDX_KERNEL_TC / TCT
KINDS = ("dense", "exact")
# The ids name the route for this device's SM count; without a device the cases are only collected (and
# skipped), named for a 132-SM H100 SXM.
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def report(name, frac):
    print(f"WORST {name} {frac:.3f}")


def assert_route(route):
    kind = _lib.load().fdx_last_kernel_kind()
    assert kind == KIND[route.split("-")[0]], (route, kind)


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


# ----------------------------------------------------------------------------------------------- operands
def draw(shape, kind, g, dtype=torch.bfloat16):
    """dense: N(0, 1); exact: integers in {-2..2}."""
    if kind == "exact":
        return torch.randint(-2, 3, tuple(shape), generator=g, device=dev).to(dtype)
    return torch.randn(tuple(shape), generator=g, device=dev).to(dtype)


def weights(shape, kind, g, fan_in, pixels, dtype=torch.bfloat16):
    """dense: N(0, 1 / fan_in); exact: +-1 on a random fraction of the taps, 0 elsewhere, so sparse that with x in
    {-2..2} (E x^2 = 2) the expected sum of y^2 over `pixels` outputs is 2^18, 64 times below 2^24."""
    if kind == "dense":
        return (torch.randn(tuple(shape), generator=g, device=dev) / math.sqrt(fan_in)).to(dtype)
    density = min(1.0, 2.0 ** 18 / pixels / (2 * fan_in))
    keep = torch.rand(tuple(shape), generator=g, device=dev) < density
    sign = torch.randint(0, 2, tuple(shape), generator=g, device=dev) * 2 - 1
    return (keep * sign).to(dtype)


def epilogue_inputs(epi, kind, g, N, Ho, Wo, Co):
    """bias [Co] f32, rowvec [N][Co] f32 (conv1's timestep row) and res (conv2's residual), each when named."""
    bias = draw((Co,), kind, g, torch.float32) if "bias" in epi else None
    rowvec = draw((N, Co), kind, g, torch.float32) if "rowvec" in epi else None
    res = draw((N, Ho, Wo, Co), kind, g) if "res" in epi.split("+") else None
    return bias, rowvec, res


def out_slot(N, H, W, C, coff, ld):
    """Channels [coff, coff + C) of an (N, H, W, ld) bf16 buffer: the slot NaN, its neighbours SENTINEL."""
    buf = torch.full((N, H, W, ld), SENTINEL, dtype=torch.bfloat16, device=dev)
    y = buf[..., coff:coff + C]
    y.fill_(math.nan)
    return buf, y


def workspace(kind, g, N, ld, slots):
    """A ColStats whose descriptor names `slots` slots of an f32 [slots + 1][N][2][ld] tensor holding a random prior
    (exact: integers in -16..16) -> (ColStats, the whole tensor, a copy of the prior)."""
    if kind == "exact":
        full = torch.randint(-16, 17, (slots + 1, N, 2, ld), generator=g, device=dev).float()
    else:
        full = 8 * torch.randn((slots + 1, N, 2, ld), generator=g, device=dev)
    cs = ops.ColStats(N, ld, dev, slots)
    cs.ws = full[:slots]
    return cs, full, full.clone()


def check_sums(kind, what, full, prior, slots, coff, y, depth):
    """The workspace against the float64 sums of the stored y on top of the prior; everything outside the slots
    and channels the descriptor names is unchanged."""
    C = y.shape[-1]
    outside = torch.cat([full[:slots, ..., :coff], full[:slots, ..., coff + C:]], -1)
    outside_prior = torch.cat([prior[:slots, ..., :coff], prior[:slots, ..., coff + C:]], -1)
    assert torch.equal(outside.view(torch.int32), outside_prior.view(torch.int32)), \
        f"{what}: the sums reached channels outside the output's slot"
    assert torch.equal(full[slots:].view(torch.int32), prior[slots:].view(torch.int32)), \
        f"{what}: the sums reached a slot the descriptor does not name"
    assert torch.isfinite(y).all(), f"{what}: output elements left unwritten"
    val, mag = R.colstats_ref(y, prior[:slots, ..., coff:coff + C])
    got = full[:slots, ..., coff:coff + C].to(F64).sum(0)           # exact in float64: what the consumers add up
    if kind == "exact":
        assert R.exact_case_ok(mag), f"{what}: the exact case's sums reach 2^24"
        bad = got != val
        if bad.any():
            i = tuple(int(j) for j in torch.nonzero(bad)[0])
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} sums differ from the exact result; "
                                 f"first at (image, sum, channel) {i}: got {got[i].item()!r}, exact {val[i].item()!r}")
        return
    report(what, R.assert_elementwise(got, val, R.f32_bound(val, R.gamma(depth) * mag), what))


def assert_same_output(what, y, y_plain):
    assert torch.equal(y.contiguous().view(torch.int16), y_plain.view(torch.int16)), \
        f"{what}: the output differs from the same convolution without column sums"


# ----------------------------------------------------------------------------------------------- conv3x3 forward
# (N, H, W, Cin, Cout, stride, epilogue, slots, channel offset); the output is channel slot [coff, coff + Cout) of a
# buffer of max(320, coff + Cout + 64) channels, and so is its workspace row
FWD = [
    (2, 64, 64, 64, 64, 1, "bias+rowvec", 4, 64),      # conv1 at 64 x 64
    (256, 64, 64, 64, 64, 1, "bias+res", 4, 128),      # C2 64 x 64, conv2
    (4, 32, 32, 128, 128, 1, "bias+rowvec", 64, 64),   # K = 128: streamed weights
    (256, 32, 32, 128, 128, 1, "bias+res", 4, 64),     # C2 32 x 32
    (256, 16, 16, 256, 256, 1, "", 4, 64),             # C2 16 x 16: pixels-as-M
    (2, 256, 256, 64, 64, 1, "bias+rowvec", 4, 64),    # C3 256 x 256
    (4, 16, 16, 64, 320, 1, "bias", 1, 64),            # 20 tiles: resident
    (32, 16, 16, 64, 320, 1, "", 4, 128),              # 160 tiles: five column blocks do not divide the grid
    (3, 32, 32, 128, 192, 1, "bias+res", 4, 64),      # three column blocks
    (8, 16, 16, 128, 448, 1, "bias+res", 4, 64),
    (8, 16, 16, 64, 256, 1, "bias", 4, 64),            # BN 256
    (4, 16, 16, 64, 512, 1, "bias+rowvec+res", 64, 64),
    (2, 16, 16, 64, 1024, 1, "bias", 4, 64),
    (4, 24, 24, 64, 64, 1, "bias+rowvec", 4, 64),      # BN 64, partial x-block
    (4, 24, 40, 64, 128, 1, "bias+res", 64, 128),      # 40 x 24: BN 128, partial x-block
    (4, 28, 20, 128, 192, 1, "bias", 1, 64),           # 20 x 28: BN 256, partial x- and y-blocks
    (2, 16, 8, 320, 64, 1, "bias+res", 4, 64),         # 8 x 16: 128 pixels, K = 320
    (8, 64, 64, 64, 64, 2, "bias", 4, 64),             # stride 2: 64 -> 32
    (8, 32, 32, 128, 128, 2, "bias", 64, 128),         # 32 -> 16
    # images of 128 pixels or more that a 128-pixel tile packing several images used to refuse
    (4, 12, 12, 64, 64, 1, "bias+rowvec", 4, 64),
    (4, 13, 13, 128, 128, 1, "bias+res", 1, 128),
    (4, 14, 14, 64, 192, 1, "bias", 64, 64),
    (4, 15, 15, 64, 256, 1, "res", 4, 64),
    (4, 24, 6, 64, 64, 1, "bias", 4, 64),              # 6 x 24
    (4, 5, 26, 64, 128, 1, "bias+rowvec+res", 4, 128),  # 26 x 5
    (4, 24, 24, 64, 64, 2, "bias", 4, 64),             # 24 -> 12
    (4, 25, 25, 64, 128, 2, "bias", 4, 64),            # 25 -> 13, pad (1, 1)
    (4, 28, 28, 128, 64, 2, "", 64, 128),              # 28 -> 14
    (4, 29, 29, 64, 64, 2, "bias", 1, 64),             # 29 -> 15
    (4, 48, 12, 64, 64, 2, "bias", 4, 64),             # -> 6 x 24
    (4, 9, 51, 64, 64, 2, "bias", 4, 64),              # -> 26 x 5
]


def _fwd_route(c):
    N, H, W, Ci, Co, s = c[:6]
    return R.launch_route(-(-W // s), -(-H // s), N, Ci, Co, s, s == 1, sms=SMS)


def _fwd_id(c):
    N, H, W, Ci, Co, s, epi, slots, coff = c
    return f"{_fwd_route(c)}-B{N}-{H}x{W}-{Ci}to{Co}-s{s}" + (f"-{epi}" if epi else "") + f"-slots{slots}-coff{coff}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", FWD, ids=[_fwd_id(c) for c in FWD])
def test_conv3x3_fwd_colstats(case, kind):
    N, H, W, Ci, Co, s, epi, slots, coff = case
    g = gen(21)
    Ho, Wo = -(-H // s), -(-W // s)
    ld = max(320, coff + Co + 64)
    x = draw((N, H, W, Ci), kind, g)
    w = weights((3, 3, Ci, Co), kind, g, 9 * Ci, Ho * Wo)
    bias, rowvec, res = epilogue_inputs(epi, kind, g, N, Ho, Wo, Co)
    cs, full, prior = workspace(kind, g, N, ld, slots)
    buf, y = out_slot(N, Ho, Wo, Co, coff, ld)
    ops.conv3x3_fwd(x, w, bias=bias, rowvec=rowvec, res=res, out=y, stride=s, colstats=(cs, coff))
    route = _fwd_route(case)
    assert_route(route)
    R.assert_guard_intact(buf, coff, Co, SENTINEL)
    what = "conv3x3_fwd_stats " + route
    y_plain = torch.full((N, Ho, Wo, Co), SENTINEL, dtype=torch.bfloat16, device=dev)
    ops.conv3x3_fwd(x, w, bias=bias, rowvec=rowvec, res=res, out=y_plain, stride=s)
    assert_same_output(what, y, y_plain)
    check_sums(kind, what, full, prior, slots, coff, y, R.colstats_depth(route, Wo, Ho, Co, slots))


# ----------------------------------------------------------------------------------------------- sub-pixel upsample
# (N, h, w, Cin, Cout, slots, channel offset) of the low-resolution input
UP = [
    (4, 16, 16, 128, 64, 4, 64),                       # per-tap transposed engine
    (2, 32, 32, 64, 128, 64, 128),
    (3, 32, 32, 128, 192, 4, 64),
    (256, 32, 32, 128, 64, 4, 64),                     # C2 32 -> 64
    (2, 16, 16, 256, 256, 4, 64),                      # 256 columns: pixels-as-M
    (4, 8, 8, 128, 128, 4, 64),                        # inputs narrower than 16 used to be refused
    (2, 8, 8, 256, 512, 1, 64),
    (4, 12, 12, 64, 64, 4, 128),
    (4, 6, 6, 64, 64, 64, 64),                         # -> 12 x 12
    (4, 7, 7, 64, 128, 4, 64),                         # -> 14 x 14
    (4, 12, 3, 64, 64, 4, 64),                         # -> 6 x 24
    (2, 16, 8, 320, 64, 4, 64),                        # 8 x 16 inputs, K = 320
]


def _up_route(c):
    N, h, w, Ci, Co = c[:5]
    return R.launch_route(w, h, N, Ci, Co, halo=False, sms=SMS)


def _up_id(c):
    N, h, w, Ci, Co, slots, coff = c
    return f"{_up_route(c)}-B{N}-{h}x{w}-{Ci}to{Co}-slots{slots}-coff{coff}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", UP, ids=[_up_id(c) for c in UP])
def test_upconv3x3_fwd_colstats(case, kind):
    """Four parity launches, each adding its quarter of the output pixels into the same sums."""
    N, h, w_, Ci, Co, slots, coff = case
    g = gen(22)
    ld = max(320, coff + Co + 64)
    x = draw((N, h, w_, Ci), kind, g)
    weff = ops.upconv3x3_pack(weights((3, 3, Ci, Co), kind, g, 9 * Ci, 4 * h * w_, torch.float32))
    bias = draw((Co,), kind, g, torch.float32)
    cs, full, prior = workspace(kind, g, N, ld, slots)
    buf, y = out_slot(N, 2 * h, 2 * w_, Co, coff, ld)
    ops.upconv3x3_fwd(x, weff, bias, y, colstats=(cs, coff))
    route = _up_route(case)
    assert_route(route)
    R.assert_guard_intact(buf, coff, Co, SENTINEL)
    what = "upconv3x3_fwd_stats " + route
    y_plain = torch.full((N, 2 * h, 2 * w_, Co), SENTINEL, dtype=torch.bfloat16, device=dev)
    ops.upconv3x3_fwd(x, weff, bias, y_plain)
    assert_same_output(what, y, y_plain)
    check_sums(kind, what, full, prior, slots, coff, y, R.colstats_depth(route, w_, h, Co, slots, launches=4))


# ----------------------------------------------------------------------------------------------- GroupNorm consumers
# (op, N, H, W, Cin, Cout, groups of the apply) of the producing launch; the workspace is an ops.ColStats as the
# UNet allocates it (zeroed, COLSTATS_SLOTS slots), the output channel slot 64 of a 320-channel buffer
CONSUMERS = [
    ("conv", 4, 32, 32, 64, 64, 8),
    ("conv", 3, 24, 24, 64, 256, 32),
    ("conv", 4, 12, 12, 128, 128, 16),
    ("upconv", 2, 16, 16, 128, 64, 8),
    ("upconv", 3, 8, 8, 64, 128, 16),
]


def _cons_route(c):
    op, N, H, W, Ci, Co = c[:6]
    return R.launch_route(W, H, N, Ci, Co, halo=op == "conv", sms=SMS)


def _cons_id(c):
    op, N, H, W, Ci, Co, G = c
    return f"{op}-{_cons_route(c)}-B{N}-{H}x{W}-{Ci}to{Co}-G{G}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", CONSUMERS, ids=[_cons_id(c) for c in CONSUMERS])
def test_groupnorm_from_engine_sums(case, kind):
    """fdx_groupnorm_stats_from_cols (8, 16 and 32 groups) against the float64 group sums of the stored output, and
    fdx_groupnorm_apply_cols (act none / silu / mish) against GroupNorm with the statistics' error of this chain:
    the engine's (colstats_depth), then each kernel's slots x ceil(cpg / 32) serial additions per lane and its
    5-level warp tree.  apply_cols hands on the statistics it computed: bit for bit stats_from_cols'."""
    op, N, H, W, Ci, Co, Ga = case
    g = gen(23)
    coff, ld, eps = 64, 320, 1e-4
    cs = ops.ColStats(N, ld, dev)
    if op == "conv":
        x = draw((N, H, W, Ci), kind, g)
        w = weights((3, 3, Ci, Co), kind, g, 9 * Ci, H * W * Co)     # group sums run over channels too
        bias = draw((Co,), kind, g, torch.float32)
        buf, y = out_slot(N, H, W, Co, coff, ld)
        ops.conv3x3_fwd(x, w, bias=bias, out=y, colstats=(cs, coff))
        depth = R.colstats_depth(_cons_route(case), W, H, Co, cs.slots)
    else:
        x = draw((N, H, W, Ci), kind, g)
        weff = ops.upconv3x3_pack(weights((3, 3, Ci, Co), kind, g, 9 * Ci, 4 * H * W * Co, torch.float32))
        bias = draw((Co,), kind, g, torch.float32)
        buf, y = out_slot(N, 2 * H, 2 * W, Co, coff, ld)
        ops.upconv3x3_fwd(x, weff, bias, y, colstats=(cs, coff))
        depth = R.colstats_depth(_cons_route(case), W, H, Co, cs.slots, launches=4)
    assert_route(_cons_route(case))
    assert torch.isfinite(y).all()
    val, mag = R.colstats_ref(y)                                    # (N, 2, C)
    stats = {}
    for G in (8, 16, 32):
        cpg = Co // G
        gval = val.reshape(N, 2, G, cpg).sum(-1).transpose(1, 2)    # (N, G, 2), as fdx_groupnorm_stats
        gmag = mag.reshape(N, 2, G, cpg).sum(-1).transpose(1, 2)
        stats[G] = st = ops.groupnorm_stats_from_cols(cs, G, coff, Co)
        what = f"groupnorm_stats_from_cols G{G} {op}"
        if kind == "exact":
            assert R.exact_case_ok(gmag), f"{what}: the exact case's sums reach 2^24"
            assert torch.equal(st.to(F64), gval), f"{what}: differs from the exact group sums"
        else:
            bound = R.f32_bound(gval, R.gamma(depth + cs.slots * math.ceil(cpg / 32) + 5) * gmag)
            report(what, R.assert_elementwise(st, gval, bound, what))
    gam = 1 + 0.2 * torch.randn(Co, generator=g, device=dev)
    bet = 0.2 * torch.randn(Co, generator=g, device=dev)
    yd, gd, bd = y.to(F64), gam.to(F64), bet.to(F64)
    D = depth + cs.slots * math.ceil(Co // Ga / 32) + 5
    refs = {ops.ACT_NONE: R.gn_forward_ref(yd, gd, bd, Ga, eps, False, depth=D),
            ops.ACT_SILU: R.gn_forward_ref(yd, gd, bd, Ga, eps, True, depth=D),
            ops.ACT_MISH: M.gn_mish_forward_ref(yd, gd, bd, Ga, eps, depth=D)}
    for act_fn, (v, d) in refs.items():
        obuf, o = out_slot(N, *y.shape[1:], coff, ld)
        o, st_out = ops.groupnorm_apply_cols(y, Ga, cs, coff, gam, bet, eps, act_fn, out=o)
        what = f"groupnorm_apply_cols act{act_fn} {op}"
        report(what, R.assert_elementwise(o, v, R.bf16_bound(v, d), what))
        R.assert_guard_intact(obuf, coff, Co, SENTINEL)
        assert torch.equal(st_out, stats[Ga]), f"{what}: its statistics differ from groupnorm_stats_from_cols"


# ----------------------------------------------------------------------------------------------- fused GroupNorm backward
@pytest.mark.parametrize("N,H,W,C,Co", [(3, 12, 12, 128, 64), (2, 14, 14, 192, 128)])
def test_conv_dgrad_groupnorm_bwd_fused_small_images(N, H, W, C, Co):
    """conv_dgrad_groupnorm_bwd(fused=True) on images of 12 x 12 and 14 x 14: the data gradient with the first pass of
    the GroupNorm(+SiLU) backward in its epilogue (EPI_GN_BWD: per-image sums of dz and dz x, the same one-image
    pixel box as the forward sums) on the pixels-as-M engine, against conv_gn_backward_ref.  Dense only: silu'
    has no exact integer form."""
    G, eps = 8, 1e-4
    g = gen(24)
    grp = (torch.arange(C, device=dev) // (C // G)).float()
    x = (torch.randn((N, H, W, C), generator=g, device=dev) * (1 + 0.05 * grp) + 0.05 * grp - 0.2).bfloat16()
    gam = 1 + 0.2 * torch.randn(C, generator=g, device=dev)
    bet = 0.2 * torch.randn(C, generator=g, device=dev)
    w = (torch.randn((3, 3, C, Co), generator=g, device=dev) / math.sqrt(9 * C)).bfloat16()
    dy = torch.randn((N, H, W, Co), generator=g, device=dev).bfloat16()
    st = ops.groupnorm_stats(x, G)
    ref = R.conv_gn_backward_ref(x.to(F64), dy.to(F64), w.to(F64), gam.to(F64), bet.to(F64), G, eps)
    dg0, db0 = torch.randn(C, generator=g, device=dev), torch.randn(C, generator=g, device=dev)
    dg, db = dg0.clone(), db0.clone()
    buf, dx = out_slot(N, H, W, C, 64, C + 128)
    ops.conv_dgrad_groupnorm_bwd(dy, w, x, G, st, gam, bet, eps, dg, db, dx, fused=True)
    assert_route("tc")
    R.assert_guard_intact(buf, 64, C, SENTINEL)
    dxv, dxd = ref["dx"]
    report("conv_dgrad_groupnorm_bwd fused dx",
           R.assert_elementwise(dx, dxv, R.bf16_bound(dxv, dxd + R.U32 * dxv.abs()), "fused dx"))
    for name, got, start in (("dgamma", dg, dg0), ("dbeta", db, db0)):
        v, d = ref[name]
        v = v + start.to(F64)
        report("conv_dgrad_groupnorm_bwd fused " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), name))
