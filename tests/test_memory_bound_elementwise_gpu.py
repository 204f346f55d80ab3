"""GroupNorm, RMSNorm, GEGLU and the streaming kernels compared element by element with the float64 references of
tests/elementwise_ref.py, up to the 2048-channel layers of the wide UNet.

Rules for every case: outputs are prefilled with NaN (an element the kernel never writes fails), outputs that are
channel slots of a wider buffer have sentinel neighbours that must come back bit-identical, and the float64
reference runs on the device.  Copies, single bf16 adds and casts are checked bit-exactly; everything else
against the per-element bound of elementwise_ref (derived there, never tuned to a run).

gn_grid reads FDX_GN_WAVES once per process: test_gn_arrangements_in_child_processes runs the GroupNorm cases again
in child pytest processes with other grid sizes (FDX_GN_WAVES = 0, 1, 8 and an uncapped grid)."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops
from flaxdiff_b200._lib import act, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
SENTINEL = -1234.0                                   # exactly representable in bf16
CHILD_FLAG = "ELEMENTWISE_GN_CHILD"                  # set in the child processes of the arrangement test
IN_CHILD = os.environ.get(CHILD_FLAG) == "1"


def sms() -> int:
    return torch.cuda.get_device_properties(dev).multi_processor_count


def report(name, frac):
    print(f"WORST {name} {frac:.3f}")


def slot(shape, lo=8, hi=16, fill=math.nan, dtype=torch.bfloat16):
    """A channel slot [lo, lo + C) of a wider NHWC buffer: the slot holds `fill`, its neighbours SENTINEL."""
    N, H, W, C = shape
    buf = torch.full((N, H, W, lo + C + hi), SENTINEL, dtype=dtype, device=dev)
    v = buf[..., lo:lo + C]
    v.fill_(fill)
    return buf, v


def assert_neighbours_intact(buf, C, lo=8):
    side = torch.cat([buf[..., :lo], buf[..., lo + C:]], -1)
    assert torch.equal(side.view(torch.int16), torch.full_like(side, SENTINEL).view(torch.int16)), \
        "a kernel wrote outside its channel slot"


def into_slot(t, lo=8, hi=16):
    buf, v = slot(tuple(t.shape), lo, hi)
    v.copy_(t)
    return buf, v


def nan_f32(*shape):
    return torch.full(shape, math.nan, dtype=torch.float32, device=dev)


# ----------------------------------------------------------------------------------------------- GroupNorm
def gn_stats(x, G):
    st = nan_f32(x.shape[0], G, 2)
    check(load().fdx_groupnorm_stats(ctypes.byref(act(x, "x")), ctypes.c_int(G), ptr(st), stream_ptr()),
          "groupnorm_stats")
    return st


def gn_loop_iters(N, HW, C, unroll, resident):
    """Pixel-loop iterations of the first CTA of an image under gn_grid (fdx_norm.cu): the grid is capped at
    waves * resident * SMs / N CTAs per image, and each iteration covers unroll * CTAs * rows pixels."""
    rows = 256 // (C // 8)
    waves = int(os.environ.get("FDX_GN_WAVES", "2"))
    need = math.ceil(HW / (rows * unroll))
    bx = max(1, min(need, max(1, waves * resident * sms() // N)))
    return need > bx, math.ceil(HW / (rows * bx * unroll))


def gn_inputs(shape, G, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    N, H, W, C = shape
    grp = (torch.arange(C, device=dev) // (C // G)).to(torch.float32)
    # every group has a mean and spread of its own, so that a channel normalised with another group's
    # statistics is visible element by element
    x = torch.randn(shape, generator=g, device=dev) * (1 + 0.05 * grp) + 0.05 * grp - 0.2
    gamma = 1 + 0.2 * torch.randn(C, generator=g, device=dev)
    beta = 0.2 * torch.randn(C, generator=g, device=dev)
    dy = torch.randn(shape, generator=g, device=dev).bfloat16()
    return x.bfloat16(), gamma, beta, dy


GN_SHAPES = [  # (N, H, W, C, G): ragged and tiny images, every channel count of the UNets, 8 channels per group
    (3, 7, 9, 64, 8), (2, 1, 1, 64, 8), (3, 32, 32, 64, 8), (4, 3, 5, 192, 8), (2, 32, 48, 192, 8),
    (2, 16, 16, 320, 8), (3, 1, 1, 512, 8), (2, 9, 7, 512, 16), (3, 8, 8, 256, 32), (2, 8, 8, 768, 8),
    (2, 16, 16, 1024, 8), (2, 7, 9, 1536, 8), (2, 3, 5, 2048, 8), (2, 32, 32, 2048, 8),
    # with 132 SMs gn_grid caps apply at 82 CTAs per image (2 iterations) and the backward at 49 (4 iterations)
    (16, 128, 128, 64, 8),
]


def _gn_check_all(shape, G, silu, seed=0):
    N, H, W, C = shape
    HW, eps = H * W, 1e-4
    x0, gamma, beta, dy0 = gn_inputs(shape, G, seed)
    xbuf, x = into_slot(x0)                                        # inputs are strided views of concat slots
    dybuf, dy = into_slot(dy0, lo=16, hi=8)
    xd, dyd = x.to(F64), dy.to(F64)
    for unroll, resident in ((4, 5), (3, 3), (3, 2)):            # apply; backward passes without / with addend
        capped, iters = gn_loop_iters(N, HW, C, unroll, resident)
        if capped:
            assert iters >= 2, (shape, unroll, resident, iters)

    st = gn_stats(x, G)
    sv, sd = R.gn_stats_ref(xd, G)
    report("groupnorm_stats", R.assert_elementwise(st, sv, R.f32_bound(sv, sd), "stats"))
    assert torch.equal(st, gn_stats(x, G)), "gn_stats_kernel is not deterministic"

    yv, yd = R.gn_forward_ref(xd, gamma.to(F64), beta.to(F64), G, eps, silu)
    ybuf, y = slot(shape)
    ops.groupnorm_apply(x, G, st, gamma, beta, eps, silu, out=y)
    report("groupnorm_apply", R.assert_elementwise(y, yv, R.bf16_bound(yv, yd), "apply"))
    assert_neighbours_intact(ybuf, C)

    # statistics straight from epilogue column sums: two of the four slots hold half the pixels each (exact sums
    # rounded once to f32), at channel offset 8 of a wider buffer
    cs = ops.ColStats(N, C + 24, dev)
    half = HW // 2
    xf = xd.reshape(N, HW, C)
    for k, (a, b) in enumerate(((0, half), (half, HW))):
        cs.ws[k, :, 0, 8:8 + C] = xf[:, a:b].sum(1).float()
        cs.ws[k, :, 1, 8:8 + C] = (xf[:, a:b] ** 2).sum(1).float()
    ybuf2, y2 = slot(shape)
    stats_out = nan_f32(N, G, 2)
    check(load().fdx_groupnorm_apply_cols(ctypes.byref(act(x, "x")), ctypes.c_int(G), ptr(cs.ws),
                                          ctypes.c_int(cs.slots), ctypes.c_int(cs.channels), ctypes.c_int(8),
                                          ptr(gamma), ptr(beta), ctypes.c_float(eps), ctypes.c_int(int(silu)),
                                          ctypes.byref(act(y2, "out")), ptr(stats_out), stream_ptr()),
          "groupnorm_apply_cols")
    report("groupnorm_apply_cols", R.assert_elementwise(y2, yv, R.bf16_bound(yv, yd), "apply_cols"))
    xg = xd.reshape(N, HW, G, C // G)
    mag = torch.stack([xg.abs().sum((1, 3)), (xg * xg).sum((1, 3))], -1)
    cols_d = R.gamma(4 * math.ceil(C // G / 32) + 6) * mag      # one rounding per slot, 4 slots x ceil(cpg/32), 5
    R.assert_elementwise(stats_out, sv, R.f32_bound(sv, cols_d), "apply_cols stats")
    assert_neighbours_intact(ybuf2, C)
    del yv, yd, y, ybuf, y2, ybuf2

    ref = R.gn_backward_ref(xd, dyd, gamma.to(F64), beta.to(F64), G, eps, silu)
    dxv, dxd = ref["dx"]

    def grads_prefilled():
        g = torch.Generator(device=dev).manual_seed(7)
        return torch.randn(C, generator=g, device=dev), torch.randn(C, generator=g, device=dev)

    def check_param_grads(dg, db, dg0, db0, tag):
        for name, got, start in (("dgamma", dg, dg0), ("dbeta", db, db0)):
            v, d = ref[name]
            v = v + start.to(F64)                                  # both accumulate into the gradient buffers
            report("groupnorm_bwd " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), f"{tag} {name}"))

    # (1) plain, with both column sums
    dg0, db0 = grads_prefilled()
    dg, db = dg0.clone(), db0.clone()
    dxbuf, dx = slot(shape)
    ci, ct = nan_f32(N, C), nan_f32(C)
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, silu, dg, db, dx, csum_img=ci, csum_tot=ct)
    report("groupnorm_bwd dx", R.assert_elementwise(dx, dxv, R.bf16_bound(dxv, dxd), "bwd dx"))
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, dg0, db0, "bwd")
    for name, got in (("csum_img", ci), ("csum_tot", ct)):
        v, d = ref[name]
        report("groupnorm_bwd " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), name))

    # (2) accumulate into an existing gradient (strided), per-image column sums only
    base = torch.randn(shape, device=dev).bfloat16()
    dxbuf, dx = into_slot(base)
    dg, db = dg0.clone(), db0.clone()
    ci = nan_f32(N, C)
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, silu, dg, db, dx, accumulate=True, csum_img=ci)
    tot = dxv + base.to(F64)
    report("groupnorm_bwd accumulate", R.assert_elementwise(dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()),
                                                            "bwd accumulate"))
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, dg0, db0, "bwd accumulate")
    v, d = ref["csum_img"]
    R.assert_elementwise(ci, v, R.f32_bound(v, d), "accumulate csum_img")

    # (3) addend from another strided tensor, no column sums
    add0 = torch.randn(shape, device=dev).bfloat16()
    addbuf, add = into_slot(add0, lo=24, hi=8)
    dxbuf, dx = slot(shape)
    dg, db = dg0.clone(), db0.clone()
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, silu, dg, db, dx, addend=add)
    tot = dxv + add0.to(F64)
    report("groupnorm_bwd_add", R.assert_elementwise(dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()), "bwd_add"))
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, dg0, db0, "bwd_add")


@pytest.mark.parametrize("silu", [True, False])
@pytest.mark.parametrize("N,H,W,C,G", GN_SHAPES)
def test_groupnorm_elementwise(N, H, W, C, G, silu):
    _gn_check_all((N, H, W, C), G, silu)


def test_groupnorm_elementwise_c2_batch():
    """The C2 training shape, N = 256 images of 64x64x64, on the default arrangement.  With 132 SMs gn_grid caps
    groupnorm_apply at 2*5*132/256 = 5 CTAs per image where 32 would cover it (7 loop iterations) and both
    backward passes at 3 CTAs (15 iterations)."""
    if IN_CHILD:
        pytest.skip("default arrangement only")
    N, H, W, C = 256, 64, 64, 64
    for unroll, resident in ((4, 5), (3, 3)):
        capped, iters = gn_loop_iters(N, H * W, C, unroll, resident)
        assert capped and iters >= 2, (unroll, resident, iters)
    _gn_check_all((N, H, W, C), 8, True, seed=3)


FUSED_SHAPES = [  # (N, H, W, Cin, Cout): Cin 64 ... 512 not a multiple of 256 (the default), and one forced case
    (2, 16, 16, 64, 64), (2, 32, 32, 192, 128), (2, 16, 16, 320, 64), (3, 16, 16, 448, 64), (2, 16, 8, 256, 64),
    (2, 32, 32, 128, 256), (1, 64, 64, 192, 64)]


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "two-pass"])
@pytest.mark.parametrize("N,H,W,C,Co", FUSED_SHAPES)
def test_groupnorm_conv_dgrad_fused_elementwise(N, H, W, C, Co, fused):
    """conv_dgrad_groupnorm_bwd(fused=True): dz = dgrad * silu'(z) in the data gradient's epilogue (a bf16
    intermediate), then one pass over x and dz; fused=False: the data gradient da as the bf16 intermediate, then
    the two-pass GroupNorm backward.  Plain with column sums, accumulating and with an addend."""
    G, eps, shape = 8, 1e-4, (N, H, W, C)
    x0, gamma, beta, _ = gn_inputs(shape, G, 11)
    _, x = into_slot(x0)
    w = (torch.randn(3, 3, C, Co, device=dev) / math.sqrt(9 * C)).bfloat16()
    dy = torch.randn(N, H, W, Co, device=dev).bfloat16()
    st = gn_stats(x, G)
    ref = R.conv_gn_backward_ref(x.to(F64), dy.to(F64), w.to(F64), gamma.to(F64), beta.to(F64), G, eps)
    dxv, dxd = ref["dx"]
    dg0, db0 = torch.randn(C, device=dev), torch.randn(C, device=dev)
    for mode in ("plain", "accumulate", "addend"):
        dg, db = dg0.clone(), db0.clone()
        ci, ct = (nan_f32(N, C), nan_f32(C)) if mode == "plain" else (None, None)
        extra = torch.zeros(shape, dtype=F64, device=dev)
        if mode == "accumulate":
            base = torch.randn(shape, device=dev).bfloat16()
            dxbuf, dx = into_slot(base)
            extra = base.to(F64)
        else:
            dxbuf, dx = slot(shape)
        add = None
        if mode == "addend":
            add = torch.randn(shape, device=dev).bfloat16()
            extra = add.to(F64)
        ops.conv_dgrad_groupnorm_bwd(dy, w, x, G, st, gamma, beta, eps, dg, db, dx, accumulate=mode == "accumulate",
                                     csum_img=ci, csum_tot=ct, fused=fused, addend=add)
        tot = dxv + extra
        report("conv_dgrad_groupnorm_bwd dx", R.assert_elementwise(
            dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()), f"fused={fused} {mode} dx"))
        assert_neighbours_intact(dxbuf, C)
        for name, got, start in (("dgamma", dg, dg0), ("dbeta", db, db0)):
            v, d = ref[name]
            v = v + start.to(F64)
            report("conv_dgrad_groupnorm_bwd " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), name))
        if mode == "plain":
            for name, got in (("csum_img", ci), ("csum_tot", ct)):
                v, d = ref[name]
                R.assert_elementwise(got, v, R.f32_bound(v, d), "fused " + name)


@pytest.mark.parametrize("env_kv", [{"FDX_GN_WAVES": "0"}, {"FDX_GN_WAVES": "1"}, {"FDX_GN_WAVES": "8"},
                                    {"FDX_GN_WAVES": "1000"}],
                         ids=["one-cta-per-image", "one-wave", "eight-waves", "uncapped"])
def test_gn_arrangements_in_child_processes(env_kv):
    """The grid size is read once per process: run every GroupNorm case above in a child with it set.
    FDX_GN_WAVES=0 caps gn_grid at one CTA per image, so the pixel loops of the apply and both backward passes
    iterate ceil(HW / (rows * unroll)) times: 128 (apply) and 171 (backward) at 128x128x64, 39 and 52 at
    32x48x192; _gn_check_all asserts >= 2 for every capped shape.  One and eight waves split the pixels of an image
    over other CTA counts than the default two.  With the uncapped grid every CTA runs at most one loop iteration, so
    the most CTAs add partial sums into the same red / dgamma / dbeta / column-sum entries (171 per image for the
    backward at 128x128x64)."""
    if IN_CHILD:
        pytest.skip("already a child")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-k", "groupnorm",
                        "-s", "-p", "no:cacheprovider"], capture_output=True, text=True,
                       env=dict(os.environ, **env_kv, **{CHILD_FLAG: "1"}), timeout=1500, cwd=root)
    print("\n".join(ln for ln in r.stdout.splitlines() if ln.startswith("WORST")))
    assert r.returncode == 0 and " passed" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


# ----------------------------------------------------------------------------------------------- RMSNorm
@pytest.mark.parametrize("C", [8, 64, 320, 768, 1024])
def test_rmsnorm_elementwise(C):
    """16x32x32 = 16384 pixels: the forward grid sweeps 8*SMs*8 = 8448 pixels per pass and the backward
    2*SMs*8 = 2112 (132 SMs), so both grid-stride loops run more than once (2 and 8 times)."""
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    shape, eps = (16, 32, 32, C), 1e-4
    npix = 16 * 32 * 32
    fwd_sweep, bwd_sweep = min(math.ceil(npix / 8), 8 * sms()) * 8, min(math.ceil(npix / 8), 2 * sms()) * 8
    assert math.ceil(npix / fwd_sweep) >= 2 and math.ceil(npix / bwd_sweep) >= 2
    g = torch.Generator(device=dev).manual_seed(C)
    xbuf, x = into_slot(torch.randn(shape, generator=g, device=dev).bfloat16())
    dybuf, dy = into_slot(torch.randn(shape, generator=g, device=dev).bfloat16(), lo=16, hi=8)
    scale = 1 + 0.2 * torch.randn(C, generator=g, device=dev)
    xd, dyd, sd = x.to(F64), dy.to(F64), scale.to(F64)
    yv, yd = R.rms_forward_ref(xd, sd, eps)
    ybuf, y = slot(shape)
    ops.rmsnorm_fwd(x, scale, eps, out=y)
    report("rmsnorm_fwd", R.assert_elementwise(y, yv, R.bf16_bound(yv, yd), "rmsnorm fwd"))
    assert_neighbours_intact(ybuf, C)
    ref = R.rms_backward_ref(xd, dyd, sd, eps, bwd_sweep)
    dxv, dxd = ref["dx"]
    for acc in (False, True):
        base = torch.randn(shape, device=dev).bfloat16()
        dxbuf, dx = into_slot(base) if acc else slot(shape)
        ds0 = torch.randn(C, device=dev)                          # the kernel adds into dscale
        ds = ds0.clone()
        ops.rmsnorm_bwd(x, dy, scale, eps, dx, ds, accumulate=acc)
        tot = dxv + base.to(F64) if acc else dxv
        report("rmsnorm_bwd dx", R.assert_elementwise(dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()),
                                                      f"rmsnorm bwd dx accumulate={acc}"))
        assert_neighbours_intact(dxbuf, C)
        v, d = ref["dscale"]
        v = v + ds0.to(F64)
        report("rmsnorm_bwd dscale", R.assert_elementwise(ds, v, R.f32_bound(v, d), "dscale"))


# ----------------------------------------------------------------------------------------------- GEGLU
@pytest.mark.parametrize("inner", [8, 1280, 4096])
@pytest.mark.parametrize("rows", [1, 77, 4096])
def test_geglu_elementwise(rows, inner):
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    g = torch.Generator(device=dev).manual_seed(rows + inner)
    u = (torch.randn(rows, 2 * inner, generator=g, device=dev) * 3).clamp(-10, 10)
    u[:, ::7] = 0                                                 # exact zeros in both halves
    u[:, 3::11] = 10 * torch.sign(torch.randn(rows, len(range(3, 2 * inner, 11)), generator=g, device=dev))
    u = u.bfloat16()
    dg = torch.randn(rows, inner, generator=g, device=dev).bfloat16()
    gout = torch.full((rows, inner), math.nan, dtype=torch.bfloat16, device=dev)
    check(load().fdx_geglu_fwd(ptr(u), ctypes.c_longlong(rows), ctypes.c_int(inner), ptr(gout), stream_ptr()),
          "geglu_fwd")
    gv, gd = R.geglu_forward_ref(u.to(F64))
    report("geglu_fwd", R.assert_elementwise(gout, gv, R.bf16_bound(gv, gd), "geglu fwd"))
    du = torch.full((rows, 2 * inner), math.nan, dtype=torch.bfloat16, device=dev)
    check(load().fdx_geglu_bwd(ptr(u), ptr(dg), ctypes.c_longlong(rows), ctypes.c_int(inner), ptr(du), stream_ptr()),
          "geglu_bwd")
    dv, dd = R.geglu_backward_ref(u.to(F64), dg.to(F64))
    b = R.bf16_bound(dv, dd)
    for half, sl in (("d hidden_linear", slice(0, inner)), ("d hidden_gelu", slice(inner, 2 * inner))):
        assert torch.isfinite(du[:, sl].float()).all(), f"geglu_bwd left part of {half} unwritten"
        report("geglu_bwd", R.assert_elementwise(du[:, sl], dv[:, sl], b[:, sl], "geglu bwd " + half))


# ----------------------------------------------------------------------------------------------- streaming
def no_tiny(t, floor=2.0 ** -6):
    """|t| >= 2^-6 (or 0): four or five such bf16 values span < 2^16 in magnitude, so their f32 sum is exact."""
    return torch.where(t.abs() < floor, torch.zeros_like(t), t)


def test_upsample2x_bit_exact():
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    for shape in ((2, 7, 9, 64), (3, 16, 16, 192), (2, 4, 4, 2048)):
        N, H, W, C = shape
        _, x = into_slot(torch.randn(shape, device=dev).bfloat16())
        ybuf, y = slot((N, 2 * H, 2 * W, C))
        ops.upsample2x(x, out=y)
        assert torch.equal(y.view(torch.int16), R.upsample2x_ref(x).view(torch.int16)), shape
        assert_neighbours_intact(ybuf, C)


@pytest.mark.parametrize("accumulate", [False, True])
def test_upsample2x_bwd_bit_exact(accumulate):
    """Exact: with every input 0 or >= 2^-6 in magnitude (and |x| < 6 for normal draws), the 4 (or, accumulating, 5)
    bf16 values of a sum lie within 2^16 of each other, their f32 sum loses no bit, and the kernel's single
    rounding to bf16 equals the float64 sum rounded to bf16."""
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    for shape in ((2, 7, 9, 64), (3, 16, 16, 320), (2, 4, 4, 2048)):
        N, H, W, C = shape
        _, dy = into_slot(no_tiny(torch.randn(N, 2 * H, 2 * W, C, device=dev)).bfloat16(), lo=16, hi=8)
        base = no_tiny(torch.randn(shape, device=dev)).bfloat16()
        dxbuf, dx = into_slot(base) if accumulate else slot(shape)
        ops.upsample2x_bwd(dy, dx, accumulate=accumulate)
        want = R.upsample2x_bwd_ref(dy) + (base.to(F64) if accumulate else 0)
        assert torch.equal(dx.view(torch.int16), want.bfloat16().view(torch.int16)), shape
        assert_neighbours_intact(dxbuf, C)


def test_act_add_bit_exact_including_in_place():
    """One f32 add of two bf16 values rounded once: bit-exact.  The model calls act_add(dx, dout, dx), so the
    output aliasing the first input (declared __restrict__ in the kernel) is checked too."""
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    for shape in ((3, 7, 9, 64), (2, 16, 16, 1024), (1, 1, 1, 2048)):
        C = shape[-1]
        a0, b0 = torch.randn(shape, device=dev).bfloat16(), torch.randn(shape, device=dev).bfloat16()
        want = (a0.float() + b0.float()).bfloat16().view(torch.int16)
        _, a = into_slot(a0)
        _, b = into_slot(b0, lo=16, hi=8)
        obuf, o = slot(shape)
        ops.act_add(a, b, o)
        assert torch.equal(o.view(torch.int16), want), shape
        assert_neighbours_intact(obuf, C)
        abuf, a = into_slot(a0)
        ops.act_add(a, b, a)                                      # in place, out = a
        assert torch.equal(a.view(torch.int16), want), ("in place", shape)
        assert_neighbours_intact(abuf, C)


def test_cast_f32_bf16_special_values_bit_exact():
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    one = 0x3F800000
    specials = torch.tensor([0.0, -0.0, math.inf, -math.inf, math.nan, -math.nan, 1e-45, -1e-45, 1.17549435e-38,
                             2.0 ** -133, 3.0e38, -3.4e38, 1.0, -1.0], dtype=torch.float32)
    # exact ties between bf16 neighbours (low half 0x8000), even and odd kept bit, and just off the tie
    bits = torch.tensor([one | 0x8000, one | 0x18000, one | 0x7FFF, one | 0x8001, 0x00008000, 0x00018000,
                         0x7F7F8000, 0x807F8000, 0x7F7FFFFF], dtype=torch.int64).to(torch.int32)
    ties = bits.view(torch.float32)
    rnd = torch.randn(4096 - 24) * torch.exp2(torch.randint(-140, 120, (4096 - 24,)).float())
    src = torch.cat([specials, ties, rnd, torch.zeros(1)]).to(dev)
    src = src[: src.numel() // 4 * 4].contiguous()
    dst = torch.full(src.shape, math.nan, dtype=torch.bfloat16, device=dev)
    ops.cast_f32_bf16(src, dst)
    want = src.bfloat16()                                         # torch: round to nearest even
    nan = torch.isnan(src)
    assert torch.equal(torch.isnan(dst), nan), "NaN must stay NaN and nothing else may become NaN"
    assert torch.equal(dst[~nan].view(torch.int16), want[~nan].view(torch.int16))


def quantized(shape):
    """k/8 with |k| <= 32: exact in bf16, and any f32 sum of at most 2^18 of them is exact (every partial sum is a
    multiple of 2^-3 below 2^20, at most 23 significant bits), so column sums must equal the float64 sums bit for bit."""
    return (torch.randint(-32, 33, shape, device=dev).float() / 8).bfloat16()


@pytest.mark.parametrize("C", [64, 192, 2048])
def test_colsum_exact(C):
    """Per image and whole batch at N = 256.  Whole-batch mode launches gridDim.y = 592 / gridDim.x < N rows of
    CTAs, so every CTA walks several images (the `n += gridDim.y` loop)."""
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    N, H, W = 256, 32, 32                                      # 2^18 pixels
    _, x = into_slot(quantized((N, H, W, C)))
    rows = 256 // (C // 8)
    bx = max(1, min(math.ceil(H * W / (4 * rows)), math.ceil(16 * sms() / N)))
    assert min(N, max(1, 592 // bx)) < N
    for per_image in (True, False):
        out = nan_f32(*((N, C) if per_image else (C,)))
        ops.colsum(x, per_image, out=out)
        assert torch.equal(out.to(F64), R.colsum_ref(x, per_image)), per_image


def test_colsum_rows_8192_columns():
    """Bias gradients of dense layers: ops.colsum_rows cuts 8192 columns into four 2048-wide slabs."""
    if IN_CHILD:
        pytest.skip("GroupNorm arrangements only")
    for rows in (1, 77, 4096):
        x = quantized((rows, 8192))
        out = nan_f32(8192)
        ops.colsum_rows(x, out)
        assert torch.equal(out.to(F64), x.to(F64).sum(0)), rows
