"""GroupNorm + mish kernels compared element by element with the float64 references of tests/elementwise_ref.py:
the apply kernels, the two-pass backward and the transposed engine's fused data-gradient epilogue (act = 2).

Same rules as test_memory_bound_elementwise_gpu.py: NaN-prefilled outputs, channel slots with sentinel
neighbours, the float64 reference on the device, per-element bounds derived in mish_ref.
The GroupNorm betas spread z = a x + b over [-100, 100] on every other channel, so both clamp regions of the
kernels' mish (e^z overflow above, underflow below) are covered next to the region around 0."""
import ctypes
import math

import pytest
import torch

import elementwise_ref as R
import mish_ref as M
from flaxdiff_b200 import ops
from flaxdiff_b200._lib import act, check, load, ptr, stream_ptr
from test_memory_bound_elementwise_gpu import (assert_neighbours_intact, gn_stats, into_slot, nan_f32, report,
                                               slot)

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
MISH = ops.ACT_MISH
FDX_ERR_INVALID_ARG, FDX_ERR_UNSUPPORTED = -1, -2
FDX_KERNEL_TCT = 1


def mish_inputs(shape, G, seed):
    """x with a mean and spread per group; beta of the odd channels spread over [-100, 100] (z spans the clamp
    regions), of the even ones small (z around 0)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    N, H, W, C = shape
    grp = (torch.arange(C, device=dev) // (C // G)).to(torch.float32)
    x = torch.randn(shape, generator=g, device=dev) * (1 + 0.05 * grp) + 0.05 * grp - 0.2
    gamma = 1 + 0.2 * torch.randn(C, generator=g, device=dev)
    spread = 100 * (2 * torch.rand(C, generator=g, device=dev) - 1)
    beta = torch.where(torch.arange(C, device=dev) % 2 == 1, spread, 0.5 * torch.randn(C, generator=g, device=dev))
    dy = torch.randn(shape, generator=g, device=dev).bfloat16()
    return x.bfloat16(), gamma, beta, dy


GN_SHAPES = [  # (N, H, W, C), 8 groups: every channel count of the UNets, ragged and tiny images
    (3, 7, 9, 64), (2, 32, 32, 64), (2, 16, 16, 128), (2, 32, 48, 192), (2, 16, 16, 320), (3, 1, 1, 512),
    (2, 8, 8, 768), (2, 16, 16, 1024), (2, 7, 9, 1536), (2, 32, 32, 2048)]


@pytest.mark.parametrize("N,H,W,C", GN_SHAPES)
def test_groupnorm_mish_elementwise(N, H, W, C):
    G, eps, shape = 8, 1e-4, (N, H, W, C)
    HW = H * W
    x0, gamma, beta, dy0 = mish_inputs(shape, G, 5)
    _, x = into_slot(x0)
    _, dy = into_slot(dy0, lo=16, hi=8)
    xd, dyd = x.to(F64), dy.to(F64)
    zmin, zmax = (x.float() * gamma + beta).min().item(), (x.float() * gamma + beta).max().item()
    assert zmin < -80 and zmax > 80, (zmin, zmax)
    st = gn_stats(x, G)

    yv, yd = M.gn_mish_forward_ref(xd, gamma.to(F64), beta.to(F64), G, eps)
    ybuf, y = slot(shape)
    ops.groupnorm_apply(x, G, st, gamma, beta, eps, MISH, out=y)
    report("groupnorm_apply mish", R.assert_elementwise(y, yv, R.bf16_bound(yv, yd), "apply mish"))
    assert_neighbours_intact(ybuf, C)

    # statistics from epilogue column sums (two of four slots, channel offset 8 of a wider buffer)
    cs = ops.ColStats(N, C + 24, dev)
    half = HW // 2
    xf = xd.reshape(N, HW, C)
    for k, (a, b) in enumerate(((0, half), (half, HW))):
        cs.ws[k, :, 0, 8:8 + C] = xf[:, a:b].sum(1).float()
        cs.ws[k, :, 1, 8:8 + C] = (xf[:, a:b] ** 2).sum(1).float()
    ybuf2, y2 = slot(shape)
    ops.groupnorm_apply_cols(x, G, cs, 8, gamma, beta, eps, MISH, out=y2)
    report("groupnorm_apply_cols mish", R.assert_elementwise(y2, yv, R.bf16_bound(yv, yd), "apply_cols mish"))
    assert_neighbours_intact(ybuf2, C)
    del yv, yd

    ref = M.gn_mish_backward_ref(xd, dyd, gamma.to(F64), beta.to(F64), G, eps)
    dxv, dxd = ref["dx"]
    # zero priors: on the channels where z << 0 mish' ~ 0 and the sums are tiny, so a non-zero prior would be
    # rounded once per CTA's atomic add, which the references' single-rounding model of the prior does not cover
    # (accumulation onto priors is the same code as with silu, checked in test_memory_bound_elementwise_gpu.py)
    dg0, db0 = torch.zeros(C, device=dev), torch.zeros(C, device=dev)

    def check_param_grads(dg, db, tag):
        for name, got, start in (("dgamma", dg, dg0), ("dbeta", db, db0)):
            v, d = ref[name]
            v = v + start.to(F64)
            report("groupnorm_bwd mish " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), f"{tag} {name}"))

    # plain, with both column sums
    dg, db = dg0.clone(), db0.clone()
    dxbuf, dx = slot(shape)
    ci, ct = nan_f32(N, C), nan_f32(C)
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, MISH, dg, db, dx, csum_img=ci, csum_tot=ct)
    report("groupnorm_bwd mish dx", R.assert_elementwise(dx, dxv, R.bf16_bound(dxv, dxd), "bwd mish dx"))
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, "bwd")
    for name, got in (("csum_img", ci), ("csum_tot", ct)):
        v, d = ref[name]
        report("groupnorm_bwd mish " + name, R.assert_elementwise(got, v, R.f32_bound(v, d), name))

    # accumulate into an existing (strided) gradient
    base = torch.randn(shape, device=dev).bfloat16()
    dxbuf, dx = into_slot(base)
    dg, db = dg0.clone(), db0.clone()
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, MISH, dg, db, dx, accumulate=True)
    tot = dxv + base.to(F64)
    R.assert_elementwise(dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()), "bwd mish accumulate")
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, "accumulate")

    # addend (fdx_groupnorm_bwd_add)
    add0 = torch.randn(shape, device=dev).bfloat16()
    _, add = into_slot(add0, lo=24, hi=8)
    dxbuf, dx = slot(shape)
    dg, db = dg0.clone(), db0.clone()
    ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, MISH, dg, db, dx, addend=add)
    tot = dxv + add0.to(F64)
    R.assert_elementwise(dx, tot, R.bf16_bound(tot, dxd + R.U32 * tot.abs()), "bwd_add mish")
    assert_neighbours_intact(dxbuf, C)
    check_param_grads(dg, db, "bwd_add")


# Transposed-engine geometries of the UNets' data gradients: 64^2 halo with resident weights (K = 64), 32^2 / 16^2
# with several K chunks, and 64 ... 448 output columns (Cin)
FUSED_SHAPES = [  # (N, H, W, Cin, Cout)
    (2, 64, 64, 64, 64), (2, 64, 64, 64, 128), (2, 32, 32, 128, 256), (2, 32, 32, 192, 128), (2, 16, 16, 320, 64),
    (2, 16, 16, 384, 512), (3, 16, 16, 448, 512)]


@pytest.mark.parametrize("N,H,W,C,Co", FUSED_SHAPES)
def test_conv_dgrad_groupnorm_mish_fused_elementwise(N, H, W, C, Co):
    """conv_dgrad_groupnorm_bwd(act_fn=mish, fused=True): dz = dgrad * mish'(z) in the transposed engine's epilogue,
    then one pass over x and dz, against float64 and against the two-pass mish route (fused=False: conv3x3_dgrad +
    groupnorm_bwd).  The default route is fused on these shapes only up to 16 x 16 pixels."""
    G, eps, shape = 8, 1e-4, (N, H, W, C)
    x0, gamma, beta, _ = mish_inputs(shape, G, 13)
    _, x = into_slot(x0)
    w = (torch.randn(3, 3, C, Co, device=dev) / math.sqrt(9 * C)).bfloat16()
    dy = torch.randn(N, H, W, Co, device=dev).bfloat16()
    assert ops._gn_fuse_default(x, dy)
    st = gn_stats(x, G)
    ref = M.conv_gn_mish_backward_ref(x.to(F64), dy.to(F64), w.to(F64), gamma.to(F64), beta.to(F64), G, eps)
    dxv, dxd = ref["dx"]
    dg0, db0 = torch.zeros(C, device=dev), torch.zeros(C, device=dev)      # zero priors, as above
    results = {}
    for fused in (True, False):
        for mode in ("plain", "accumulate", "addend"):
            dg, db = dg0.clone(), db0.clone()
            ci, ct = (nan_f32(N, C), nan_f32(C)) if mode == "plain" else (None, None)
            extra = torch.zeros(shape, dtype=F64, device=dev)
            if mode == "accumulate":
                base = torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(3), device=dev).bfloat16()
                dxbuf, dx = into_slot(base)
                extra = base.to(F64)
            else:
                dxbuf, dx = slot(shape)
            add = None
            if mode == "addend":
                add = torch.randn(shape, generator=torch.Generator(device=dev).manual_seed(4), device=dev).bfloat16()
                extra = add.to(F64)
            ops.conv_dgrad_groupnorm_bwd(dy, w, x, G, st, gamma, beta, eps, dg, db, dx,
                                         accumulate=mode == "accumulate", csum_img=ci, csum_tot=ct, fused=fused,
                                         addend=add, act_fn=MISH)
            if fused and mode == "plain":
                torch.cuda.synchronize()
                assert load().fdx_last_kernel_kind() == FDX_KERNEL_TCT
            tot = dxv + extra
            bound = R.bf16_bound(tot, dxd + R.U32 * tot.abs())
            report("conv_dgrad_groupnorm_bwd mish dx", R.assert_elementwise(dx, tot, bound, f"fused={fused} {mode}"))
            assert_neighbours_intact(dxbuf, C)
            for name, got, start in (("dgamma", dg, dg0), ("dbeta", db, db0)):
                v, d = ref[name]
                v = v + start.to(F64)
                R.assert_elementwise(got, v, R.f32_bound(v, d), f"fused={fused} {mode} {name}")
            if mode == "plain":
                for name, got in (("csum_img", ci), ("csum_tot", ct)):
                    v, d = ref[name]
                    R.assert_elementwise(got, v, R.f32_bound(v, d), f"fused={fused} {name}")
            results[(fused, mode)] = (dx.clone(), bound)
    # the two routes agree with each other within the sum of their bounds
    for mode in ("plain", "accumulate", "addend"):
        (a, ba), (b, _) = results[(True, mode)], results[(False, mode)]
        R.assert_elementwise(a, b.to(F64), 2 * ba, f"fused vs two-pass {mode}")


def _dgrad_gn_raw(dy, w, dz, x, ab, ws, act_code):
    return load().fdx_conv3x3_dgrad_gn_act(ctypes.byref(act(dy, "dy")), ptr(w), ctypes.byref(act(dz, "dz")),
                                           ctypes.byref(act(x, "x")), ptr(ab), ptr(ws), ctypes.c_int(ws.shape[0]),
                                           ctypes.c_int(act_code), stream_ptr())


@pytest.mark.parametrize("N,H,W,C,Co", [(2, 64, 64, 64, 64), (2, 32, 32, 192, 128), (2, 16, 16, 256, 64)])
def test_dgrad_gn_act_silu_is_the_old_entry_point(N, H, W, C, Co):
    """fdx_conv3x3_dgrad_gn_act(act = 1) writes the same dz, bit for bit, as fdx_conv3x3_dgrad_gn, on both
    engines (Cin = 256 runs on the pixels-as-M engine).  The sums are float atomics (order-dependent): f32-close."""
    G, eps = 8, 1e-4
    x0, gamma, beta, _ = mish_inputs((N, H, W, C), G, 21)
    x = x0
    w = (torch.randn(3, 3, C, Co, device=dev) / math.sqrt(9 * C)).bfloat16()
    dy = torch.randn(N, H, W, Co, device=dev).bfloat16()
    ab = ops.groupnorm_coeffs(gn_stats(x, G), gamma, beta, H * W, eps)
    dz_old, dz_new = (torch.full((N, H, W, C), math.nan, dtype=torch.bfloat16, device=dev) for _ in range(2))
    ws_old = torch.empty((ops.GN_FUSE_SLOTS, N, 2, C), dtype=torch.float32, device=dev)
    ws_new = torch.empty_like(ws_old)
    check(load().fdx_conv3x3_dgrad_gn(ctypes.byref(act(dy, "dy")), ptr(w), ctypes.byref(act(dz_old, "dz")),
                                      ctypes.byref(act(x, "x")), ptr(ab), ptr(ws_old), ctypes.c_int(ops.GN_FUSE_SLOTS),
                                      stream_ptr()), "conv3x3_dgrad_gn")
    check(_dgrad_gn_raw(dy, w, dz_new, x, ab, ws_new, 1), "conv3x3_dgrad_gn_act")
    assert torch.equal(dz_old.view(torch.int16), dz_new.view(torch.int16))
    a, b = ws_old.sum(0).double(), ws_new.sum(0).double()
    assert ((a - b).abs() <= 1e-5 * (a.abs() + 1)).all()


def test_act_argument_errors():
    N, H, W, C, Co, G, eps = 2, 16, 16, 64, 64, 8, 1e-4
    x, gamma, beta, dy0 = mish_inputs((N, H, W, C), G, 1)
    st = gn_stats(x, G)
    y = torch.empty_like(x)
    lib = load()
    for bad in (3, -1):
        assert lib.fdx_groupnorm_apply(ctypes.byref(act(x, "x")), ctypes.c_int(G), ptr(st), ptr(gamma), ptr(beta),
                                       ctypes.c_float(eps), ctypes.c_int(bad), ctypes.byref(act(y, "y")),
                                       stream_ptr()) == FDX_ERR_INVALID_ARG
        assert b"act" in lib.fdx_last_error()
        with pytest.raises(ValueError):
            ops.groupnorm_bwd(x, dy0, G, st, gamma, beta, eps, bad, torch.zeros(C, device=dev),
                              torch.zeros(C, device=dev), torch.empty_like(x))
    red = torch.empty(2 * N * G, device=dev)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    for add in (False, True):
        fn = lib.fdx_groupnorm_bwd_add if add else lib.fdx_groupnorm_bwd
        last = ctypes.byref(act(y, "a")) if add else ctypes.c_int(0)
        assert fn(ctypes.byref(act(x, "x")), ctypes.byref(act(dy0, "dy")), ctypes.c_int(G), ptr(st), ptr(gamma),
                  ptr(beta), ctypes.c_float(eps), ctypes.c_int(3), ptr(red), ptr(dg), ptr(db),
                  ctypes.byref(act(y, "dx")), last, None, None, stream_ptr()) == FDX_ERR_INVALID_ARG
    cs = ops.ColStats(N, C, dev)
    assert lib.fdx_groupnorm_apply_cols(ctypes.byref(act(x, "x")), ctypes.c_int(G), ptr(cs.ws), ctypes.c_int(cs.slots),
                                        ctypes.c_int(C), ctypes.c_int(0), ptr(gamma), ptr(beta), ctypes.c_float(eps),
                                        ctypes.c_int(3), ctypes.byref(act(y, "y")), ptr(nan_f32(N, G, 2)),
                                        stream_ptr()) == FDX_ERR_INVALID_ARG
    # the fused data gradient: act 0 and 3 are refused; mish where only the pixels-as-M engine could run is
    # unsupported (Cin = 256 is a multiple of 256; H = 8 is not 16-aligned)
    ab = ops.groupnorm_coeffs(st, gamma, beta, H * W, eps)
    w = (torch.randn(3, 3, C, Co, device=dev) / 24).bfloat16()
    dy = torch.randn(N, H, W, Co, device=dev).bfloat16()
    ws = torch.empty((ops.GN_FUSE_SLOTS, N, 2, C), dtype=torch.float32, device=dev)
    for bad in (0, 3):
        assert _dgrad_gn_raw(dy, w, torch.empty_like(x), x, ab, ws, bad) == FDX_ERR_INVALID_ARG
    for (h, wd, c) in ((16, 16, 256), (8, 32, 64)):
        xx, gg, bb, _ = mish_inputs((N, h, wd, c), G, 2)
        ab2 = ops.groupnorm_coeffs(gn_stats(xx, G), gg, bb, h * wd, eps)
        w2 = (torch.randn(3, 3, c, Co, device=dev) / 24).bfloat16()
        dy2 = torch.randn(N, h, wd, Co, device=dev).bfloat16()
        ws2 = torch.empty((ops.GN_FUSE_SLOTS, N, 2, c), dtype=torch.float32, device=dev)
        assert _dgrad_gn_raw(dy2, w2, torch.empty_like(xx), xx, ab2, ws2, 2) == FDX_ERR_UNSUPPORTED
        assert b"mish" in lib.fdx_last_error()
        assert not ops._gn_fuse_default(xx, dy2)
    torch.cuda.synchronize()
