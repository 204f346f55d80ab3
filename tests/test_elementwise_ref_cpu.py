"""The float64 references and the element-wise comparator of tests/elementwise_ref.py, without a GPU:
the closed-form forwards and backwards agree with float64 autograd, the comparator accepts the exact answer
rounded to bf16, and it rejects planted defects that a relative-L2 check of 1e-2 lets through."""
import math

import pytest
import torch
import torch.nn.functional as Fnn

import elementwise_ref as R


def _bf(t):
    return t.bfloat16().double()


def _close(a, b, tol=1e-10):
    a, b = a.detach().double(), b.detach().double()
    assert (a - b).abs().max().item() <= tol * (b.abs().max().item() + 1e-30), (a - b).abs().max().item()


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def _gn_inputs(shape, G, seed=0):
    g = torch.Generator().manual_seed(seed)
    N, H, W, C = shape
    grp = torch.arange(C) // (C // G)
    # every group has a mean and a spread of its own, so that a channel mapped to the wrong group shows
    x = _bf(torch.randn(shape, generator=g, dtype=torch.float64) * (1 + 0.05 * grp) + 0.05 * grp - 0.2)
    gam = 1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64)
    bet = 0.2 * torch.randn(C, generator=g, dtype=torch.float64)
    return x, gam, bet


def _gn_autograd(x, gam, bet, G, eps, silu):
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x, gam, bet))
    y = Fnn.group_norm(xr.permute(0, 3, 1, 2), G, gr, br, eps).permute(0, 2, 3, 1)
    return xr, gr, br, (Fnn.silu(y) if silu else y)


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("shape,G", [((2, 3, 5, 64), 8), ((3, 4, 4, 256), 32), ((1, 7, 9, 192), 8), ((2, 1, 1, 128), 16)])
def test_groupnorm_references_match_autograd(shape, G, silu):
    eps = 1e-4
    x, gam, bet = _gn_inputs(shape, G)
    xr, gr, br, yr = _gn_autograd(x, gam, bet, G, eps, silu)
    y, d = R.gn_forward_ref(x, gam, bet, G, eps, silu)
    _close(y, yr)
    assert (d >= 0).all() and torch.isfinite(d).all()
    st, _ = R.gn_stats_ref(x, G)
    xg = x.reshape(shape[0], -1, G, shape[-1] // G)
    _close(st[..., 0], xg.sum((1, 3)))
    dy = _bf(torch.randn(shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64))
    yr.backward(dy)
    out = R.gn_backward_ref(x, dy, gam, bet, G, eps, silu)
    _close(out["dx"][0], xr.grad)
    _close(out["dgamma"][0], gr.grad)
    _close(out["dbeta"][0], br.grad)
    _close(out["csum_img"][0], xr.grad.sum((1, 2)))
    _close(out["csum_tot"][0], xr.grad.sum((0, 1, 2)))


def test_conv_groupnorm_backward_reference_matches_autograd():
    eps, G = 1e-4, 8
    x, gam, bet = _gn_inputs((2, 8, 8, 64), G)
    w = _bf(torch.randn(3, 3, 64, 32, generator=torch.Generator().manual_seed(2), dtype=torch.float64) / 24)
    dy = _bf(torch.randn(2, 8, 8, 32, generator=torch.Generator().manual_seed(3), dtype=torch.float64))
    xr, gr, br, a = _gn_autograd(x, gam, bet, G, eps, True)
    out = Fnn.conv2d(a.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1)
    out.backward(dy)
    ref = R.conv_gn_backward_ref(x, dy, w, gam, bet, G, eps)
    _close(ref["dx"][0], xr.grad)
    _close(ref["dgamma"][0], gr.grad)
    _close(ref["dbeta"][0], br.grad)


@pytest.mark.parametrize("C", [8, 64, 320, 1024])
def test_rmsnorm_references_match_autograd(C):
    g = torch.Generator().manual_seed(4)
    x = _bf(torch.randn(2, 3, 5, C, generator=g, dtype=torch.float64))
    s = 1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64)
    dy = _bf(torch.randn(2, 3, 5, C, generator=g, dtype=torch.float64))
    xr, sr = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    yr = xr * torch.rsqrt((xr * xr).mean(-1, keepdim=True) + 1e-4) * sr
    yr.backward(dy)
    y, _ = R.rms_forward_ref(x, s, 1e-4)
    _close(y, yr)
    out = R.rms_backward_ref(x, dy, s, 1e-4, 2112)
    _close(out["dx"][0], xr.grad)
    _close(out["dscale"][0], sr.grad)


def test_geglu_references_match_autograd():
    g = torch.Generator().manual_seed(5)
    u = _bf(torch.randn(77, 2 * 1280, generator=g, dtype=torch.float64) * 3)
    u[0, :16] = 0
    dg = _bf(torch.randn(77, 1280, generator=g, dtype=torch.float64))
    ur = u.clone().requires_grad_(True)
    gr = ur[:, :1280] * Fnn.gelu(ur[:, 1280:], approximate="tanh")
    gr.backward(dg)
    _close(R.geglu_forward_ref(u)[0], gr)
    _close(R.geglu_backward_ref(u, dg)[0], ur.grad)


def test_streaming_references_match_autograd():
    g = torch.Generator().manual_seed(6)
    x = _bf(torch.randn(2, 3, 5, 16, generator=g, dtype=torch.float64))
    xr = x.clone().requires_grad_(True)
    up = Fnn.interpolate(xr.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(R.upsample2x_ref(x), up.detach())
    dy = _bf(torch.randn(2, 6, 10, 16, generator=g, dtype=torch.float64))
    up.backward(dy)
    _close(R.upsample2x_bwd_ref(dy), xr.grad)
    _close(R.colsum_ref(x, True), x.sum((1, 2)))
    _close(R.colsum_ref(x, False), x.sum((0, 1, 2)))


def test_ulp_bf16():
    v = torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 2.0 ** -130, 1e30], dtype=torch.float64)
    assert R.ulp_bf16(v).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -6, 2.0 ** -133, 2.0 ** -133,
                                      2.0 ** (math.frexp(1e30)[1] - 8)]


@pytest.mark.parametrize("silu", [False, True])
def test_comparator_accepts_the_rounded_reference(silu):
    x, gam, bet = _gn_inputs((4, 16, 16, 64), 8)
    y, d = R.gn_forward_ref(x, gam, bet, 8, 1e-4, silu)
    R.assert_elementwise(_bf(y), y, R.bf16_bound(y, d), "groupnorm forward")
    dy = _bf(torch.randn(4, 16, 16, 64, dtype=torch.float64))
    out = R.gn_backward_ref(x, dy, gam, bet, 8, 1e-4, silu)
    R.assert_elementwise(_bf(out["dx"][0]), out["dx"][0], R.bf16_bound(*out["dx"]), "dx")
    for k in ("dgamma", "dbeta", "csum_img", "csum_tot"):
        v, dv = out[k]
        R.assert_elementwise(v.float(), v, R.f32_bound(v, dv), k)
    u = _bf(torch.randn(64, 2 * 256, dtype=torch.float64) * 4)
    gv, gd = R.geglu_forward_ref(u)
    R.assert_elementwise(_bf(gv), gv, R.bf16_bound(gv, gd), "geglu")


def test_comparator_rejects_what_relative_l2_accepts():
    """Three confined defects, each invisible to `rel(got, ref) < 1e-2`, each caught element by element."""
    G, eps = 8, 1e-4
    x, gam, bet = _gn_inputs((40, 32, 32, 64), G)
    y, d = R.gn_forward_ref(x, gam, bet, G, eps, True)
    bound = R.bf16_bound(y, d)
    good = _bf(y)
    R.assert_elementwise(good, y, bound)

    zeroed = good.clone()
    zeroed[17, 5, 9] = 0                                         # one pixel of one image never written
    scaled = good.clone()
    scaled[3] = _bf(scaled[3] * (1 + 2.0 ** -5))                 # one image of a cluster off by 2^-5
    # the last channel vector (channels C-8 .. C-1, group G-1) normalised with group G-2's statistics
    xw, gw, bw = _gn_inputs((2, 4, 4, 2048), G)
    yw, dw = R.gn_forward_ref(xw, gw, bw, G, eps, True)
    xg = xw.reshape(2, -1, G, 256)
    mu, r = xg.mean((1, 3)), 1 / torch.sqrt(xg.var((1, 3), unbiased=False) + eps)
    wrong = _bf(yw).clone()
    z = (xw[..., -8:] - mu[:, G - 2].view(2, 1, 1, 1)) * r[:, G - 2].view(2, 1, 1, 1) * gw[-8:] + bw[-8:]
    wrong[..., -8:] = _bf(Fnn.silu(z))

    for got, ref, b in ((zeroed, y, bound), (scaled, y, bound), (wrong, yw, R.bf16_bound(yw, dw))):
        assert rel(got, ref) < 1e-2                             # what the relative-L2 tests accept ...
        with pytest.raises(AssertionError, match="outside the bound"):
            R.assert_elementwise(got, ref, b)                   # ... the element-wise comparator does not

    nan = good.clone()
    nan[0, 0, 0, 0] = math.nan                                  # an element left at its NaN prefill
    with pytest.raises(AssertionError, match="1 of"):
        R.assert_elementwise(nan, y, bound)
