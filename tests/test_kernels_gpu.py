"""Parity of the non-tensor-core libfdx kernels through the C-ABI against the CPU oracle
(oracle/unet_ref.py, oracle/diffusion_ref.py) on identical inputs.  Tolerances: f32 kernels 1e-5
relative; kernels with bf16 outputs 5e-3 (one bf16 rounding); bf16-in/bf16-out backward 1e-2."""
import math

import numpy as np
import pytest
import torch

from flaxdiff_b200 import ops
from oracle import diffusion_ref as R
from oracle import unet_ref as U

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


@pytest.mark.parametrize("shape", [(2, 16, 16, 64), (3, 8, 8, 192), (2, 32, 32, 320), (1, 4, 4, 768), (5, 2, 2, 512),
                                   # >= 1024 pixels per image: many CTAs per image in both backward passes,
                                   # ragged pixel counts, many images
                                   (3, 64, 64, 64), (21, 32, 32, 128), (2, 48, 40, 192), (40, 32, 32, 64)])
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_fwd_bwd(shape, silu):
    torch.manual_seed(0)
    B, H, W, C = shape
    big = (torch.randn(B, H, W, C + 64, device=dev) * 1.5 + 0.3).bfloat16()
    x = big[..., 64:]                                     # strided view (concat slot)
    gamma = 1 + 0.2 * torch.randn(C, device=dev)
    beta = 0.2 * torch.randn(C, device=dev)
    st = ops.groupnorm_stats(x, 8)
    y = ops.groupnorm_apply(x, 8, st, gamma, beta, 1e-4, silu)
    xr = x.float().cpu().requires_grad_(True)
    gr, br = gamma.cpu().requires_grad_(True), beta.cpu().requires_grad_(True)
    yr = U.group_norm(xr, gr, br, 8, 1e-4)
    if silu:
        yr = U.swish(yr)
    assert rel(y, yr) < 5e-3
    dy = torch.randn(B, H, W, C, device=dev).bfloat16()
    yr.backward(dy.float().cpu())
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    dx = torch.empty(B, H, W, C, device=dev, dtype=torch.bfloat16)
    ci, ct = torch.empty(B, C, device=dev), torch.empty(C, device=dev)
    ops.groupnorm_bwd(x, dy, 8, st, gamma, beta, 1e-4, silu, dg, db, dx, csum_img=ci, csum_tot=ct)
    assert rel(dx, xr.grad) < 1e-2
    assert rel(ci, xr.grad.sum((1, 2))) < 2e-2 and rel(ct, xr.grad.sum((0, 1, 2))) < 2e-2
    assert rel(dg, gr.grad) < 5e-3 and rel(db, br.grad) < 5e-3
    base = torch.randn_like(dx.float()).bfloat16()
    dx2 = base.clone()
    dg.zero_(); db.zero_()
    ops.groupnorm_bwd(x, dy, 8, st, gamma, beta, 1e-4, silu, dg, db, dx2, accumulate=True)
    assert rel(dx2, xr.grad + base.float().cpu()) < 1e-2
    # addend from ANOTHER tensor (the ResidualBlock's skip gradient joins inside the kernel), itself a strided slot
    wide = torch.randn(B, H, W, C + 64, device=dev).bfloat16()
    add = wide[..., 64:]
    dx3 = torch.empty_like(dx)
    dg.zero_(); db.zero_()
    ops.groupnorm_bwd(x, dy, 8, st, gamma, beta, 1e-4, silu, dg, db, dx3, addend=add)
    assert rel(dx3, xr.grad + add.float().cpu()) < 1e-2
    if H * W >= 1024:      # dgamma / dbeta again, from the addend call
        assert rel(dg, gr.grad) < 5e-3 and rel(db, br.grad) < 5e-3


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("shape", [(2, 16, 16, 64, 64), (3, 16, 8, 192, 128), (2, 32, 32, 320, 64), (4, 8, 8, 128, 128)])
def test_conv_dgrad_groupnorm_bwd_fused(shape, fused):
    """d/dx of conv3x3(silu(groupnorm(x))): fused dgrad-epilogue path (>= 128 pixels / image) and the
    two-pass fallback (8x8) against autograd on the fp32 oracle."""
    torch.manual_seed(1)
    B, H, W, C, Co = shape
    big = (torch.randn(B, H, W, C + 64, device=dev) * 1.5 + 0.3).bfloat16()
    x = big[..., :C]                                      # strided view (concat slot)
    gamma = 1 + 0.2 * torch.randn(C, device=dev)
    beta = 0.2 * torch.randn(C, device=dev)
    w = (torch.randn(3, 3, C, Co, device=dev) / math.sqrt(9 * C))
    w16 = w.bfloat16()
    dy = torch.randn(B, H, W, Co, device=dev).bfloat16()
    st = ops.groupnorm_stats(x, 8)
    xr = x.float().cpu().requires_grad_(True)
    gr, br = gamma.cpu().requires_grad_(True), beta.cpu().requires_grad_(True)
    yr = U.conv_same(U.swish(U.group_norm(xr, gr, br, 8, 1e-4)), w16.float().cpu(), None)
    yr.backward(dy.float().cpu())
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    dx = torch.empty(B, H, W, C, device=dev, dtype=torch.bfloat16)
    ci, ct = torch.empty(B, C, device=dev), torch.empty(C, device=dev)
    ops.conv_dgrad_groupnorm_bwd(dy, w16, x, 8, st, gamma, beta, 1e-4, dg, db, dx, csum_img=ci, csum_tot=ct, fused=fused)
    assert rel(dx, xr.grad) < 1.2e-2
    assert rel(ci, xr.grad.sum((1, 2))) < 3e-2 and rel(ct, xr.grad.sum((0, 1, 2))) < 3e-2
    assert rel(dg, gr.grad) < 8e-3 and rel(db, br.grad) < 8e-3
    base = torch.randn_like(dx.float()).bfloat16()
    dx2 = base.clone()
    dg.zero_(); db.zero_()
    ops.conv_dgrad_groupnorm_bwd(dy, w16, x, 8, st, gamma, beta, 1e-4, dg, db, dx2, accumulate=True, fused=fused)
    assert rel(dx2, xr.grad + base.float().cpu()) < 1.2e-2
    # the identity-residual gradient as an addend of the second pass (fdx_groupnorm_bwd_add / _bwd_dz_add)
    add = torch.randn(B, H, W, C, device=dev).bfloat16()
    dx3 = torch.empty_like(dx)
    dg.zero_(); db.zero_()
    ops.conv_dgrad_groupnorm_bwd(dy, w16, x, 8, st, gamma, beta, 1e-4, dg, db, dx3, fused=fused, addend=add)
    assert rel(dx3, xr.grad + add.float().cpu()) < 1.2e-2
    assert rel(dg, gr.grad) < 8e-3 and rel(db, br.grad) < 8e-3


@pytest.mark.parametrize("C", [256, 512])
def test_rmsnorm_fwd_bwd(C):
    torch.manual_seed(0)
    x = torch.randn(2, 8, 8, C, device=dev).bfloat16()
    scale = 1 + 0.2 * torch.randn(C, device=dev)
    y = ops.rmsnorm_fwd(x, scale, 1e-4)
    xr, sr = x.float().cpu().requires_grad_(True), scale.cpu().requires_grad_(True)
    yr = U.rms_norm(xr, sr, 1e-4)
    assert rel(y, yr) < 5e-3
    dy = torch.randn_like(x.float()).bfloat16()
    yr.backward(dy.float().cpu())
    dx = torch.empty_like(x)
    ds = torch.zeros(C, device=dev)
    ops.rmsnorm_bwd(x, dy, scale, 1e-4, dx, ds)
    assert rel(dx, xr.grad) < 1e-2 and rel(ds, sr.grad) < 5e-3


# B = 256, 64x64x3 (BASELINE): B*E/4 = 786,432 four-element items over 8*SMs*256 = 270,336 threads (132 SMs), so
# the grid-stride loop runs about three times and the per-sample index b changes inside a thread's sweep
BASELINE_BH = (256, 64)


@pytest.mark.parametrize("kind,u8,B,H", [pytest.param(k, u, 5, 16, id=f"{k}-{u}") for k in (0, 1, 2) for u in (True, False)] +
                         [pytest.param(k, u, *BASELINE_BH, id=f"{k}-{u}-B256") for k in (0, 1, 2) for u in (True, False)])
def test_diffuse_forward(u8, kind, B, H):
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (B, H, H, 3), dtype=np.uint8)
    x0 = img if u8 else img.astype(np.float32)
    eps = rng.standard_normal((B, H, H, 3), dtype=np.float32)
    sigma = np.resize(np.array([0.002, 0.3, 1.0, 7.0, 80.0], dtype=np.float32), B)
    alpha = np.ones(B, np.float32) if kind == 0 else np.sqrt(np.maximum(1 - np.minimum(sigma, 0.99) ** 2, 0)).astype(np.float32)
    c_in, _, _ = R.karras_coeffs(sigma)
    x_t, tgt, mi = ops.diffuse_forward(torch.from_numpy(x0).to(dev), torch.from_numpy(eps).to(dev),
                                       torch.from_numpy(alpha).to(dev), torch.from_numpy(sigma).to(dev),
                                       torch.from_numpy(c_in).to(dev), True, kind)
    data = (img.astype(np.float32) - 127.5) / 127.5
    want = R.forward_diffusion(data, eps, alpha, sigma)
    np.testing.assert_allclose(x_t.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    a4, s4 = alpha.reshape(-1, 1, 1, 1), sigma.reshape(-1, 1, 1, 1)
    wt = [data, eps, (a4 * eps - s4 * data) / np.sqrt(a4 ** 2 + s4 ** 2)][kind]
    np.testing.assert_allclose(tgt.cpu().numpy(), wt, rtol=2e-6, atol=2e-6)
    assert rel(mi, torch.from_numpy(want * c_in.reshape(-1, 1, 1, 1))) < 4e-3


def test_loss_fwd_bwd():
    for B, H in ((4, 16), BASELINE_BH):
        rng = np.random.default_rng(1)
        F, x_t, tg = (rng.standard_normal((B, H, H, 3), dtype=np.float32) for _ in range(3))
        sigma = np.resize(np.array([0.01, 0.5, 2.0, 50.0], dtype=np.float32), B)
        _, c_out, c_skip = R.karras_coeffs(sigma)
        w = R.karras_weight(sigma)
        Ft = torch.from_numpy(F).to(dev)
        loss, dF = ops.loss_fwd_bwd(Ft, torch.from_numpy(x_t).to(dev), torch.from_numpy(tg).to(dev),
                                    torch.from_numpy(c_out).to(dev), torch.from_numpy(c_skip).to(dev),
                                    torch.from_numpy(w).to(dev))
        pred = c_out.reshape(-1, 1, 1, 1) * F + c_skip.reshape(-1, 1, 1, 1) * x_t
        want = R.weighted_l2_loss(pred, tg, w)
        assert abs(loss.item() - want) / want < 1e-5
        Fr = torch.from_numpy(F).requires_grad_(True)
        pr = torch.from_numpy(c_out).view(-1, 1, 1, 1) * Fr + torch.from_numpy(c_skip).view(-1, 1, 1, 1) * torch.from_numpy(x_t)
        (0.5 * (pr - torch.from_numpy(tg)) ** 2 * torch.from_numpy(w).view(-1, 1, 1, 1)).mean().backward()
        assert rel(dF, Fr.grad) < 1e-5


def test_affine_combine_sampler_rules():
    for B, H in ((3, 8), BASELINE_BH):
        rng = np.random.default_rng(2)
        x, x0, noise = (torch.from_numpy(rng.standard_normal((B, H, H, 3), dtype=np.float32)).to(dev) for _ in range(3))
        cs = np.resize(np.array([80.0, 3.0, 0.5], dtype=np.float32), B)
        ns = np.resize(np.array([40.0, 1.0, 0.1], dtype=np.float32), B)
        one = np.ones(B, np.float32)
        from flaxdiff_b200.predictors import _affine
        t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
        dt = ns - cs
        k = (one * ns - one * cs) / dt
        g = dt / cs
        got = _affine([x, x0], [t(1 + g), t(-k * g)])
        want = R.euler_step(x.cpu().numpy(), x0.cpu().numpy(), one, cs, one, ns)
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=2e-5, atol=2e-5)
        up = (ns ** 2 * (cs ** 2 - ns ** 2) / cs ** 2) ** 0.5
        down = (ns ** 2 - up ** 2) ** 0.5
        g2 = (down - cs) / cs
        got = _affine([x, x0, noise], [t(1 + g2), t(-k * g2), t(up)])
        want = R.euler_ancestral_step(x.cpu().numpy(), x0.cpu().numpy(), noise.cpu().numpy(), one, cs, one, ns)
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=2e-5, atol=2e-5)
        o1, o2 = _affine([x, x0], [t(one), t(one * 2)], [t(one * 0), t(one * -1)])
        np.testing.assert_allclose(o2.cpu().numpy(), -x0.cpu().numpy(), rtol=0, atol=0)
        out, _, _ = ops.affine_combine([x.contiguous()], torch.ones(1, B, device=dev), clip=(-1.0, 1.0))
        assert out.max().item() <= 1.0 and out.min().item() >= -1.0


def test_adamw_ema_matches_oracle():
    rng = np.random.default_rng(3)
    n = 4096
    p, g, m, v = (rng.standard_normal(n).astype(np.float32) for _ in range(4))
    v = np.abs(v)
    ema = p.copy()
    tp, tg, tm, tv, te = (torch.from_numpy(a.copy()).to(dev) for a in (p, g, m, v, ema))
    sh = torch.empty(n, dtype=torch.bfloat16, device=dev)
    ops.adamw_ema_step(tp, tg, tm, tv, te, sh, 2.7e-4, 0.9, 0.999, 1e-8, 1e-4, 7, 0.999, grad_scale=0.5)
    wp, wm, wv, we = R.adamw_ema(p.astype(np.float64), 0.5 * g.astype(np.float64), m.astype(np.float64),
                                 v.astype(np.float64), ema.astype(np.float64), 7, 2.7e-4, wd=1e-4)
    np.testing.assert_allclose(tp.cpu().numpy(), wp, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(tm.cpu().numpy(), wm, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(tv.cpu().numpy(), wv, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(te.cpu().numpy(), we, rtol=1e-5, atol=1e-7)
    assert rel(sh, torch.from_numpy(wp)) < 4e-3
    # device-side hyper-parameters (CUDA-graph path) give the same update
    tp2, tm2, tv2, te2 = (torch.from_numpy(a.copy()).to(dev) for a in (p, m, v, ema))
    dyn = torch.tensor([2.7e-4, 1 - 0.9 ** 7, 1 - 0.999 ** 7], device=dev)
    ops.adamw_ema_step(tp2, tg, tm2, tv2, te2, None, 1.0, 0.9, 0.999, 1e-8, 1e-4, 1, 0.999, grad_scale=0.5, dyn=dyn)
    np.testing.assert_allclose(tp2.cpu().numpy(), tp.cpu().numpy(), rtol=1e-6, atol=1e-8)


def test_conv_in_out_and_grads():
    torch.manual_seed(0)
    B, H = 2, 16
    x = torch.randn(B, H, H, 3, device=dev).bfloat16()
    w_in = torch.randn(3, 3, 3, 64, device=dev) * 0.2
    b_in = torch.randn(64, device=dev) * 0.1
    y = torch.empty(B, H, H, 64, device=dev, dtype=torch.bfloat16)
    ops.conv_in_fwd(x, w_in, b_in, y)             # im2col + tensor-core GEMM (bf16 weights)
    wr, br = w_in.cpu().requires_grad_(True), b_in.cpu().requires_grad_(True)
    yr = U.conv_same(x.float().cpu(), wr, br)
    assert rel(y, yr) < 6e-3
    y2 = torch.empty_like(y)
    ops.conv_in_fwd_direct(x, w_in, b_in, y2)     # CUDA-core variant (f32 weights)
    assert rel(y2, yr) < 5e-3
    dy = torch.randn(B, H, H, 64, device=dev).bfloat16()
    yr.backward(dy.float().cpu())
    dw, dbi = torch.zeros_like(w_in), torch.zeros_like(b_in)
    ops.conv_in_wgrad(x, dy, dw, dbi)
    assert rel(dw, wr.grad) < 1e-4 and rel(dbi, br.grad) < 1e-4
    a = torch.randn(B, H, H, 64, device=dev).bfloat16()
    w_out = torch.randn(3, 3, 64, 3, device=dev) * 0.1
    b_out = torch.randn(3, device=dev) * 0.1
    Fo = ops.conv_out_fwd(a, w_out, b_out)
    ar, wo, bo = a.float().cpu().requires_grad_(True), w_out.cpu().requires_grad_(True), b_out.cpu().requires_grad_(True)
    Fr = U.conv_same(ar, wo, bo)
    assert rel(Fo, Fr) < 5e-3                     # tensor-core GEMM (bf16 weights) + col2im scatter
    assert rel(ops.conv_out_fwd_direct(a, w_out, b_out), Fr) < 1e-5   # CUDA-core variant, f32 weights
    dF = torch.randn(B, H, H, 3, device=dev)
    Fr.backward(dF.cpu())
    da = torch.empty_like(a)
    ops.conv_out_dgrad(dF, w_out, da)             # im2col + tensor-core GEMM (dF and weights in bf16)
    assert rel(da, ar.grad) < 8e-3
    da2 = torch.empty_like(a)
    ops.conv_out_dgrad_direct(dF, w_out, da2)
    assert rel(da2, ar.grad) < 5e-3
    dwo, dbo = torch.zeros_like(w_out), torch.zeros_like(b_out)
    ops.conv_out_wgrad(a, dF, dwo, dbo)          # im2col + tensor-core GEMM (dF rounded to bf16)
    assert rel(dwo, wo.grad) < 5e-3 and rel(dbo, bo.grad) < 5e-3
    dwo2, dbo2 = torch.zeros_like(w_out), torch.zeros_like(b_out)
    ops.conv_out_wgrad_direct(a, dF, dwo2, dbo2)  # CUDA-core variant, f32 dF
    assert rel(dwo2, wo.grad) < 1e-4 and rel(dbo2, bo.grad) < 1e-4
    dw2, dbi2 = torch.zeros_like(w_in), torch.zeros_like(b_in)
    ops.conv_in_wgrad_direct(x, dy, dw2, dbi2)
    assert rel(dw2, wr.grad) < 1e-4 and rel(dbi2, br.grad) < 1e-4


def test_time_embedding_fwd_bwd():
    torch.manual_seed(0)
    from flaxdiff_b200 import utils
    B, D = 6, 256
    freqs = torch.from_numpy(utils.normal(utils.PRNGKey(42), D // 2) * 16.0).to(dev)
    W1, W2 = torch.randn(D, D, device=dev) / 16, torch.randn(D, D, device=dev) / 16
    b1, b2 = torch.randn(D, device=dev) * 0.1, torch.randn(D, device=dev) * 0.1
    t = torch.tensor([-1.5, -0.3, 0.0, 0.27, 1.0, 1.0955], device=dev)      # EDM / Karras model-time range
    emb, emb16, saved = ops.time_embed_fwd(t, freqs, W1, b1, W2, b2)
    P = {"TimeProjection_0/DenseGeneral_0/kernel": W1.cpu().requires_grad_(True),
         "TimeProjection_0/DenseGeneral_0/bias": b1.cpu().requires_grad_(True),
         "TimeProjection_0/DenseGeneral_1/kernel": W2.cpu().requires_grad_(True),
         "TimeProjection_0/DenseGeneral_1/bias": b2.cpu().requires_grad_(True)}
    er = U.time_embedding(t.cpu(), freqs.cpu(), P)
    assert rel(emb, er) < 2e-5 and rel(emb16, er) < 4e-3
    de = torch.randn(B, D, device=dev)
    er.backward(de.cpu())
    dW1, dW2, db1, db2 = (torch.zeros_like(a) for a in (W1, W2, b1, b2))
    ops.time_embed_bwd(de, saved, W2, dW1, db1, dW2, db2)
    for got, name in ((dW1, "0/kernel"), (db1, "0/bias"), (dW2, "1/kernel"), (db2, "1/bias")):
        assert rel(got, P["TimeProjection_0/DenseGeneral_" + name].grad) < 5e-5, name


def test_time_embedding_large_integer_steps():
    """DDPM integer timesteps (t <= 999): phases reach ~1e5 rad; f32 sin is ill-conditioned there, so
    parity is judged at a loose tolerance (SURVEY.md $7 'hard parts')."""
    from flaxdiff_b200 import utils
    D = 256
    freqs = torch.from_numpy(utils.normal(utils.PRNGKey(42), D // 2) * 16.0).to(dev)
    eye = torch.eye(D, device=dev)
    z = torch.zeros(D, device=dev)
    t = torch.tensor([0.0, 1.0, 17.0, 500.0, 999.0], device=dev)
    _, _, (four, _, _) = ops.time_embed_fwd(t, freqs, eye, z, eye, z)
    ph = t.cpu()[:, None] * (torch.tensor(2 * math.pi, dtype=torch.float32) * freqs.cpu())[None, :]
    want = torch.cat([torch.sin(ph), torch.cos(ph)], -1)
    assert (four.cpu() - want).abs().max().item() < 2e-2


def test_softmax_fwd_bwd():
    torch.manual_seed(0)
    S = torch.randn(2, 8, 64, 64, device=dev) * 3
    Pm = ops.softmax_fwd(S)
    Sr = S.cpu().requires_grad_(True)
    Pr = torch.softmax(Sr, -1)
    assert rel(Pm, Pr) < 4e-3
    dP = torch.randn_like(S)
    (Pr * dP.cpu()).sum().backward()
    dS = ops.softmax_bwd(Pm, dP, 0.5)
    assert rel(dS, 0.5 * Sr.grad) < 1e-2


def test_upsample_colsum_add():
    torch.manual_seed(0)
    x = torch.randn(2, 4, 4, 64, device=dev).bfloat16()
    u = ops.upsample2x(x)
    assert torch.equal(u, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    du = torch.randn(2, 8, 8, 64, device=dev).bfloat16()
    dx = torch.empty_like(x)
    ops.upsample2x_bwd(du, dx)
    want = du.float().view(2, 4, 2, 4, 2, 64).sum((2, 4))
    assert rel(dx, want) < 5e-3
    cs = ops.colsum(du, per_image=True)
    assert rel(cs, du.float().sum((1, 2))) < 1e-5
    assert rel(ops.colsum(du, per_image=False), du.float().sum((0, 1, 2))) < 1e-5
    y = torch.randn_like(x.float()).bfloat16()
    o = torch.empty_like(x)
    ops.act_add(x, y, o)
    assert rel(o, x.float() + y.float()) < 4e-3


@pytest.mark.parametrize("shape", [(2, 8, 8, 128, 64), (3, 16, 16, 64, 128), (2, 4, 4, 512, 64), (2, 16, 8, 256, 192)])
def test_upconv3x3_subpixel_fwd_dgrad_wgrad(shape):
    """nearest-2x + conv3x3 (common.py:210-226) as four 2x2 parity convolutions: forward, data gradient
    (plain and accumulating) and weight gradient against autograd on the fp32 oracle."""
    torch.manual_seed(3)
    B, h, w, cin, cout = shape
    big = torch.randn(B, h, w, cin + 64, device=dev).bfloat16()
    x = big[..., 64:]                                           # strided view (concat slot)
    wt = torch.randn(3, 3, cin, cout, device=dev) / math.sqrt(9 * cin)
    bias = torch.randn(cout, device=dev) * 0.1
    weff = ops.upconv3x3_pack(wt)
    ybig = torch.zeros(B, 2 * h, 2 * w, cout + 64, device=dev, dtype=torch.bfloat16)
    y = ybig[..., :cout]
    ops.upconv3x3_fwd(x, weff, bias, y)
    xr = x.float().cpu().requires_grad_(True)
    wr, br = wt.cpu().requires_grad_(True), bias.cpu().requires_grad_(True)
    up = xr.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    yr = U.conv_same(up, wr, br)
    assert rel(y, yr) < 6e-3
    assert float(ybig[..., cout:].abs().max()) == 0.0           # neighbouring slot untouched
    dy = torch.randn(B, 2 * h, 2 * w, cout, device=dev).bfloat16()
    yr.backward(dy.float().cpu())
    dx = torch.empty(B, h, w, cin, device=dev, dtype=torch.bfloat16)
    ops.upconv3x3_dgrad(dy, weff, dx)
    assert rel(dx, xr.grad) < 8e-3
    base = torch.randn(B, h, w, cin, device=dev).bfloat16()
    dx2 = base.clone()
    ops.upconv3x3_dgrad(dy, weff, dx2, accumulate=True)
    assert rel(dx2, xr.grad + base.float().cpu()) < 8e-3
    dw = torch.zeros_like(wt)
    ops.upconv3x3_wgrad(x, dy, dw)
    assert rel(dw, wr.grad) < 5e-3
    ops.upconv3x3_wgrad(x, dy, dw)                              # accumulates
    assert rel(dw, 2 * wr.grad) < 5e-3


@pytest.mark.parametrize("case", [(2, 16, 16, 64, 64, 1, 0), (3, 32, 32, 128, 192, 1, 64), (2, 32, 32, 64, 128, 2, 128),
                                  (2, 16, 8, 320, 64, 1, 0)])
def test_conv_fwd_fused_groupnorm_statistics(case):
    """fdx_conv3x3_fwd_stats / fdx_upconv3x3_fwd_stats: the per-image channel sums accumulated by the
    epilogue reproduce fdx_groupnorm_stats of the stored bf16 output (same values, different order)."""
    torch.manual_seed(5)
    B, h, w, cin, cout, stride, coff = case
    x = torch.randn(B, h, w, cin, device=dev).bfloat16()
    wt = (torch.randn(3, 3, cin, cout, device=dev) / math.sqrt(9 * cin)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    ho, wo = h // stride, w // stride
    buf = torch.zeros(B, ho, wo, coff + cout + 64, device=dev, dtype=torch.bfloat16)
    y = buf[..., coff:coff + cout]
    res = torch.randn(B, ho, wo, cout, device=dev).bfloat16() if stride == 1 else None
    cs = ops.ColStats(B, buf.shape[-1], dev)
    ops.conv3x3_fwd(x, wt, bias, res=res, out=y, stride=stride, colstats=(cs, coff))
    y2 = torch.empty(B, ho, wo, cout, device=dev, dtype=torch.bfloat16)
    ops.conv3x3_fwd(x, wt, bias, res=res, out=y2, stride=stride)
    assert torch.equal(y, y2)                                   # the statistics do not change the output
    st = ops.groupnorm_stats_from_cols(cs, 8, coff, cout)
    ref = ops.groupnorm_stats(y, 8)
    assert rel(st, ref) < 1e-5
    # GroupNorm(+SiLU) straight from the column sums (fdx_groupnorm_apply_cols) = stats_from_cols + apply
    gamma, beta = 1 + 0.2 * torch.randn(cout, device=dev), 0.2 * torch.randn(cout, device=dev)
    a_ref = ops.groupnorm_apply(y, 8, st, gamma, beta, 1e-4, True)
    a_one, st_one = ops.groupnorm_apply_cols(y, 8, cs, coff, gamma, beta, 1e-4, True)
    assert rel(st_one, st) < 1e-6 and rel(a_one, a_ref) < 1e-3
    # the sub-pixel upsample convolution: four parity launches add up to the same sums
    wf = torch.randn(3, 3, cin, cout, device=dev) / math.sqrt(9 * cin)
    weff = ops.upconv3x3_pack(wf)
    ubuf = torch.zeros(B, 2 * h, 2 * w, coff + cout, device=dev, dtype=torch.bfloat16)
    yu = ubuf[..., coff:]
    cs2 = ops.ColStats(B, ubuf.shape[-1], dev)
    ops.upconv3x3_fwd(x, weff, bias, yu, colstats=(cs2, coff))
    assert rel(ops.groupnorm_stats_from_cols(cs2, 8, coff, cout), ops.groupnorm_stats(yu, 8)) < 1e-5
