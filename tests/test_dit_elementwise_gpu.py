"""fdx_dit.cu's kernels element by element against float64 references computed from the same bf16 inputs.

Per-element bounds: a bf16 output may differ from the exact value by one bf16 ulp of that value (the store rounding)
plus `delta`, the f32 arithmetic's error before the store; an f32 sum by gamma(n) * sum |terms| (Higham, eq. 4.4, n
the number of terms) plus one f32 rounding.  delta for the row-wise kernels is 2^-18 times the row's scale (the
normalisation's statistics and a handful of f32 roundings), for RoPE 2^-19 times the pair's magnitude (sincosf and
powf are within 2 ulp)."""
import math

import pytest
import torch

from flaxdiff_b200 import ops
from flaxdiff_b200._lib import ACT_GELU_TANH

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
U = 2.0 ** -24


def ulp_bf16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def check_bf16(got, ref, delta, what):
    got, ref = got.double(), ref.double()
    bound = ulp_bf16(ref) + (1 + 2 ** -8) * delta
    err = (got - ref).abs()
    bad = err > bound
    assert not bad.any(), (what, int(bad.sum()), float((err / bound).max()))


def check_f32(got, ref, abs_terms, n, what):
    got, ref = got.double(), ref.double()
    g = n * U / (1 - n * U)
    bound = g * abs_terms + U * ref.abs() + 1e-30
    err = (got - ref).abs()
    assert not (err > bound).any(), (what, float((err / bound).max()))


def bf(shape, scale=1.0, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=dev) * scale).bfloat16()


SHAPES = [(2, 16, 64), (3, 100, 200), (1, 1024, 768), (2, 37, 1152), (2, 16, 1536)]   # (B, L, F)


@pytest.mark.parametrize("B,L,F", SHAPES)
def test_adaln_forward_and_backward(B, L, F):
    x = bf((B * L, F), 2.0, 1).contiguous()
    x = (x.float() + 0.5).bfloat16()
    ada = torch.randn(B, 6 * F, device=dev) * 0.5
    y, mean, rstd = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=1e-5)
    X = x.double()
    mu = X.mean(-1, keepdim=True)
    var = ((X - mu) ** 2).mean(-1, keepdim=True)
    xh = (X - mu) / torch.sqrt(var + 1e-5)
    A = ada.double().repeat_interleave(L, 0)
    sc, sh = A[:, 3 * F:4 * F], A[:, 4 * F:5 * F]
    ref = xh * (1 + sc) + sh
    scale = (xh.abs().amax(-1, keepdim=True) * (1 + sc.abs()) + sh.abs())
    check_bf16(y, ref, 2.0 ** -18 * scale, "adaln_fwd")
    # backward: dx (+ addend) and the per-sample d(scale), d(shift)
    dy = bf((B * L, F), 1.0, 2)
    add = bf((B * L, F), 1.0, 3)
    d_ada = torch.zeros(B, 6 * F, device=dev)
    dx = ops.dit_adaln_bwd(x, dy, L, mean, rstd, d_ada[:, 3 * F:4 * F], d_ada[:, 4 * F:5 * F], ada=ada,
                           scale_off=3 * F, addend=add)
    DY = dy.double()
    g = DY * (1 + sc)
    rs = 1 / torch.sqrt(var + 1e-5)
    ref_dx = rs * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True)) + add.double()
    sdx = rs * (g.abs().amax(-1, keepdim=True) * (1 + xh.abs())) + add.double().abs()
    check_bf16(dx, ref_dx, 2.0 ** -18 * sdx, "adaln_bwd dx")
    t0 = (DY * xh).view(B, L, F)
    check_f32(d_ada[:, 3 * F:4 * F], t0.sum(1), t0.abs().sum(1) * 4, L, "d_scale")
    t1 = DY.view(B, L, F)
    check_f32(d_ada[:, 4 * F:5 * F], t1.sum(1), t1.abs().sum(1), L, "d_shift")
    assert d_ada[:, :3 * F].abs().max() == 0 and d_ada[:, 5 * F:].abs().max() == 0      # other chunks untouched


@pytest.mark.parametrize("B,L,F", SHAPES[:3])
def test_layernorm_affine_backward_reduces_over_samples(B, L, F):
    x = bf((B * L, F), 1.5, 4)
    gamma = torch.rand(F, device=dev) + 0.5
    beta = torch.randn(F, device=dev)
    y, mean, rstd = ops.dit_adaln_fwd(x, L, gamma=gamma, beta=beta, eps=1e-5)
    X = x.double()
    mu = X.mean(-1, keepdim=True)
    var = ((X - mu) ** 2).mean(-1, keepdim=True)
    xh = (X - mu) / torch.sqrt(var + 1e-5)
    ref = xh * gamma.double() + beta.double()
    check_bf16(y, ref, 2.0 ** -18 * (xh.abs().amax(-1, keepdim=True) * gamma.double().abs() + beta.double().abs()),
               "layernorm affine fwd")
    dy = bf((B * L, F), 1.0, 5)
    dg = torch.ones(F, device=dev)
    db = torch.ones(F, device=dev)
    dx = ops.dit_adaln_bwd(x, dy, L, mean, rstd, dg, db, gamma=gamma, reduce_samples=True, accumulate=True)
    DY = dy.double()
    g = DY * gamma.double()
    rs = 1 / torch.sqrt(var + 1e-5)
    ref_dx = rs * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    check_bf16(dx, ref_dx, 2.0 ** -18 * rs * g.abs().amax(-1, keepdim=True) * (1 + xh.abs()), "layernorm affine dx")
    check_f32(dg, 1 + (DY * xh).sum(0), (DY * xh).abs().sum(0) * 4 + 1, B * L + 1, "d_gamma")
    check_f32(db, 1 + DY.sum(0), DY.abs().sum(0) + 1, B * L + 1, "d_beta")


@pytest.mark.parametrize("B,L,F", SHAPES)
def test_gated_residual_forward_and_backward(B, L, F):
    x, y = bf((B * L, F), 1.0, 6), bf((B * L, F), 1.0, 7)
    ada = torch.randn(B, 6 * F, device=dev)
    out = ops.dit_gate_fwd(x, y, L, ada[:, 5 * F:])
    G = ada[:, 5 * F:].double().repeat_interleave(L, 0)
    ref = x.double() + G * y.double()
    check_bf16(out, ref, 4 * U * (x.double().abs() + (G * y.double()).abs()), "gate fwd")
    dout = bf((B * L, F), 1.0, 8)
    dg = torch.zeros(B, 6 * F, device=dev)
    dy = ops.dit_gate_bwd(dout, y, L, ada[:, 5 * F:], dg[:, 5 * F:])
    check_bf16(dy, G * dout.double(), 2 * U * (G * dout.double()).abs(), "gate bwd dy")
    t = (dout.double() * y.double()).view(B, L, F)
    check_f32(dg[:, 5 * F:], t.sum(1), t.abs().sum(1), L + 1, "d_gate")


@pytest.mark.parametrize("L,heads,d", [(16, 2, 32), (100, 4, 48), (1024, 12, 64), (37, 1, 136), (64, 1, 256)])
def test_rope_forward_and_inverse(L, heads, d):
    B = 2
    dp = 32 if d <= 32 else 64 if d <= 64 else 128 if d <= 128 else 256
    HD = heads * dp
    qkv = bf((B * L, 3 * HD), 1.0, 9)
    orig = qkv.clone()
    ops.dit_rope(qkv, L, heads, d, dp, nmat=2, mat_off=HD)
    for m in range(2):
        X = orig[:, m * HD:(m + 1) * HD].double().view(B, L, heads, dp)[..., :d]
        inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float64) / d))
        ang = torch.arange(L, dtype=torch.float64)[:, None] * inv[None]
        cs, sn = ang.cos().repeat(1, 2)[None, :, None], ang.sin().repeat(1, 2)[None, :, None]
        Xc = X.cpu()
        rot = torch.cat([-Xc[..., d // 2:], Xc[..., :d // 2]], -1)
        ref = Xc * cs + rot * sn
        got = qkv[:, m * HD:(m + 1) * HD].view(B, L, heads, dp)
        mag = (Xc.abs() + rot.abs())
        # the angle l * inv_freq is formed in f32: its rounding (|angle| u) moves the result by up to |angle| u |x|
        delta = (2.0 ** -19 + 4 * U * ang.abs().max().item()) * mag
        check_bf16(got[..., :d].cpu(), ref, delta, f"rope m={m}")
        assert (got[..., d:] == 0).all()
    assert torch.equal(qkv[:, 2 * HD:], orig[:, 2 * HD:])                          # v untouched
    # the inverse rotation undoes the forward one (up to the two bf16 roundings)
    back = qkv.clone()
    ops.dit_rope(back, L, heads, d, dp, nmat=2, mat_off=HD, inverse=True)
    o = orig[:, :2 * HD].view(B * L, 2, heads, dp)[..., :d].double()
    b_ = back[:, :2 * HD].view(B * L, 2, heads, dp)[..., :d].double()
    assert ((b_ - o).abs() <= 2 ** -6 * (o.abs().amax(-1, keepdim=True)) + 1e-6).all()


@pytest.mark.parametrize("rows,C", [(7, 64), (1000, 3072), (33, 6144)])
def test_bias_gelu_tanh_forward_and_backward(rows, C):
    x = bf((rows, C), 2.0, 10)
    bias = torch.randn(C, device=dev) * 0.5
    y = ops.bias_act(x, bias, ACT_GELU_TANH)
    z = x.double() + bias.double()
    k = math.sqrt(2 / math.pi)
    th = torch.tanh(k * (z + 0.044715 * z ** 3))
    ref = 0.5 * z * (1 + th)
    scale = z.abs() * (1 + 0.2 * z * z) + 1e-3
    check_bf16(y, ref, 2.0 ** -20 * scale, "gelu_tanh fwd")
    dy = bf((rows, C), 1.0, 11)
    dx = ops.bias_act_bwd(x, bias, ACT_GELU_TANH, dy)
    dref = dy.double() * (0.5 * (1 + th) + 0.5 * z * (1 - th * th) * k * (1 + 3 * 0.044715 * z * z))
    check_bf16(dx, dref, 2.0 ** -19 * dy.double().abs() * scale, "gelu_tanh bwd")


@pytest.mark.parametrize("p", [2, 4, 8, 16])
@pytest.mark.parametrize("src_dtype", [torch.float32, torch.bfloat16])
def test_patchify_and_unpatchify_are_exact_transposes(p, src_dtype):
    B, H, W, C = 2, 2 * p * 3, p * 5, 3
    x = torch.randn(B, H, W, C, device=dev).to(src_dtype)
    K = p * p * C
    ld = -(-K // 32) * 32
    rows = ops.dit_patchify(x, p, ld)
    HP, WP = H // p, W // p
    ref = x.float().reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B * HP * WP, K)
    assert torch.equal(rows[:, :K].float(), ref.bfloat16().float())
    assert (rows[:, K:] == 0).all()
    y = torch.randn(B * HP * WP, ld, device=dev)
    img = ops.dit_unpatchify(y, B, H, W, C, p)
    ref_img = y[:, :K].reshape(B, HP, WP, p, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)
    assert torch.equal(img, ref_img)


@pytest.mark.parametrize("B,T,C", [(2, 77, 768), (3, 5, 64), (1, 1024, 1536)])
def test_token_mean(B, T, C):
    x = bf((B, T, C), 1.0, 12)
    got = ops.dit_token_mean(x)
    X = x.double()
    check_f32(got, X.mean(1), X.abs().sum(1) / T, T + 2, "token_mean")


def test_fourier_features():
    t = torch.rand(5, device=dev) * 2 - 1
    freqs = torch.randn(96, device=dev) * 16
    got = ops.dit_fourier(t, freqs)
    w = (2 * math.pi * freqs.double())
    arg = t.double()[:, None] * w[None]
    ref = torch.cat([arg.sin(), arg.cos()], -1)
    # the f32 argument is within 3 u |arg| of the exact one; sinf / cosf add 2 ulp
    check_bf16(got, ref, 3 * U * torch.cat([arg.abs(), arg.abs()], -1) + 4 * U, "fourier")
