"""fdx_mmdit.cu's kernels element by element against float64 references computed from the same bf16 inputs, with the
bounds of test_dit_elementwise_gpu.py: a bf16 output within one bf16 ulp of the exact value plus `delta` (the f32
arithmetic's error before the store), an f32 sum within gamma(n) * sum |terms| plus one f32 rounding.

The ada rows carry MLP scale / shift values on both sides of the clip at +-10 and exactly on it, so the clipped forward
and the clip's derivative (1 inside, 0 outside, 1/2 at a tie) are both exercised.  Each kernel is also run twice and
compared bit for bit, and run in place where its ABI allows (the gated residual onto x, dx onto the addend)."""
import pytest
import torch

from flaxdiff_b200 import ops
from test_dit_elementwise_gpu import bf, check_bf16, check_f32

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

SHAPES = [(3, 37, 8), (2, 100, 64), (1, 1024, 768), (2, 33, 1536), (5, 7, 1536)]   # (B, L, C): ragged and full rows
TIES = torch.tensor([10.0, -10.0, 10.5, -10.5, 9.99, -9.99, 30.0, -30.0, 0.0])


def _ada(B, C, seed):
    """f32 [B, 6C] with ordinary values, the MLP scale / shift chunks seeded with clip ties and overshoots."""
    g = torch.Generator(device=dev).manual_seed(seed)
    ada = torch.randn(B, 6 * C, generator=g, device=dev) * 0.5
    for chunk in (0, 1):
        idx = torch.randint(0, B * C, (max(1, B * C // 4),), generator=g, device=dev)
        vals = TIES.to(dev)[torch.randint(0, len(TIES), idx.shape, generator=g, device=dev)]
        ada[:, chunk * C:(chunk + 1) * C].reshape(-1)[idx] = vals
    return ada


def _clip_grad(v):
    inside = ((v > -10) & (v < 10)).double()
    return inside + 0.5 * ((v == 10) | (v == -10)).double()


def _ln(x):
    X = x.double()
    mu = X.mean(-1, keepdim=True)
    var = ((X - mu) ** 2).mean(-1, keepdim=True)
    return (X - mu) / torch.sqrt(var + 1e-5), 1 / torch.sqrt(var + 1e-5)


@pytest.mark.parametrize("B,L,C", SHAPES)
def test_adaln_forward(B, L, C):
    x = (bf((B * L, C), 2.0, 1).float() + 0.5).bfloat16()
    ada = _ada(B, C, 2)
    ya, ym, mean, rstd = ops.mmdit_adaln_fwd(x, L, ada)
    xh, rs = _ln(x)
    A = ada.double().repeat_interleave(L, 0)
    sa, ha = A[:, 3 * C:4 * C], A[:, 4 * C:5 * C]
    sm, hm = A[:, 0:C].clamp(-10, 10), A[:, C:2 * C].clamp(-10, 10)
    check_bf16(ya, xh * (1 + sa) + ha, 2.0 ** -18 * (xh.abs().amax(-1, keepdim=True) * (1 + sa.abs()) + ha.abs()),
               "y_attn")
    check_bf16(ym, xh * (1 + sm) + hm, 2.0 ** -18 * (xh.abs().amax(-1, keepdim=True) * (1 + sm.abs()) + hm.abs()),
               "y_mlp")
    X = x.double()
    torch.testing.assert_close(mean.double(), X.mean(-1), rtol=0, atol=2.0 ** -18 * X.abs().amax().item())
    torch.testing.assert_close(rstd.double(), rs[:, 0], rtol=2.0 ** -18, atol=0)
    again = ops.mmdit_adaln_fwd(x, L, ada)
    assert all(torch.equal(a, b) for a, b in zip((ya, ym, mean, rstd), again))
    ya2, ym2, none_m, none_r = ops.mmdit_adaln_fwd(x, L, ada, stats=False)
    assert torch.equal(ya2, ya) and torch.equal(ym2, ym) and none_m is None and none_r is None


@pytest.mark.parametrize("B,L,C", SHAPES)
def test_adaln_backward(B, L, C):
    x = (bf((B * L, C), 2.0, 1).float() + 0.5).bfloat16()
    ada = _ada(B, C, 3)
    _, _, mean, rstd = ops.mmdit_adaln_fwd(x, L, ada)
    dya, dym, add = bf((B * L, C), 1.0, 4), bf((B * L, C), 1.0, 5), bf((B * L, C), 1.0, 6)
    d_ada = torch.full((B, 6 * C), 7.0, device=dev)
    dx = ops.mmdit_adaln_bwd(x, dya, dym, L, ada, mean, rstd, d_ada, addend=add)
    xh, rs = _ln(x)
    A = ada.double().repeat_interleave(L, 0)
    sa, sm = A[:, 3 * C:4 * C], A[:, 0:C].clamp(-10, 10)
    DA, DM = dya.double(), dym.double()
    g = DA * (1 + sa) + DM * (1 + sm)
    ref_dx = rs * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True)) + add.double()
    sdx = rs * ((DA.abs() * (1 + sa.abs()) + DM.abs() * (1 + sm.abs())).amax(-1, keepdim=True) * (1 + xh.abs()))
    check_bf16(dx, ref_dx, 2.0 ** -18 * (sdx + add.double().abs()), "dx")
    for chunk, dy, weighted in ((3, DA, True), (4, DA, False), (0, DM, True), (1, DM, False)):
        t = (dy * xh if weighted else dy).view(B, L, C)
        ref = t.sum(1)
        terms = t.abs().sum(1) * (4 if weighted else 1)
        if chunk in (0, 1):
            mask = _clip_grad(ada[:, chunk * C:(chunk + 1) * C].double())
            ref, terms = ref * mask, terms * mask
        check_f32(d_ada[:, chunk * C:(chunk + 1) * C], ref, terms, L, f"d_ada chunk {chunk}")
    assert (d_ada[:, 2 * C:3 * C] == 7).all() and (d_ada[:, 5 * C:] == 7).all()   # the gate chunks are not touched
    # bitwise repeatable, and in place onto the addend
    d2 = torch.zeros_like(d_ada)
    dx2 = ops.mmdit_adaln_bwd(x, dya, dym, L, ada, mean, rstd, d2, addend=add)
    assert torch.equal(dx2, dx) and torch.equal(d2[:, :2 * C], d_ada[:, :2 * C])
    assert torch.equal(d2[:, 3 * C:5 * C], d_ada[:, 3 * C:5 * C])
    inplace = add.clone()
    ops.mmdit_adaln_bwd(x, dya, dym, L, ada, mean, rstd, d2, addend=inplace, out=inplace)
    assert torch.equal(inplace, dx)


@pytest.mark.parametrize("B,L,C", SHAPES + [(2, 64, 3072)])
def test_gate_forward(B, L, C):
    x, ya, ym = bf((B * L, C), 1.0, 1), bf((B * L, C), 1.0, 2), bf((B * L, C), 1.0, 3)
    ada = _ada(B, C, 4)
    out = ops.mmdit_gate_fwd(x, ya, ym, L, ada)
    A = ada.double().repeat_interleave(L, 0)
    ga, gm = A[:, 5 * C:], A[:, 2 * C:3 * C]
    ref = x.double() + ga * ya.double() + gm * ym.double()
    delta = 2.0 ** -22 * (x.double().abs() + (ga * ya.double()).abs() + (gm * ym.double()).abs())
    check_bf16(out, ref, delta, "gate_fwd")
    assert torch.equal(ops.mmdit_gate_fwd(x, ya, ym, L, ada), out)
    xi = x.clone()
    ops.mmdit_gate_fwd(xi, ya, ym, L, ada, out=xi)
    assert torch.equal(xi, out)


@pytest.mark.parametrize("B,L,C", SHAPES + [(2, 64, 3072)])
def test_gate_backward(B, L, C):
    dout, ya, ym = bf((B * L, C), 1.0, 1), bf((B * L, C), 1.0, 2), bf((B * L, C), 1.0, 3)
    ada = _ada(B, C, 5)
    d_ada = torch.full((B, 6 * C), 7.0, device=dev)
    dya, dym = ops.mmdit_gate_bwd(dout, ya, ym, L, ada, d_ada)
    A = ada.double().repeat_interleave(L, 0)
    D = dout.double()
    for got, gate, what in ((dya, A[:, 5 * C:], "dy_attn"), (dym, A[:, 2 * C:3 * C], "dy_mlp")):
        check_bf16(got, gate * D, 2.0 ** -24 * (gate * D).abs(), what)
    for chunk, y in ((5, ya), (2, ym)):
        t = (D * y.double()).view(B, L, C)
        check_f32(d_ada[:, chunk * C:(chunk + 1) * C], t.sum(1), t.abs().sum(1), L, f"d_gate chunk {chunk}")
    for chunk in (0, 1, 3, 4):
        assert (d_ada[:, chunk * C:(chunk + 1) * C] == 7).all()
    d2 = torch.zeros_like(d_ada)
    dya2, dym2 = ops.mmdit_gate_bwd(dout, ya, ym, L, ada, d2)
    assert torch.equal(dya2, dya) and torch.equal(dym2, dym)
    assert torch.equal(d2[:, 2 * C:3 * C], d_ada[:, 2 * C:3 * C]) and torch.equal(d2[:, 5 * C:], d_ada[:, 5 * C:])


def test_refusals():
    x = bf((64, 1544), 1.0, 1)
    ada = torch.zeros(1, 6 * 1544, device=dev)
    with pytest.raises(Exception, match="C=1544"):
        ops.mmdit_adaln_fwd(x, 64, ada)
    x = bf((64, 64), 1.0, 1)
    with pytest.raises(AssertionError):
        ops.mmdit_adaln_fwd(x, 64, torch.zeros(1, 5 * 64, device=dev))      # ada rows shorter than 6 C


# ---------------------------------------------------------------------- fdx_layernorm_rows: gather / concat / scatter
def _merge(x, B, HP, WP):
    C = x.shape[-1]
    return x.reshape(B, HP // 2, 2, WP // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C)


def _expand(y, B, HPc, WPc):
    C = y.shape[-1] // 4
    return y.reshape(B, HPc, WPc, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, C)


ROW_CASES = [("gather", 2, 6, 4, 64), ("gather", 1, 4, 8, 1536), ("gather", 3, 2, 2, 8),
             ("concat", 3, 37, 1, 64), ("concat", 2, 16, 1, 3072), ("concat", 1, 5, 1, 8),
             ("scatter", 2, 3, 2, 256), ("scatter", 1, 2, 4, 1536), ("scatter", 5, 1, 1, 8)]


@pytest.mark.parametrize("mode,B,H_,W_,Cin", ROW_CASES)
def test_layernorm_rows_forward_and_backward(mode, B, H_, W_, Cin):
    """gather: a fine grid H_ x W_ of Cin-wide rows -> C = 4 Cin (up to 6144); concat: B * H_ rows of [Cin, Cin]
    -> C = 2 Cin; scatter: a coarse grid H_ x W_ of C = 4 Cin rows -> fine rows.  Both accumulate settings."""
    code = {"gather": ops.LN_GATHER, "concat": ops.LN_CONCAT, "scatter": ops.LN_SCATTER}[mode]
    if mode == "gather":
        src0, src1 = (bf((B * H_ * W_, Cin), 2.0, 1).float() + 0.3).bfloat16(), None
        rows, C, grid = B * (H_ // 2) * (W_ // 2), 4 * Cin, (H_ // 2, W_ // 2)
        X = _merge(src0.double(), B, H_, W_)
    elif mode == "concat":
        src0, src1 = bf((B * H_, Cin), 2.0, 1), (bf((B * H_, Cin), 1.0, 2).float() - 0.4).bfloat16()
        rows, C, grid = B * H_, 2 * Cin, (0, 0)
        X = torch.cat([src0.double(), src1.double()], -1)
    else:
        src0, src1 = (bf((B * H_ * W_, 4 * Cin), 2.0, 1).float() + 0.3).bfloat16(), None
        rows, C, grid = B * H_ * W_, 4 * Cin, (H_, W_)
        X = src0.double()
    g = torch.Generator(device=dev).manual_seed(9)
    gamma = 1 + 0.3 * torch.randn(C, generator=g, device=dev)
    beta = 0.3 * torch.randn(C, generator=g, device=dev)
    y, mean, rstd = ops.layernorm_rows_fwd(code, src0, src1, rows, C, gamma, beta, 1e-5, grid=grid)
    mu = X.mean(-1, keepdim=True)
    rs = 1 / torch.sqrt(((X - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
    xh = (X - mu) * rs
    ref = xh * gamma.double() + beta.double()
    delta = 2.0 ** -18 * (xh.abs().amax(-1, keepdim=True) * gamma.double().abs() + beta.double().abs())
    if mode == "scatter":
        ref, delta = _expand(ref, B, H_, W_), _expand(delta.expand_as(ref), B, H_, W_)
    check_bf16(y, ref, delta, f"{mode} forward")
    assert all(torch.equal(a, b) for a, b in zip((y, mean, rstd), ops.layernorm_rows_fwd(
        code, src0, src1, rows, C, gamma, beta, 1e-5, grid=grid)))
    # backward: dy in y's layout
    dy = bf(tuple(y.shape), 1.0, 3)
    DY = _merge(dy.double(), B, 2 * H_, 2 * W_) if mode == "scatter" else dy.double()
    dgam = torch.zeros(C, device=dev)
    dbet = torch.zeros(C, device=dev)
    G = DY * gamma.double()
    ref_dx = rs * (G - G.mean(-1, keepdim=True) - xh * (G * xh).mean(-1, keepdim=True))
    sdx = rs * G.abs().amax(-1, keepdim=True) * (1 + xh.abs())
    for acc in (False, True):
        prior = [bf(tuple(t.shape), 1.0, 7 + i) if t is not None else None for i, t in enumerate((src0, src1))]
        d0 = prior[0].clone() if acc else None
        d1 = prior[1].clone() if acc and src1 is not None else None
        d0, d1 = ops.layernorm_rows_bwd(code, src0, src1, dy, rows, C, gamma, mean, rstd, dgam, dbet, grid=grid,
                                        dx0=d0, dx1=d1, accumulate0=acc, accumulate1=acc)
        want, bound = ref_dx, 2.0 ** -18 * sdx
        if mode == "gather":
            want, bound = _expand(want, B, H_ // 2, W_ // 2), _expand(bound.expand_as(want), B, H_ // 2, W_ // 2)
            parts = [(d0, want, bound, prior[0])]
        elif mode == "concat":
            bound = bound.expand_as(want)
            parts = [(d0, want[:, :Cin], bound[:, :Cin], prior[0]), (d1, want[:, Cin:], bound[:, Cin:], prior[1])]
        else:
            parts = [(d0, want, bound, prior[0])]
        for got, w, b, pr in parts:
            if acc:
                w, b = w + pr.double(), b + pr.double().abs() * 2.0 ** -18
            check_bf16(got, w, b, f"{mode} dx acc={acc}")
    # the two calls added dgamma / dbeta twice onto zeros (0 + S + S = 2S exactly)
    t_g, t_b = DY * xh, DY
    check_f32(dgam / 2, t_g.sum(0), t_g.abs().sum(0) * 4, rows, f"{mode} dgamma")
    check_f32(dbet / 2, t_b.sum(0), t_b.abs().sum(0), rows, f"{mode} dbeta")
    dg2, db2 = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    for _ in range(2):
        ops.layernorm_rows_bwd(code, src0, src1, dy, rows, C, gamma, mean, rstd, dg2, db2, grid=grid)
    assert torch.equal(dg2, dgam) and torch.equal(db2, dbet)


def test_layernorm_rows_refusals():
    x = bf((16, 6152), 1.0, 1)
    one = torch.ones(6152, device=dev)
    with pytest.raises(Exception, match="C=6152"):
        ops.layernorm_rows_fwd(ops.LN_SCATTER, x, None, 16, 6152, one, one, grid=(4, 4))
    x = bf((16, 64), 1.0, 1)
    one = torch.ones(256, device=dev)
    with pytest.raises(Exception, match="multiple of HPc"):
        ops.layernorm_rows_fwd(ops.LN_GATHER, x, None, 3, 256, one, one, grid=(2, 2))
