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


# ----------------------------------------------------------------------------------------------- attention
LOG2E32 = float(torch.tensor(math.log2(math.e), dtype=torch.float32))
LN2_32 = float(torch.tensor(math.log(2), dtype=torch.float32))


def _f32(t):
    return t.to(torch.float64).float()


def _ex2(x):
    """ex2.ftz in f32: subnormal results flush to 0."""
    y = torch.exp2(x)
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def _attn_inputs(B, heads, L, Lk, dh, d_true, regime, seed=0):
    """bf16 q, k, v, dO (as float64) whose logits sc q.k follow `regime`."""
    g = torch.Generator().manual_seed(seed)

    def rn(rows, s=1.0):
        return torch.randn(B, rows, heads, dh, generator=g, dtype=torch.float64) * s
    q, k, v, dO = rn(L), rn(Lk), rn(Lk), rn(L)
    e = torch.zeros(dh, dtype=torch.float64)
    e[0] = 1.0
    root = math.sqrt(d_true)                         # sc * root = 1: a logit unit per unit along e
    kpos = torch.arange(Lk, dtype=torch.float64).view(1, Lk, 1, 1) / 128
    if regime == "random":
        q = q * 1.5
    elif regime == "rising":                         # every key block holds a larger maximum: each one rescales
        q, k = 0.5 * q + root * e, 0.5 * k + 3 * kpos * e
    elif regime == "first_max":                      # the first key block holds the maximum
        q, k = 0.5 * q + root * e, 0.5 * k + 3 * (Lk / 128 - kpos) * e
    elif regime == "one_hot":                        # logit spread ~40: most exponentials flush to 0
        q = 40 * q
    elif regime == "negative":                       # every valid logit about -30: a leaked logit 0 would dominate
        q, k = 0.1 * q - 6 * root * e, 0.1 * k + 5 * e
    elif regime == "constant":
        q = torch.zeros_like(q)
    else:
        raise ValueError(regime)
    out = []
    for t in (q, k, v, dO):
        t = t.clone()
        t[..., d_true:] = 0
        out.append(_bf(t.reshape(t.shape[0], t.shape[1], heads * dh)))
    return out


def _attn_emulate(q, k, v, dO, heads, dh, scale, leak=False, drop_tile=None, lse_off=None):
    """f32 emulation of fdx_attn.cu's arithmetic per (image, head): 128-key blocks with zero-filled, masked tail
    keys, the online maximum and corr, P rounded to bf16 for PV with l from the unrounded p, D from the bf16 O,
    and in the backward P recomputed from the emulated lse, bf16 P and dS.  Planted defects: `leak` counts one
    zero-filled tail key in l; `drop_tile` = t drops query tile t's contribution to dK / dV of the last key in
    head 0;
    `lse_off` = (row, offset) recomputes that row's P from lse + offset."""
    B, L, HD = q.shape
    Lk = k.shape[1]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    sl2 = float(torch.tensor(sc * LOG2E32, dtype=torch.float32))
    nblk = math.ceil(Lk / 128)
    o, lse = torch.zeros(B, L, HD), torch.zeros(B, heads, L)
    dq, dk, dv = torch.zeros(B, L, HD), torch.zeros(B, Lk, HD), torch.zeros(B, Lk, HD)
    for b in range(B):
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            qh, kh, vh, dOh = (t[b, :, cs].float() for t in (q, k, v, dO))
            kp = torch.zeros(128 * nblk, dh)
            vp = torch.zeros(128 * nblk, dh)
            kp[:Lk], vp[:Lk] = kh, vh
            m = torch.full((L, 1), -math.inf)
            l, acc = torch.zeros(L, 1), torch.zeros(L, dh)
            for j in range(nblk):
                kb, vb = kp[128 * j:128 * j + 128], vp[128 * j:128 * j + 128]
                S = qh @ kb.T
                valid = torch.arange(128) < Lk - 128 * j
                mx = torch.where(valid, S, torch.full_like(S, -math.inf)).amax(1, keepdim=True)
                m_new = torch.maximum(m, _f32(mx.double() * sl2))
                corr = _ex2(_f32(m.double() - m_new.double()))
                pe = _ex2(_f32(S.double() * sl2 - m_new.double()))
                pe = torch.where(valid, pe, torch.zeros_like(pe))
                rs = pe.sum(1, keepdim=True)
                if leak and j == nblk - 1 and not valid.all():
                    rs = rs + _ex2(-m_new)                       # a zero-filled key: logit 0 counted in l
                Oj = pe.bfloat16().float() @ vb
                l = _f32(l.double() * corr.double() + rs.double())
                acc = _f32(acc.double() * corr.double() + Oj.double())
                m = m_new
            ob = (acc * (1 / l)).bfloat16().float()
            o[b, :, cs] = ob
            lse_h = _f32(_f32(m.double() * LN2_32).double() + torch.log(l.double()))
            lse[b, h] = lse_h.squeeze(1)
            # backward, fed the emulated o and lse
            D = (dOh * ob).sum(1, keepdim=True)
            lse_used = lse_h.clone()
            if lse_off is not None:
                lse_used[lse_off[0]] += lse_off[1]
            lse_r = _f32(lse_used.double() * LOG2E32)
            d_r = _f32(D.double() * sc)
            S = qh @ kh.T
            dP = dOh @ vh.T
            p = _ex2(_f32(S.double() * sl2 - lse_r.double()))
            ds = _f32(p.double() * _f32(dP.double() * sc - d_r.double()).double())
            pb, dsb = p.bfloat16().float(), ds.bfloat16().float()
            dq[b, :, cs] = dsb @ kh
            if drop_tile is not None and h == 0:
                keep = torch.ones(L, 1)
                keep[128 * drop_tile:128 * drop_tile + 128] = 0
                pk, dk_last = pb[:, -1:] * keep, dsb[:, -1:] * keep
                pb, dsb = torch.cat([pb[:, :-1], pk], 1), torch.cat([dsb[:, :-1], dk_last], 1)
            dk[b, :, cs] = dsb.T @ qh
            dv[b, :, cs] = pb.T @ dOh
    bf = lambda t: t.bfloat16().double()  # noqa: E731
    return {"o": bf(o), "lse": lse.double(), "dq": bf(dq), "dk": bf(dk), "dv": bf(dv)}


def _attn_autograd(q, k, v, dO, heads, dh, scale):
    B, L, HD = q.shape
    Lk = k.shape[1]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    qr, kr, vr = (t.view(t.shape[0], t.shape[1], heads, dh).clone().requires_grad_(True) for t in (q, k, v))
    logits = torch.einsum("blhd,bkhd->bhlk", qr, kr) * sc
    o = torch.einsum("bhlk,bkhd->blhd", torch.softmax(logits, -1), vr).reshape(B, L, HD)
    o.backward(dO)
    return (o.detach(), torch.logsumexp(logits, -1).detach(), qr.grad.reshape(B, L, HD),
            kr.grad.reshape(B, Lk, HD), vr.grad.reshape(B, Lk, HD))


def _attn_check(got, ref, names=("o", "lse", "dq", "dk", "dv")):
    worst = {}
    for n in names:
        val, d = ref[n]
        bound = R.f32_bound(val, d) if n == "lse" else R.bf16_bound(val, d)
        worst[n] = R.assert_elementwise(got[n], val, bound, n)
    return worst


@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", [(2, 2, 70, 77, 32, 16), (1, 3, 130, 129, 64, 48),
                                                     (1, 2, 65, 300, 128, 80), (2, 1, 1, 1, 64, 64)])
def test_attention_reference_matches_autograd(B, heads, L, Lk, dh, d_true):
    q, k, v, dO = _attn_inputs(B, heads, L, Lk, dh, d_true, "random")
    ref = R.attention_ref(q, k, v, heads, dh, d_true ** -0.5, dO, max_elems=4096)   # several row chunks
    o, lse, gq, gk, gv = _attn_autograd(q, k, v, dO, heads, dh, d_true ** -0.5)
    for n, want in (("o", o), ("lse", lse), ("dq", gq), ("dk", gk), ("dv", gv)):
        _close(ref[n][0], want)
        assert (ref[n][1] >= 0).all() and torch.isfinite(ref[n][1]).all(), n
    for n, rows in (("o", L), ("dq", L), ("dk", Lk), ("dv", Lk)):
        assert (ref[n][0].view(B, rows, heads, dh)[..., d_true:] == 0).all(), n


_EMU_WORST = {}


@pytest.mark.parametrize("regime", ["random", "rising", "first_max", "one_hot", "negative", "constant"])
@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", [(1, 2, 200, 300, 32, 32), (1, 1, 130, 520, 64, 64),
                                                     (1, 1, 70, 77, 64, 48), (1, 1, 129, 257, 128, 128)])
def test_attention_emulation_within_bound(B, heads, L, Lk, dh, d_true, regime):
    """An f32 emulation of the kernels' arithmetic lies inside the float64 bound at every element, across the
    logit regimes the GPU tests use.  The worst |err| / bound per output is printed (pytest -s)."""
    q, k, v, dO = _attn_inputs(B, heads, L, Lk, dh, d_true, regime, seed=Lk)
    scale = d_true ** -0.5
    ref = R.attention_ref(q, k, v, heads, dh, scale, dO)
    worst = _attn_check(_attn_emulate(q, k, v, dO, heads, dh, scale), ref)
    print(f"EMU dh={dh} {regime}: " + " ".join(f"{n} {w:.3f}" for n, w in worst.items()))
    for n, w in worst.items():
        _EMU_WORST[n] = max(_EMU_WORST.get(n, 0.0), w)


def _old_gates(got, ref):
    """The relative-L2 / absolute lse checks the attention GPU tests used before the element-wise comparator."""
    return (rel(got["o"], ref["o"][0]) < 1.5e-2 and (got["lse"] - ref["lse"][0]).abs().max().item() < 2e-2
            and all(rel(got[n], ref[n][0]) < 2e-2 for n in ("dq", "dk", "dv")))


@pytest.mark.parametrize("defect", ["leak", "drop_tile", "lse_off"])
def test_attention_comparator_rejects_what_relative_l2_accepts(defect):
    """Three confined attention defects, each accepted by the old gates and rejected element by element:
    (a) a zero-filled tail key counted in l at Lk = 77 (seen through lse, and through O in the negative-logit
    regime), (b) one CTA's query tile missing from dK and dV of the last key of a ragged key block (one head),
    (c) the last row of a ragged query tile recomputing P from an lse that is off by 2^-3.  An offset of 2^-7
    scales that row's P by 0.8 %, about two bf16 roundings of dS, which the kernels' own arithmetic may reach
    (0.2 - 0.4 of the bound); 2^-4 lands at 1.0 - 1.5 depending on the inputs, 2^-3 clears it about twofold."""
    heads, dh, L, Lk = 2, 64, 1000, 77
    q, k, v, dO = _attn_inputs(1, heads, L, Lk, dh, dh, "random", seed=7)
    scale = dh ** -0.5
    ref = R.attention_ref(q, k, v, heads, dh, scale, dO)
    _attn_check(_attn_emulate(q, k, v, dO, heads, dh, scale), ref)
    kw = {"leak": dict(leak=True), "drop_tile": dict(drop_tile=(L - 1) // 128),
          "lse_off": dict(lse_off=(L - 1, 2.0 ** -3))}
    bad = _attn_emulate(q, k, v, dO, heads, dh, scale, **kw[defect])
    assert _old_gates(bad, ref)                                  # what the relative-L2 tests accept ...
    with pytest.raises(AssertionError, match="outside the bound"):
        _attn_check(bad, ref)                                    # ... the element-wise comparator does not
    if defect == "leak":
        qn, kn, vn, dOn = _attn_inputs(1, heads, L, Lk, dh, dh, "negative", seed=7)
        refn = R.attention_ref(qn, kn, vn, heads, dh, scale)
        badn = _attn_emulate(qn, kn, vn, dOn, heads, dh, scale, leak=True)
        with pytest.raises(AssertionError, match="outside the bound"):
            _attn_check(badn, refn, ("o",))


def test_attention_emulation_bound_is_not_vacuous():
    """Runs after the emulation cases: somewhere the emulation comes within 2 % of the bound in every output
    (bounds that no f32 arithmetic approaches would let real defects through)."""
    if len(_EMU_WORST) < 5:
        pytest.skip("the emulation cases did not run in this session")
    print("EMU worst overall: " + " ".join(f"{n} {w:.3f}" for n, w in sorted(_EMU_WORST.items())))
    assert all(w >= 0.02 for w in _EMU_WORST.values()), _EMU_WORST


# ----------------------------------------------------------------------------------------------- training step
def _fl(t):
    """Round a float64 tensor to f32 and back: one f32 rounding (how an FMA's single rounding is emulated)."""
    return t.float().double()


HP = dict(lr=R.f32(2.7e-4), b1=R.f32(0.9), b2=R.f32(0.999), eps=R.f32(1e-8), wd=R.f32(1e-4))


def _opt_inputs(n=1 << 18, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda s=1.0: torch.randn(n, generator=g, dtype=torch.float64) * s  # noqa: E731
    p, gr, m = r(0.05), r(), r(0.1 / 8)
    v = r(1 / 8) ** 2 * r().abs()
    gr[100:600], m[100:600], v[100:600] = 0, 0, 0                 # unused parameters
    gr[1000:1500] *= 1e-40                                       # subnormal
    gr[2000:2500] *= 1e15                                        # large
    return [_fl(t) for t in (p, gr, m, v)]


def _adam_emulate(p, g, m, v, *, lr, b1, b2, eps, wd, bc1, bc2, mul, fused):
    """adam_kernel in f32, with every product rounded (fused=False) or with the FMA contractions nvcc may make
    (fused=True: a*b + c rounded once)."""
    c1, c2 = 1.0 - b1, 1.0 - b2
    if not fused:
        f = lambda x: torch.tensor(x, dtype=torch.float32)  # noqa: E731
        P, G, M, V = (t.float() for t in (p, g, m, v))
        gj = G * f(mul)
        M1 = f(b1) * M + f(c1) * gj
        V1 = f(b2) * V + f(c2) * gj * gj
        T = (M1 / f(bc1)) / (torch.sqrt(V1 / f(bc2)) + f(eps)) + f(wd) * P
        return (P - f(lr) * T).double(), M1.double(), V1.double(), T.double()
    gj = _fl(g * mul)
    m1 = _fl(b1 * m + _fl(c1 * gj))
    v1 = _fl(b2 * v + _fl(_fl(c2 * gj) * gj))
    q = _fl(_fl(m1 / bc1) / _fl(_fl(torch.sqrt(_fl(v1 / bc2))) + eps))
    t = _fl(wd * p + q)
    return _fl(p - lr * t), m1, v1, t


def test_optimizer_references_match_optax_restatement():
    """adam_ref / lamb_ref / ema_ref / sumsq_ref against oracle/diffusion_ref.py (optax.adamw, optax.lamb,
    clip_by_global_norm, apply_ema written out in numpy float64)."""
    from oracle import diffusion_ref as O
    p, g, m, v = _opt_inputs(4096)
    step, mul = 7, 0.125
    bc1, bc2 = 1 - HP["b1"] ** step, 1 - HP["b2"] ** step
    r = R.adam_ref(p, g, m, v, bc1=bc1, bc2=bc2, mul=mul, **HP)
    wp, wm, wv, we = O.adamw_ema(p.numpy(), mul * g.numpy(), m.numpy(), v.numpy(), p.numpy(), step, HP["lr"],
                                 HP["b1"], HP["b2"], HP["eps"], HP["wd"], decay=0.999)
    for k, w in (("p", wp), ("m", wm), ("v", wv)):
        _close(r[k][0], torch.from_numpy(w), 1e-13)
    _close(R.ema_ref(p, r["p"][0], 0.999)[0], torch.from_numpy(we), 1e-9)    # 1 - decay as the kernel's f32
    # clip_by_global_norm then adam: the clipped multiplier
    (gc,), nrm = O.clip_by_global_norm([(mul * g).numpy()], 1.0)
    assert nrm > 1
    r = R.adam_ref(p, g, m, v, bc1=bc1, bc2=bc2, mul=mul / nrm, **HP)
    wp = O.adamw_ema(p.numpy(), gc.astype("float64"), m.numpy(), v.numpy(), p.numpy(), step, HP["lr"], HP["b1"],
                     HP["b2"], HP["eps"], HP["wd"])[0]
    _close(r["p"][0], torch.from_numpy(wp), 1e-6)              # the oracle rounds the clipped gradient to f32
    val, _ = R.sumsq_ref(g, mul, 10)
    _close(val, torch.tensor(nrm ** 2), 1e-12)
    # lamb over three segments, the third with p = 0
    lens = [128, 576, 64]
    starts = torch.tensor([0, 128, 704])
    p[704:768] = 0
    r = R.lamb_ref(p[:768], g[:768], m[:768], v[:768], starts, torch.tensor(lens), bc1=bc1, bc2=bc2, mul=1.0,
                   **HP)
    sl = [slice(0, 128), slice(128, 704), slice(704, 768)]
    wp, wm, wv = O.lamb_step([p[s].numpy() for s in sl], [g[s].numpy() for s in sl], [m[s].numpy() for s in sl],
                             [v[s].numpy() for s in sl], step, HP["lr"], HP["b1"], HP["b2"], HP["eps"], HP["wd"])
    for s, a, b, c in zip(sl, wp, wm, wv):
        _close(r["p"][0][s], torch.from_numpy(a).double(), 1e-6)    # the oracle returns f32
        _close(r["m"][0][s], torch.from_numpy(b).double(), 1e-6)
        _close(r["v"][0][s], torch.from_numpy(c).double(), 1e-6)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("step", [1, 2, 1000, 10 ** 6])
def test_adam_emulation_within_bound(step, fused):
    p, g, m, v = _opt_inputs()
    bc1, bc2 = R.f32(1 - HP["b1"] ** step), R.f32(1 - HP["b2"] ** step)
    kw = dict(bc1=bc1, bc2=bc2, mul=0.125, **HP)
    r = R.adam_ref(p, g, m, v, **kw)
    ep, em, ev, et = _adam_emulate(p, g, m, v, fused=fused, **kw)
    for got, k in ((ep, "p"), (em, "m"), (ev, "v"), (et, "t")):
        R.assert_elementwise(got, r[k][0], R.f32_bound(*r[k]), k)
    e, ed = R.ema_ref(p, r["p"][0], R.f32(0.999), r["p"][1])
    d32 = torch.tensor(0.999, dtype=torch.float32)
    emu = (d32 * p.float() + (1 - d32) * ep.float()).double()
    R.assert_elementwise(emu, e, R.f32_bound(e, ed), "ema")


def test_lamb_and_sumsq_emulation_within_bound():
    p, g, m, v = _opt_inputs(64 * 300)
    lens = torch.tensor([64, 64, 128, 1024, 64] + [64 * 59] * 3 + [64 * 102])
    starts = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)[:-1]])
    kw = dict(bc1=R.f32(1 - HP["b1"] ** 5), bc2=R.f32(1 - HP["b2"] ** 5), mul=1.0, **HP)
    r = R.lamb_ref(p, g, m, v, starts, lens, **kw)
    _, _, _, u = _adam_emulate(p, g, m, v, fused=False, **kw)
    seg = torch.repeat_interleave(torch.arange(lens.numel()), lens)
    np2 = torch.zeros(lens.numel(), dtype=torch.float32).index_add_(0, seg, (p.float() ** 2))
    nu2 = torch.zeros(lens.numel(), dtype=torch.float32).index_add_(0, seg, (u.float() ** 2))
    ratio = torch.sqrt(np2) / torch.sqrt(nu2)
    a = torch.tensor(kw["lr"], dtype=torch.float32) * ratio
    pe = (p.float() - a[seg] * u.float()).double()
    R.assert_elementwise(np2.double(), r["np2"][0], R.f32_bound(*r["np2"]), "sum p^2")
    R.assert_elementwise(nu2.double(), r["nu2"][0], R.f32_bound(*r["nu2"]), "sum u^2")
    R.assert_elementwise(pe, r["p"][0], R.f32_bound(*r["p"]), "lamb p")
    # grad stats: float4 chains, per-thread running sums over the grid-stride loop, then the rest
    x = (g * 0.125).float()
    q = (x * x).view(-1, 4).sum(1)                              # 4800 float4 groups: 8 blocks x 256 threads, 3 rounds
    s = torch.cat([q, q.new_zeros(3 * 2048 - q.numel())]).view(3, 2048).sum(0).sum()
    val, d = R.sumsq_ref(g, 0.125, R.grad_stats_depth(g.numel(), 1))
    R.assert_elementwise(s.double().reshape(1), val.reshape(1), R.f32_bound(val, d).reshape(1), "sumsq")


def _gelu32(x):
    k, a = torch.tensor(R.GELU_K, dtype=torch.float32), torch.tensor(R.GELU_A, dtype=torch.float32)
    return 0.5 * x * (1 + torch.tanh(k * (x + a * x * x * x)))


def _gelu_grad32(x):
    k, a = torch.tensor(R.GELU_K, dtype=torch.float32), torch.tensor(R.GELU_A, dtype=torch.float32)
    th = torch.tanh(k * (x + a * x * x * x))
    return 0.5 * (1 + th) + 0.5 * x * (1 - th * th) * k * (1 + 3 * a * x * x)


def _temb_inputs(D, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    freqs = torch.randn(D // 2, generator=g) * 16
    t = torch.cat([torch.rand(B // 2, generator=g) * 2.65 - 1.55, torch.randint(0, 1000, (B - B // 2,),
                                                                               generator=g).float()])
    W1, W2 = (torch.randn(D, D, generator=g) / math.sqrt(D) for _ in range(2))
    b1, b2 = (torch.randn(D, generator=g) * 0.1 for _ in range(2))
    return freqs, t, W1, b1, W2, b2, torch.randn(B, D, generator=g)


def test_time_embedding_references_match_autograd():
    """time_embed_fwd_ref / _bwd_ref against float64 autograd of FourierEmbedding + TimeProjection."""
    D, B = 64, 9
    freqs, t, W1, b1, W2, b2, demb = (x.double() for x in _temb_inputs(D, B))
    ph = R.time_phase_f32(t, freqs).double()
    four = torch.cat([torch.sin(ph), torch.cos(ph)], 1)
    P = [x.clone().requires_grad_(True) for x in (W1, b1, W2, b2)]
    gelu = lambda x: 0.5 * x * (1 + torch.tanh(R.GELU_K * (x + R.GELU_A * x ** 3)))  # noqa: E731
    h1 = b1 + four @ P[0] + (P[1] - b1)
    h1.retain_grad()
    h2 = gelu(h1) @ P[2] + P[3]
    h2.retain_grad()
    emb = gelu(h2)
    (emb * demb).sum().backward()
    f = R.time_embed_fwd_ref(ph, four, h1.detach(), h2.detach(), W1, b1, W2, b2)
    _close(f["four"][0], four, 1e-15)
    _close(f["h1"][0], h1, 1e-13)
    _close(f["h2"][0], h2, 1e-13)
    _close(f["emb"][0], emb, 1e-13)
    z = [torch.zeros_like(x) for x in (W1, b1, W2, b2)]
    r = R.time_embed_bwd_ref(demb, four, h1.detach(), h2.detach(), h1.grad, h2.grad, W2, *z)
    _close(r["dh2"][0], h2.grad, 1e-12)
    _close(r["dh1"][0], h1.grad, 1e-12)
    for k, x in (("dW1", P[0]), ("db1", P[1]), ("dW2", P[2]), ("db2", P[3])):
        _close(r[k][0], x.grad, 1e-12)


@pytest.mark.parametrize("B", [1, 8, 65])
def test_time_embedding_emulation_within_bound(B):
    D = 256
    freqs, t, W1, b1, W2, b2, demb = _temb_inputs(D, B, 1)
    ph = R.time_phase_f32(t, freqs)
    four = torch.cat([torch.sin(ph), torch.cos(ph)], 1)
    h1 = b1 + four @ W1
    h2 = b2 + _gelu32(h1) @ W2
    emb = _gelu32(h2)
    d = lambda x: x.double()  # noqa: E731
    f = R.time_embed_fwd_ref(ph, d(four), d(h1), d(h2), d(W1), d(b1), d(W2), d(b2))
    R.assert_elementwise(d(four), f["four"][0], f["four"][1], "four")
    for k, x in (("h1", h1), ("h2", h2), ("emb", emb)):
        R.assert_elementwise(d(x), f[k][0], R.f32_bound(*f[k]), k)
    dh2 = demb * _gelu_grad32(h2)
    dh1 = (dh2 @ W2.T) * _gelu_grad32(h1)
    pri = [torch.randn_like(x) * 0.3 for x in (W1, b1, W2, b2)]
    got = {"dh2": dh2, "dh1": dh1, "dW1": pri[0] + four.T @ dh1, "db1": pri[1] + dh1.sum(0),
           "dW2": pri[2] + _gelu32(h1).T @ dh2, "db2": pri[3] + dh2.sum(0)}
    r = R.time_embed_bwd_ref(d(demb), d(four), d(h1), d(h2), d(dh1), d(dh2), d(W2), *[d(x) for x in pri])
    for k, x in got.items():
        R.assert_elementwise(d(x), r[k][0], R.f32_bound(*r[k]), k)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_diffuse_and_loss_references_and_emulation(kind):
    """diffuse_ref / loss_ref against a float64 restatement (autograd for dF), and an f32 emulation of the
    kernels inside their bounds."""
    g = torch.Generator().manual_seed(kind)
    B, E = 3, 4096
    x0 = torch.randint(0, 256, (B, E), generator=g).double()
    x0[:, :2] = torch.tensor([0.0, 255.0])
    eps = _fl(torch.randn(B, E, generator=g, dtype=torch.float64))
    sig = _fl(torch.rand(B, generator=g, dtype=torch.float64) * 3 + 0.01)
    al = _fl(1 / torch.sqrt(1 + sig * sig))
    r = R.diffuse_ref(x0, eps, al, sig, True, kind)
    x = (x0 - 127.5) / 127.5
    assert x[0, 0].item() == -1.0 and x[0, 1].item() == 1.0
    want = [x, eps, (al[:, None] * eps - sig[:, None] * x) / torch.sqrt(al * al + sig * sig)[:, None]][kind]
    _close(r["x_t"][0], al[:, None] * x + sig[:, None] * eps, 1e-14)
    _close(r["target"][0], want, 1e-14)
    a32, s32 = al.float()[:, None], sig.float()[:, None]
    x32 = (x0.float() - 127.5) / 127.5
    xt32 = a32 * x32 + s32 * eps.float()
    tg32 = [x32, eps.float(), (a32 * eps.float() - s32 * x32) * torch.rsqrt(a32 * a32 + s32 * s32)][kind]
    R.assert_elementwise(xt32.double(), r["x_t"][0], R.f32_bound(*r["x_t"]), "x_t")
    R.assert_elementwise(tg32.double(), r["target"][0], R.f32_bound(*r["target"]), "target")
    F = _fl(torch.randn(B, E, generator=g, dtype=torch.float64)).requires_grad_(True)
    co, cs, w = (_fl(torch.rand(B, generator=g, dtype=torch.float64) + 0.2) for _ in range(3))
    xt, tg = xt32.double(), tg32.double()
    lr_ = R.loss_ref(F.detach(), xt, tg, co, cs, w, 20)
    loss = (0.5 * w[:, None] * (co[:, None] * F + cs[:, None] * xt - tg) ** 2).mean()
    loss.backward()
    _close(lr_["loss"][0], loss.detach(), 1e-13)
    _close(lr_["dF"][0], F.grad, 1e-13)
    d32 = co.float()[:, None] * F.detach().float() + cs.float()[:, None] * xt32 - tg32
    l32 = (0.5 * w.float()[:, None] * d32 * d32).sum() * torch.tensor(1 / (B * E), dtype=torch.float32)
    g32 = w.float()[:, None] * co.float()[:, None] * torch.tensor(1 / (B * E), dtype=torch.float32)
    R.assert_elementwise(l32.double().reshape(1), lr_["loss"][0].reshape(1),
                         R.f32_bound(*lr_["loss"]).reshape(1), "loss")
    R.assert_elementwise((g32 * d32).double(), lr_["dF"][0], R.f32_bound(*lr_["dF"]), "dF")


def test_training_comparator_rejects_what_relative_l2_accepts():
    """One parameter of the optimiser's output off by 2^-12 relative, or one DDPM sample's time embedding
    computed from a phase one f32 ulp off: relative L2 (1e-6, 1e-2) lets them through, the element-wise bound
    does not."""
    p, g, m, v = _opt_inputs()
    kw = dict(bc1=R.f32(1 - HP["b1"] ** 3), bc2=R.f32(1 - HP["b2"] ** 3), mul=0.125, **HP)
    r = R.adam_ref(p, g, m, v, **kw)
    got = _adam_emulate(p, g, m, v, fused=False, **kw)[0]
    got[12345] *= 1 + 2.0 ** -12
    assert rel(got, r["p"][0]) < 1e-6
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_elementwise(got, r["p"][0], R.f32_bound(*r["p"]))
    freqs, t, *_ = _temb_inputs(256, 8, 2)
    ph = R.time_phase_f32(t, freqs)
    bad = ph.clone()
    bad[5] = torch.nextafter(bad[5], torch.tensor(math.inf))
    four = torch.cat([torch.sin(bad.double()), torch.cos(bad.double())], 1)
    ref = torch.cat([torch.sin(ph.double()), torch.cos(ph.double())], 1)
    assert rel(four, ref) < 1e-2
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_elementwise(four, ref, 2 * R.ulp_f32(ref))


# ----------------------------------------------------------------------------------------------- convolutions
def _flax_same(x, w, stride):
    """conv2d with flax SAME written from its definition: total padding max((out - 1) s + 3 - size, 0), the
    smaller half first."""
    pads = []
    for size in (x.shape[2], x.shape[1]):
        out = -(-size // stride)
        tot = max((out - 1) * stride + 3 - size, 0)
        pads += [tot // 2, tot - tot // 2]
    return Fnn.conv2d(Fnn.pad(x.permute(0, 3, 1, 2), pads), w.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def _ints(shape, g, lo=-2, hi=2):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


@pytest.mark.parametrize("stride,H,W", [(1, 5, 7), (1, 8, 8), (2, 8, 12), (2, 7, 9)])
def test_conv_references_match_autograd(stride, H, W):
    g = torch.Generator().manual_seed(7)
    x = _bf(torch.randn(2, H, W, 16, generator=g, dtype=torch.float64))
    w = _bf(torch.randn(3, 3, 16, 24, generator=g, dtype=torch.float64) / 12)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = _flax_same(xr, wr, stride)
    _close(R.conv3x3_fwd_ref(x, w, stride)[0], y)
    dy = _bf(torch.randn(tuple(y.shape), generator=g, dtype=torch.float64))
    y.backward(dy)
    _close(R.conv3x3_wgrad_ref(x, dy, 100, stride)[0], wr.grad)
    prior = torch.randn(3, 3, 16, 24, generator=g, dtype=torch.float64)
    _close(R.conv3x3_wgrad_ref(x, dy, 100, stride, prior=prior)[0], wr.grad + prior)
    if stride == 1 or (H % 2 == 0 and W % 2 == 0):       # the stride-2 data gradient needs even sizes
        _close(R.conv3x3_dgrad_ref(dy, w, stride)[0], xr.grad)
    # every delta is depth TC_ADD times the same operation on |inputs|
    _, d = R.conv3x3_fwd_ref(x, w, stride)
    _close(d, (9 * 16 + R.EPI) * R.TC_ADD * _flax_same(x.abs(), w.abs(), stride))


def test_gemm_upconv_and_3channel_references_match_autograd():
    g = torch.Generator().manual_seed(8)
    a, b = torch.randn(3, 5, 7, generator=g, dtype=torch.float64), torch.randn(3, 7, 4, generator=g, dtype=torch.float64)
    bias, res = torch.randn(4, generator=g, dtype=torch.float64), torch.randn(3, 5, 4, generator=g, dtype=torch.float64)
    v, d = R.gemm_ref(a, b, 7 + R.EPI, alpha=0.5, bias=bias, res=res)
    _close(v, 0.5 * torch.bmm(a, b) + bias + res)
    _close(d, (7 + R.EPI) * R.TC_ADD * (0.5 * torch.bmm(a.abs(), b.abs()) + bias.abs() + res.abs()))
    # nearest 2x + conv3x3 and its gradients
    x = _bf(torch.randn(2, 4, 6, 8, generator=g, dtype=torch.float64))
    w = torch.randn(3, 3, 8, 16, generator=g, dtype=torch.float64).float().double()
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    up = Fnn.interpolate(xr.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    y = _flax_same(up, wr, 1) + bias.repeat(4)
    _close(R.upconv_fwd_ref(x, w, bias.repeat(4))[0], y)
    dy = _bf(torch.randn(tuple(y.shape), generator=g, dtype=torch.float64))
    y.backward(dy)
    _close(R.upconv_dgrad_ref(dy, w)[0], xr.grad)
    _close(R.upconv_wgrad_ref(x, dy, 100)[0], wr.grad)
    # the pack: bf16 of the f32 sums, within one rounding of the exact sums; an integer kernel packs exactly
    weff = R.upconv_pack_ref(w).double()
    ex, ex_abs = torch.zeros_like(weff), torch.zeros_like(weff)
    for ph in range(4):
        for ky in range(3):
            for kx in range(3):
                ex[ph * 4 + R.up_slot(ph >> 1, ky) * 2 + R.up_slot(ph & 1, kx)] += w[ky, kx]
                ex_abs[ph * 4 + R.up_slot(ph >> 1, ky) * 2 + R.up_slot(ph & 1, kx)] += w[ky, kx].abs()
    assert ((weff - ex).abs() <= R.PACK * ex_abs).all()
    wi = _ints((3, 3, 8, 16), g)
    assert torch.equal(R.upconv_pack_ref(wi).double(), torch.stack([
        sum(wi[ky, kx] for ky in range(3) for kx in range(3)
            if R.up_slot(ph >> 1, ky) * 2 + R.up_slot(ph & 1, kx) == s) for ph in range(4) for s in range(4)]))
    # 3-channel convolutions: im2col3 / GEMM / col2im3 restate the convolution
    x3 = _bf(torch.randn(2, 5, 6, 3, generator=g, dtype=torch.float64))
    w3 = torch.randn(3, 3, 3, 8, generator=g, dtype=torch.float64)
    col = R.im2col3_ref(x3, +1, True).double()
    assert torch.equal(col[:, 27], torch.ones(60, dtype=torch.float64)) and not col[:, 28:].any()
    _close((col[:, :27] @ w3.reshape(27, 8)).reshape(2, 5, 6, 8), R.conv_in_fwd_ref(x3, w3, None)[0])
    xo = _bf(torch.randn(2, 5, 6, 8, generator=g, dtype=torch.float64))
    wo = torch.randn(3, 3, 8, 3, generator=g, dtype=torch.float64)
    bo = torch.randn(3, generator=g, dtype=torch.float64)
    colo = xo.reshape(-1, 8) @ Fnn.pad(wo.reshape(9, 8, 3).permute(1, 0, 2).reshape(8, 27), (0, 5))
    yo = R.col2im3_ref(colo.float(), bo.float(), 2, 5, 6).double()
    _close(yo, R.conv_out_fwd_ref(xo, wo, bo)[0], 1e-6)
    xor, wor, bor = (t.clone().requires_grad_(True) for t in (xo, wo, bo))
    (_flax_same(xor, wor, 1) + bor).backward(_bf(dF := torch.randn(2, 5, 6, 3, generator=g, dtype=torch.float64)))
    dFb = _bf(dF)
    _close(R.conv_out_dgrad_ref(dFb, wo)[0], xor.grad)
    (dw, _), (db, _) = R.conv_out_wgrad_ref(xo, dFb, 100)
    _close(dw, wor.grad)
    _close(db, bor.grad)
    # conv_out's data gradient is im2col3(dF, -1) times the re-arranged kernel
    colf = R.im2col3_ref(dFb, -1, False).double()[:, :27]
    _close((colf @ wo.reshape(9, 8, 3).permute(0, 2, 1).reshape(27, 8)).reshape(2, 5, 6, 8), xor.grad)


@pytest.mark.parametrize("sms", [132, 114])
def test_split_counts_follow_the_sm_count(sms):
    # C2's 64 x 64 weight gradient: one (ci, co) block, 16384 pixel blocks: one split per SM
    assert R.wgrad9_depth(256, 64, 64, 64, 64, sms) == 64 * math.ceil(16384 / sms) + sms + 1
    # 1024 channels: 256 blocks, two waves on 132 SMs at one split, so no split-K
    assert R.split_count(sms, 256, 4) == 1
    assert R.tc_bn(64) == 64 and R.tc_bn(128) == 128 and R.tc_bn(256) == 256 and R.tc_bn(320) == 128


def _trunc32(v):
    """v (float64) rounded to f32 toward zero."""
    f = v.float()
    over = f.double().abs() > v.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def test_conv_emulation_within_bound():
    """The weight gradient as wgrad9 computes it, in f32: per split a truncating chain over its 64-pixel blocks,
    then the splits added onto the prior in a random order; and a truncating 9 Cin forward chain rounded to
    bf16.  Both stay inside the bound; the exact integer case is exact."""
    g = torch.Generator().manual_seed(9)
    sms = 12
    N, H, W, Ci, Co = 3, 16, 16, 8, 8
    for kind in ("dense", "exact"):
        if kind == "dense":
            x = _bf(torch.randn(N, H, W, Ci, generator=g, dtype=torch.float64))
            dy = _bf(torch.randn(N, H, W, Co, generator=g, dtype=torch.float64))
            prior = torch.randn(3, 3, Ci, Co, generator=g, dtype=torch.float64).float().double()
        else:
            x, dy, prior = _ints((N, H, W, Ci), g), _ints((N, H, W, Co), g), _ints((3, 3, Ci, Co), g)
        depth = R.wgrad9_depth(N, H, W, Ci, Co, sms)
        val, delta = R.conv3x3_wgrad_ref(x, dy, depth, prior=prior)
        TW, TH = 16, 4
        nxb, nyb = W // TW, H // TH
        kb = nxb * nyb * N
        splits = R.split_count(sms, 1, kb)
        xp = Fnn.pad(x, (0, 0, 1, 1, 1, 1))
        parts = []
        for s in range(splits):
            acc = torch.zeros(3, 3, Ci, Co, dtype=torch.float32)
            for pb in range(kb * s // splits, kb * (s + 1) // splits):
                xb, yb, nb = pb % nxb, (pb // nxb) % nyb, pb // (nxb * nyb)
                for py in range(yb * TH, yb * TH + TH):
                    for px in range(xb * TW, xb * TW + TW):
                        t = xp[nb, py:py + 3, px:px + 3, :, None] * dy[nb, py, px]
                        acc = _trunc32(acc.double() + t)
            parts.append(acc)
        out = prior.float()
        for s in torch.randperm(splits, generator=g).tolist():
            out = out + parts[s]
        if kind == "exact":
            assert R.exact_case_ok(R.conv3x3_wgrad_ref(x.abs(), dy.abs(), depth, prior=prior.abs())[0])
            assert torch.equal(out.double(), val)
        R.assert_elementwise(out, val, R.f32_bound(val, delta), "emulated wgrad9 " + kind)
    # forward: 9 Cin terms in one truncating chain, then bf16
    w = _bf(torch.randn(3, 3, Ci, Co, generator=g, dtype=torch.float64) / 8)
    val, delta = R.conv3x3_fwd_ref(x, w)
    xp = Fnn.pad(x, (0, 0, 1, 1, 1, 1))
    acc = torch.zeros(N, H, W, Co, dtype=torch.float32)
    for ky in range(3):
        for kx in range(3):
            for ci in range(Ci):
                acc = _trunc32(acc.double() + xp[:, ky:ky + H, kx:kx + W, ci, None] * w[ky, kx, ci])
    R.assert_elementwise(acc.bfloat16(), val, R.bf16_bound(val, delta), "emulated forward")


def test_conv_comparator_rejects_what_relative_l2_accepts():
    """Four faults of the convolution engines, each inside the relative-L2 tolerances of the existing tests, each
    caught: a dropped pixel block (rel < 1e-4, the f32 tolerance) and a skipped split (rel < 5e-3, the tolerance of
    the full-size checks) by the exact integer case at C2's full weight-gradient reduction (256 images of
    64 x 64), a missing border tap by the element-wise bound, a write into the neighbouring channel slot by the
    sentinels."""
    g = torch.Generator().manual_seed(10)
    sms = 132
    N, H, W, C = 256, 64, 64, 8
    # non-negative integers: the sums grow with the pixel count, so that one block is 64 / 2^20 of them
    x, dy = _ints((N, H, W, C), g, 0, 2), _ints((N, H, W, C), g, 0, 2)
    depth = R.wgrad9_depth(N, H, W, C, C, sms)
    exact, _ = R.conv3x3_wgrad_ref(x, dy, depth, chunk=64)
    assert R.exact_case_ok(exact)
    pb = ((torch.arange(N)[:, None, None] * (H // 4) + torch.arange(H)[None, :, None] // 4) * (W // 16)
          + torch.arange(W)[None, None, :] // 16)                     # wgrad9's pixel block of every pixel
    kb = N * (H // 4) * (W // 16)
    splits = R.split_count(sms, 1, kb)

    def without(mask):
        return exact - R.conv3x3_wgrad_ref(x, dy * mask[..., None], depth, chunk=64)[0]

    dropped = without(pb == 1000)
    assert rel(dropped, exact) < 1e-4
    # a skipped split (1/132 of the pixels), in a gradient accumulated onto an earlier micro-batch's
    prior = exact.flip(2)
    s0, s1 = kb * 7 // splits, kb * 8 // splits
    skipped = without((pb >= s0) & (pb < s1)) + prior
    assert R.exact_case_ok(exact + prior) and rel(skipped, exact + prior) < 5e-3
    for got, ref in ((dropped, exact), (skipped, exact + prior)):
        assert not torch.equal(got, ref)                             # the exact integer case sees both
    # one border tap missing at one pixel of a bf16 forward
    xd = _bf(torch.randn(4, 16, 16, 64, generator=g, dtype=torch.float64))
    wd = _bf(torch.randn(3, 3, 64, 64, generator=g, dtype=torch.float64) / 24)
    val, delta = R.conv3x3_fwd_ref(xd, wd)
    bad = val.clone()
    bad[2, 15, 0, 5] -= (xd[2, 14, 0] * wd[0, 1, :, 5]).sum()        # tap (ky, kx) = (0, 1) of the bottom-left pixel
    got = _bf(bad)
    assert rel(got, val) < 5e-3
    with pytest.raises(AssertionError, match="outside the bound"):
        R.assert_elementwise(got, val, R.bf16_bound(val, delta))
    R.assert_elementwise(_bf(val), val, R.bf16_bound(val, delta))
    # a write into the neighbouring slot: the slot itself is right
    buf = torch.full((2, 4, 4, 8 + 64 + 16), -1234.0, dtype=torch.bfloat16)
    buf[..., 8:72] = _bf(val[:2, :4, :4]).bfloat16()
    R.assert_guard_intact(buf, 8, 64, -1234.0)
    buf[1, 3, 3, 72] = buf[1, 3, 3, 71]
    assert rel(buf[..., 8:72], val[:2, :4, :4]) < 5e-3
    with pytest.raises(AssertionError, match="outside its channel slot"):
        R.assert_guard_intact(buf, 8, 64, -1234.0)


def test_gemm_comparator_rejects_what_relative_l2_accepts():
    """Five faults of the dense GEMM engine at shapes the models issue, each inside 5e-3 relative L2 (the tolerance
    of test_tc_epilogue_gpu.py) and each caught by the exact integer case of test_gemm_layers_elementwise_gpu.py:
    one 64-deep k-chunk dropped in one output tile of a K = 4F = 3072 projection, one split of the wave-aware
    split-K weight gradient dropped or added twice (UNet c4's 128 x 128 attention projections, 32768 rows, 132
    splits) in a gradient accumulated onto a prior, the ragged last 64-column tile of N = 576 = 2 x 256 + 64 left
    holding a previous step's output, the bias added by every split of a split-K launch (the GPU file's fixed
    split-K bias cases, since no model passes a bias to a split-K reduction), and a residual read at the wrong row
    stride."""
    g = torch.Generator().manual_seed(11)
    sms = 132

    def caught(got, exact):
        assert rel(got, exact) < 5e-3
        assert not torch.equal(got, exact)

    # KMN, K = 3072 (48 k-chunks): chunk 17 missing from the tile of rows 256..383 and columns 256..511
    M, N, K = 1024, 768, 3072
    a, b = _ints((M, K), g, 0, 2), _ints((K, N), g, 0, 2)
    exact = a @ b
    assert R.exact_case_ok(exact) and R.tc_bn(N) == 256
    got = exact.clone()
    got[256:384, 256:512] -= a[256:384, 17 * 64:18 * 64] @ b[17 * 64:18 * 64, 256:512]
    caught(got, exact)
    # MNMN weight gradient dW = x^T dy over 32768 rows, split-K onto a prior
    rows, F = 32768, 128
    x, dy = _ints((rows, F), g, 0, 2), _ints((rows, F), g, 0, 2)
    splits, kblocks = R.mnmn_splits(rows, 1, 1, F, F, 1, sms, gemm=True)
    assert splits == 132 and kblocks == rows // 64
    prior = (x.T @ dy).flip(1)
    exact = x.T @ dy + prior
    assert R.exact_case_ok(exact)
    r0, r1 = 64 * (kblocks * 7 // splits), 64 * (kblocks * 8 // splits)
    part = x[r0:r1].T @ dy[r0:r1]
    caught(exact - part, exact)
    caught(exact + part, exact)
    # the bias of a split-K launch added by every split
    bias = _ints((F,), g)
    caught(exact + splits * bias, exact + bias)
    # N = 576: the last column tile [512, 576) of one row tile keeps the output of a step earlier (weights 1e-3 off)
    M, N, K = 512, 576, 768
    a, b = _ints((M, K), g, 0, 2), _ints((K, N), g, 0, 2)
    exact = a @ b
    assert R.tc_bn(N) == 256 and N % 256 == 64
    got = exact.clone()
    got[128:256, 512:] = a[128:256] @ (b[:, 512:] * (1 - 1e-3))
    caught(got, exact)
    # KK data gradient with a residual [M][r_ld = N + 64] read at row stride N
    M, N, K = 512, 768, 3072
    a, w = _ints((M, K), g, 0, 2), _ints((N, K), g, 0, 2)
    resbuf = _ints((M, N + 64), g)
    exact = a @ w.T + resbuf[:, :N]
    got = a @ w.T + resbuf.reshape(-1)[:M * N].reshape(M, N)
    caught(got, exact)
