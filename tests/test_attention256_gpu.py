"""Fused attention at stored head width 256 (fdx_attn_fwd256_kernel / fdx_attn_bwd256_kernel) against float64,
element by element.  Cases: the UNet's 8², 16² and 32² self-attention levels (64, 256, 1024 queries and keys) with
1, 2 and 4 heads and B = 1 .. 3; cross-attention to 77 text keys; ragged query and key counts on both sides of
the 64-key block and 128-query tile edges and of the single-stage / ring switch at 128 keys; true head widths 160
and 192 zero-padded to 256.

The width-256 kernels walk the keys (and, in the dK / dV kernel, the queries) in 64-row blocks, not the 128-row
blocks that tests/elementwise_ref.py's attention bound counts.  `attention_ref_blocks` below is that bound with
the block size as a parameter: the number of blocks enters the online-softmax rescaling chain (one ex2 and one
f32 multiply-add per block) and the zero-filled padding sets the depth of every sum over keys or queries."""
import math

import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops
from flaxdiff_b200._lib import FdxError

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
BLK = 64


def _attn_rows_blocks(q, k, v, dO, sc, blk):
    """elementwise_ref._attn_rows with key blocks of `blk` rows (the derivation is written out there)."""
    R_, dh = q.shape
    Lk = k.shape[0]
    nblk = math.ceil(Lk / blk)
    Lkp = blk * nblk
    ka, va = k.abs(), v.abs()
    S = q @ k.T
    t = sc * S
    tmax = t.amax(1, keepdim=True)
    e = torch.exp(t - tmax)
    lsum = e.sum(1, keepdim=True)
    lse = tmax + torch.log(lsum)
    P = e / lsum
    O = P @ v
    es = sc * dh * R.TC_ADD * (q.abs() @ ka.T)
    # weight error: S, scale_log2, the fma, one ex2 per block (the rescaling factors) -- per key
    eta = es + 2 * R.U32 * t.abs() + 2 * R.U32 * (tmax - t) + nblk * R.EX2
    Pe = P * eta
    eps_l = R.gamma(Lkp + nblk + 2)
    spa = P @ va
    d_o = (Pe @ va + O.abs() * Pe.sum(1, keepdim=True)
           + (R.U_BF16 + R.TC_ADD * Lkp + R.gamma(nblk) + eps_l + 2 * R.U32) * spa + R.FTZ * Lk * va.amax(0))
    d_lse = Pe.sum(1) + eps_l + R.LOGF * torch.log(lsum).squeeze(1) + 2 * R.U32 * tmax.abs().squeeze(1)
    out = {"o": (O, d_o), "lse": (lse.squeeze(1), d_lse)}
    if dO is None:
        return out
    ob = R.bf16_bound(O, d_o)
    dOa = dO.abs()
    D = (dO * O).sum(1, keepdim=True)
    e_D = (dOa * ob).sum(1, keepdim=True) + R.gamma(dh) * (dOa * (O.abs() + ob)).sum(1, keepdim=True)
    dP = dO @ v.T
    e_dP = dh * R.TC_ADD * (dOa @ va.T)
    lse_b = R.f32_bound(lse, d_lse.unsqueeze(1))
    eps_p = es + 2 * R.U32 * t.abs() + lse_b + 2 * R.U32 * lse.abs() + R.U32 * (t - lse).abs() + R.EX2
    ep = P * eps_p + R.FTZ
    g = sc * (dP - D)
    e_g = sc * (e_dP + e_D + R.U32 * D.abs()) + R.U32 * g.abs()
    dS = P * g
    e_dS = ep * g.abs() + P * e_g + R.U32 * dS.abs()
    dSa = dS.abs() + e_dS
    e_dSb = e_dS + R.U_BF16 * dSa
    Pa = P + ep
    e_Pb = ep + R.U_BF16 * Pa
    out["dq"] = (dS @ k, e_dSb @ ka + R.TC_ADD * Lkp * (dSa @ ka))
    out["dk"] = (dS.T @ q, e_dSb.T @ q.abs(), dSa.T @ q.abs())
    out["dv"] = (P.T @ dO, e_Pb.T @ dOa, Pa.T @ dOa)
    return out


def attention_ref_blocks(q, k, v, heads, dh, scale, d_o=None, blk=BLK, max_elems=1 << 22):
    """elementwise_ref.attention_ref for kernels that walk keys and queries in `blk`-row blocks."""
    B, L, HD = q.shape
    Lk = k.shape[1]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    Lp = blk * math.ceil(L / blk)
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=q.device)  # noqa: E731
    res = {"o": (z(B, L, HD), z(B, L, HD)), "lse": (z(B, heads, L), z(B, heads, L))}
    if d_o is not None:
        res.update({n: (z(B, r, HD), z(B, r, HD)) for n, r in (("dq", L), ("dk", Lk), ("dv", Lk))})
    Rr = max(1, max_elems // Lk)
    for b in range(B):
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            kh, vh = k[b, :, cs], v[b, :, cs]
            acc = {n: [z(Lk, dh), z(Lk, dh), z(Lk, dh)] for n in ("dk", "dv")} if d_o is not None else {}
            for r0 in range(0, L, Rr):
                rs = slice(r0, min(L, r0 + Rr))
                out = _attn_rows_blocks(q[b, rs, cs], kh, vh, None if d_o is None else d_o[b, rs, cs], sc, blk)
                for n in ("o", "dq") if d_o is not None else ("o",):
                    res[n][0][b, rs, cs], res[n][1][b, rs, cs] = out[n]
                res["lse"][0][b, h, rs], res["lse"][1][b, h, rs] = out["lse"]
                for n in acc:
                    for i in range(3):
                        acc[n][i] += out[n][i]
            for n in acc:
                val, err, mag = acc[n]
                res[n][0][b, :, cs], res[n][1][b, :, cs] = val, err + R.TC_ADD * Lp * mag
    return res


def assert_attention256(q, k, v, heads, scale, got, d_o=None, what=""):
    ref = attention_ref_blocks(*(t.double() for t in (q, k, v)), heads, 256, scale,
                               None if d_o is None else d_o.double())
    for n, t in got.items():
        val, d = ref[n]
        R.assert_elementwise(t, val, R.f32_bound(val, d) if n == "lse" else R.bf16_bound(val, d), f"{what} {n}")


def test_block_bound_matches_the_shared_one_at_128():
    """With 128-row blocks the parametrised bound is elementwise_ref's own (checked on the CPU values)."""
    g = torch.Generator().manual_seed(3)
    q, k, v, d_o = (torch.randn(1, n, 64, generator=g, dtype=torch.float64) for n in (100, 200, 200, 100))
    a = attention_ref_blocks(q, k, v, 1, 64, 0.125, d_o, blk=128)
    b = R.attention_ref(q, k, v, 1, 64, 0.125, d_o)
    for n in a:
        assert torch.equal(a[n][0], b[n][0]) and torch.equal(a[n][1], b[n][1]), n


CASES = [
    # B, heads, L, Lk, d_true
    (2, 2, 64, 64, 256),            # 8x8 level of a 2-head 512-channel block
    (2, 2, 256, 256, 256),          # 16x16
    (1, 2, 1024, 1024, 256),        # 32x32
    (3, 1, 256, 256, 256),
    (2, 4, 256, 256, 256),
    (2, 2, 1024, 77, 256),          # cross-attention to the text context (single stage)
    (3, 4, 64, 77, 192),
    (1, 1, 1, 1, 256),
    (2, 2, 77, 77, 160),
    (3, 2, 200, 200, 256),
    (1, 2, 130, 129, 256),          # one key past the single-stage limit: the ring
    (1, 2, 128, 128, 192),          # the last single-stage shape
    (2, 1, 65, 63, 256),
    (1, 2, 300, 320, 160),
]


@pytest.mark.parametrize("B,heads,L,Lk,d_true", CASES)
def test_attention256_forward_backward(B, heads, L, Lk, d_true):
    torch.manual_seed(L * 7 + Lk)
    HD = heads * 256

    def mk(rows):
        t = torch.randn(B, rows, heads, 256, device=dev)
        t[..., d_true:] = 0                       # zero-padded head columns, as the UNet produces them
        return t.reshape(B, rows, HD).bfloat16()
    q, k, v = mk(L), mk(Lk), mk(Lk)
    q = q * 1.5                                    # logits with a spread the online softmax has to rescale
    scale = d_true ** -0.5
    o, lse = ops.attention_fwd(q, k, v, heads, 256, scale)
    d_o = mk(L)
    dq, dk, dv = ops.attention_bwd(q, k, v, o, lse, d_o, heads, 256, scale)
    assert_attention256(q, k, v, heads, scale, {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}, d_o)
    if d_true < 256:
        for t, rows in ((o, L), (dq, L), (dk, Lk), (dv, Lk)):
            assert t.view(B, rows, heads, 256)[..., d_true:].abs().max().item() == 0


def test_attention256_strided_views_and_determinism():
    """q / k / v as column slices of one fused projection buffer; two runs agree bit for bit."""
    torch.manual_seed(1)
    B, heads, L = 2, 2, 384
    HD = heads * 256
    qkv = torch.randn(B, L, 3 * HD, device=dev).bfloat16()
    q, k, v = qkv[..., :HD], qkv[..., HD:2 * HD], qkv[..., 2 * HD:]
    sc = 256 ** -0.5
    o1, lse1 = ops.attention_fwd(q, k, v, heads, 256, sc)
    o2, lse2 = ops.attention_fwd(q, k, v, heads, 256, sc)
    assert torch.equal(o1, o2) and torch.equal(lse1, lse2)
    d_o = torch.randn(B, L, HD, device=dev).bfloat16()
    g1 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, 256, sc)
    g2 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, 256, sc)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert_attention256(q, k, v, heads, sc, {"o": o1, "lse": lse1, "dq": g1[0], "dk": g1[1], "dv": g1[2]}, d_o)


def test_masked_attention_refuses_head_width_256():
    q = torch.zeros(1, 77, 256, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="status -2"):
        ops.attention_fwd_masked(q, q, q, 1, 256, 256 ** -0.5, True)


def test_attention_refuses_stored_head_width_512():
    q = torch.zeros(1, 8, 512, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="32 or 64, or 128 or 256"):
        ops.attention_fwd(q, q, q, 1, 512, 512 ** -0.5)
