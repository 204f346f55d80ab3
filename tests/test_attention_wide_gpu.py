"""Fused attention at stored head width 128 (fdx_attn_fwd128_kernel / fdx_attn_bwd128_kernel) against the fp32 torch
reference of tests/test_attention_gpu.py, with its tolerances: forward <= 1.5e-2 relative L2, lse within 2e-2,
dQ / dK / dV <= 2e-2.  Cases: the 16 x 16 level of a 1024-channel UNet (256 tokens), 1024 keys (8 key blocks:
the online-softmax rescaling), 77 text keys (the single-stage arrangement), ragged query and key counts, one tiny
tile, and true widths 96 / 80 zero-padded to 128."""
import pytest
import torch

from flaxdiff_b200 import ops
from test_attention_gpu import reference, rel

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

CASES = [
    # B, heads, L, Lk, dh(stored), d_true
    (2, 8, 256, 256, 128, 128),
    (2, 8, 1024, 1024, 128, 128),
    (2, 8, 256, 77, 128, 128),
    (1, 8, 1024, 77, 128, 96),
    (3, 4, 200, 300, 128, 128),
    (1, 2, 130, 129, 128, 80),
    (2, 8, 4, 4, 128, 128),
]


@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", CASES)
def test_wide_attention_forward_backward(B, heads, L, Lk, dh, d_true):
    torch.manual_seed(0)
    HD = heads * dh

    def mk(rows):
        t = torch.randn(B, rows, heads, dh, device=dev)
        t[..., d_true:] = 0                       # zero-padded head columns, as the UNet produces them
        return t.reshape(B, rows, HD).bfloat16()
    q, k, v = mk(L), mk(Lk), mk(Lk)
    q = q * 1.5                                    # logits with a spread the online softmax has to rescale
    scale = d_true ** -0.5
    o, lse = ops.attention_fwd(q, k, v, heads, dh, scale)
    d_o = mk(L)
    orf, lser, gq, gk, gv = reference(q, k, v, heads, dh, d_true, scale, d_o)
    assert rel(o, orf) < 1.5e-2, rel(o, orf)
    assert (lse - lser).abs().max().item() < 2e-2
    dq, dk, dv = ops.attention_bwd(q, k, v, o, lse, d_o, heads, dh, scale)
    assert rel(dq, gq) < 2e-2, ("dq", rel(dq, gq))
    assert rel(dk, gk) < 2e-2, ("dk", rel(dk, gk))
    assert rel(dv, gv) < 2e-2, ("dv", rel(dv, gv))
    if d_true < dh:
        assert o.view(B, L, heads, dh)[..., d_true:].abs().max().item() == 0
        assert dv.view(B, Lk, heads, dh)[..., d_true:].abs().max().item() == 0


def test_wide_attention_strided_views_and_determinism():
    """q / k / v as column slices of one fused projection buffer (row stride 3 * heads * 128); two runs agree
    bit for bit."""
    torch.manual_seed(1)
    B, heads, L, dh = 2, 8, 384, 128
    HD = heads * dh
    qkv = torch.randn(B, L, 3 * HD, device=dev).bfloat16()
    q, k, v = qkv[..., :HD], qkv[..., HD:2 * HD], qkv[..., 2 * HD:]
    o1, lse1 = ops.attention_fwd(q, k, v, heads, dh, dh ** -0.5)
    o2, lse2 = ops.attention_fwd(q, k, v, heads, dh, dh ** -0.5)
    assert torch.equal(o1, o2) and torch.equal(lse1, lse2)
    d_o = torch.randn(B, L, HD, device=dev).bfloat16()
    orf, lser, gq, gk, gv = reference(q, k, v, heads, dh, dh, dh ** -0.5, d_o)
    assert rel(o1, orf) < 1.5e-2
    g1 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    g2 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    for g, r in zip(g1, (gq, gk, gv)):
        assert rel(g, r) < 2e-2


@pytest.mark.parametrize("B,heads,L,Lk", [(2, 8, 256, 77), (1, 4, 200, 128), (2, 2, 1024, 5)])
def test_wide_attention_kernel_arrangements_agree(B, heads, L, Lk, monkeypatch):
    """At <= 128 keys the single-stage forward equals the K/V ring (FDX_ATTN_NO_SHORT) bit for bit."""
    torch.manual_seed(2)
    dh = 128
    HD = heads * dh
    q, k, v, d_o = (torch.randn(B, n, HD, device=dev).bfloat16() for n in (L, Lk, Lk, L))
    o, lse = ops.attention_fwd(q, k, v, heads, dh, dh ** -0.5)
    g = ops.attention_bwd(q, k, v, o, lse, d_o, heads, dh, dh ** -0.5)
    monkeypatch.setenv("FDX_ATTN_NO_SHORT", "1")
    o1, lse1 = ops.attention_fwd(q, k, v, heads, dh, dh ** -0.5)
    g1 = ops.attention_bwd(q, k, v, o, lse, d_o, heads, dh, dh ** -0.5)
    torch.cuda.synchronize()
    assert torch.equal(o, o1) and torch.equal(lse, lse1)
    assert all(torch.equal(a, b) for a, b in zip(g, g1))


def test_attention_still_rejects_other_head_widths():
    from flaxdiff_b200._lib import FdxError
    q = torch.zeros(1, 8, 2 * 96, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="32 or 64, or 128"):
        ops.attention_fwd(q, q, q, 2, 96, 0.1)
