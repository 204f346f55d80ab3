"""Fused attention at stored head width 128 (fdx_attn_fwd128_kernel / fdx_attn_bwd128_kernel) compared element by
element with the float64 reference and derived bound of tests/elementwise_ref.py, as tests/test_attention_gpu.py
does.  Cases: the 16 x 16 level of a 1024-channel UNet (256 tokens), 1024 keys (8 key blocks:
the online-softmax rescaling), 77 text keys (the single-stage arrangement), ragged query and key counts, one tiny
tile, and true widths 96 / 80 zero-padded to 128."""
import pytest
import torch

from flaxdiff_b200 import ops
from test_attention_gpu import assert_attention_elementwise

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
    dq, dk, dv = ops.attention_bwd(q, k, v, o, lse, d_o, heads, dh, scale)
    assert_attention_elementwise(q, k, v, heads, dh, scale, {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}, d_o)
    if d_true < dh:
        for t, rows in ((o, L), (dq, L), (dk, Lk), (dv, Lk)):
            assert t.view(B, rows, heads, dh)[..., d_true:].abs().max().item() == 0


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
    g1 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    g2 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert_attention_elementwise(q, k, v, heads, dh, dh ** -0.5,
                                 {"o": o1, "lse": lse1, "dq": g1[0], "dk": g1[1], "dv": g1[2]}, d_o)


def test_attention_still_rejects_other_head_widths():
    from flaxdiff_b200._lib import FdxError
    q = torch.zeros(1, 8, 2 * 96, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="32 or 64, or 128"):
        ops.attention_fwd(q, q, q, 2, 96, 0.1)
