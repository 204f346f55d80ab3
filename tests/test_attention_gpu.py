"""Fused attention (fdx_attention_fwd / fdx_attention_bwd) against a float64 reference of
nn.dot_product_attention (models/attention.py:170-174): softmax(q k^T / sqrt(d)) v and its gradients.
Cases: stored head widths 32 and 64 (true widths 8 / 16 zero-padded to 32), 77 text keys (masked tail of a
128-key block), 1024 keys (8 blocks: the online-softmax rescaling), query counts that are not multiples of
128, a single tiny tile.  Every output is compared element by element with the float64 reference and the bound
derived in tests/elementwise_ref.py (attention_ref)."""
import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def assert_attention_elementwise(q, k, v, heads, dh, scale, got, d_o=None, what=""):
    """got: dict of kernel outputs among o, lse, dq, dk, dv -> each within its float64 bound."""
    ref = R.attention_ref(*(t.double() for t in (q, k, v)), heads, dh, scale, None if d_o is None else d_o.double())
    for n, t in got.items():
        val, d = ref[n]
        R.assert_elementwise(t, val, R.f32_bound(val, d) if n == "lse" else R.bf16_bound(val, d), f"{what} {n}")


CASES = [
    # B, heads, L, Lk, dh(stored), d_true
    (2, 8, 1024, 1024, 64, 64),
    (2, 8, 1024, 1024, 32, 32),
    (2, 8, 256, 77, 64, 64),
    (2, 8, 1024, 77, 32, 16),
    (1, 8, 4096, 77, 32, 8),
    (3, 8, 200, 200, 32, 32),
    (2, 8, 4, 4, 64, 64),
    (1, 4, 64, 300, 64, 64),
    (1, 2, 130, 129, 32, 32),
]


@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", CASES)
def test_attention_forward_backward(B, heads, L, Lk, dh, d_true):
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
    # padded head columns must come out exactly zero (their weights are zero rows / columns in the UNet)
    if d_true < dh:
        for t, rows in ((o, L), (dq, L), (dk, Lk), (dv, Lk)):
            assert t.view(B, rows, heads, dh)[..., d_true:].abs().max().item() == 0


def test_attention_strided_views_and_determinism():
    """q / k / v as column slices of one fused projection buffer (row stride > heads*dh); two runs agree bit
    for bit (no atomics anywhere in the fused path)."""
    torch.manual_seed(1)
    B, heads, L, dh = 2, 8, 384, 64
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


def test_attention_rejects_unsupported_head_width():
    from flaxdiff_b200._lib import FdxError
    q = torch.zeros(1, 8, 8 * 16, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="32 or 64"):
        ops.attention_fwd(q, q, q, 8, 16, 0.25)
