"""Fused attention (fdx_attention_fwd / fdx_attention_bwd) against a plain fp32 torch reference of
nn.dot_product_attention (models/attention.py:170-174): softmax(q k^T / sqrt(d)) v and its gradients.
Cases: stored head widths 32 and 64 (true widths 8 / 16 zero-padded to 32), 77 text keys (masked tail of a
128-key block), 1024 keys (8 blocks: the online-softmax rescaling), query counts that are not multiples of
128, a single tiny tile.  Tolerances: bf16 operands / bf16 P, f32 accumulation: <= 1.5e-2 relative L2."""
import pytest
import torch

from flaxdiff_b200 import ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def reference(q, k, v, heads, dh, d_true, scale, d_o=None):
    B, L, HD = q.shape
    Lk = k.shape[1]
    qf, kf, vf = (t.float().view(t.shape[0], t.shape[1], heads, dh).requires_grad_(True) for t in (q, k, v))
    logits = torch.einsum("blhd,bkhd->bhlk", qf, kf) * scale
    w = torch.softmax(logits, dim=-1)
    o = torch.einsum("bhlk,bkhd->blhd", w, vf).reshape(B, L, HD)
    lse = torch.logsumexp(logits, dim=-1)
    if d_o is None:
        return o, lse
    gq, gk, gv = torch.autograd.grad(o, (qf, kf, vf), d_o.float())
    return o, lse, gq.reshape(B, L, HD), gk.reshape(B, Lk, HD), gv.reshape(B, Lk, HD)


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
    orf, lser, gq, gk, gv = reference(q, k, v, heads, dh, d_true, scale, d_o)
    assert rel(o, orf) < 1.5e-2, rel(o, orf)
    assert (lse - lser).abs().max().item() < 2e-2
    dq, dk, dv = ops.attention_bwd(q, k, v, o, lse, d_o, heads, dh, scale)
    assert rel(dq, gq) < 2e-2, ("dq", rel(dq, gq))
    assert rel(dk, gk) < 2e-2, ("dk", rel(dk, gk))
    assert rel(dv, gv) < 2e-2, ("dv", rel(dv, gv))
    # padded head columns must come out exactly zero (their weights are zero rows / columns in the UNet)
    if d_true < dh:
        assert o.view(B, L, heads, dh)[..., d_true:].abs().max().item() == 0
        assert dv.view(B, Lk, heads, dh)[..., d_true:].abs().max().item() == 0


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
    orf, _ = reference(q, k, v, heads, dh, dh, dh ** -0.5)
    assert rel(o1, orf) < 1.5e-2
    d_o = torch.randn(B, L, HD, device=dev).bfloat16()
    g1 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    g2 = ops.attention_bwd(q, k, v, o1, lse1, d_o, heads, dh, dh ** -0.5)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))


@pytest.mark.parametrize("B,heads,L,Lk,dh", [(2, 8, 1024, 1024, 64), (1, 4, 200, 300, 32), (2, 8, 384, 77, 64)])
def test_attention_kernel_arrangements_agree(B, heads, L, Lk, dh, monkeypatch):
    """The forward's single-stage arrangement for key sequences that fit one 128-key block against the K/V ring
    (FDX_ATTN_NO_SHORT, read per launch).  Same arithmetic in the same order per element, so the results are
    bit-identical."""
    torch.manual_seed(2)
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


def test_attention_rejects_unsupported_head_width():
    from flaxdiff_b200._lib import FdxError
    q = torch.zeros(1, 8, 8 * 16, device=dev, dtype=torch.bfloat16)
    with pytest.raises(FdxError, match="32 or 64"):
        ops.attention_fwd(q, q, q, 8, 16, 0.25)
