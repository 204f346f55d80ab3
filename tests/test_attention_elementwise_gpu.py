"""Fused attention (fdx_attention_fwd / fdx_attention_bwd) compared element by element with the float64 reference
and the derived bound of tests/elementwise_ref.py (attention_ref), for all three kernel families (stored head
widths 32, 64 and 128).

Every call goes through the C ABI with buffers the test owns: o, lse, dq, dk, dv are prefilled with NaN (an
element the kernels never write fails), o / dq / dk / dv have a row stride of heads * dh + 64 and a padded batch
stride with sentinels in the gaps, lse has a sentinel tail; every sentinel must come back bit-identical.  The
backward is fed the kernel's own o and lse, as the UNet does.  Cases: L and Lk on and around every 64- and
128-row tile edge, one query / one key, 1, 3 and 6 heads, zero-padded head widths, the UNet's own attention
shapes (C3 self-attention at 32 x 32, C4 text cross-attention at 128 x 128, 64 x 64 and 32 x 32 with the doubled
CFG batch, the gallery UNet's 128-wide heads), and logit regimes that stress the online softmax.  The worst
|err| / bound per output and family is printed at the end (pytest -s)."""
import ctypes
import math

import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops
from flaxdiff_b200._lib import check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
SENTINEL = -1234.0                                   # exactly representable in bf16 and f32
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for (dh, n), w in sorted(WORST.items()):
        print(f"WORST attention dh={dh} {n} {w:.3f}")


def padded(B, rows, HD):
    """A [B][rows][HD] view with row stride HD + 64 and batch stride (rows + 1) (HD + 64) into a sentinel-filled
    buffer; the view itself is NaN."""
    buf = torch.full((B, rows + 1, HD + 64), SENTINEL, dtype=torch.bfloat16, device=dev)
    view = buf[:, :rows, :HD]
    view.fill_(math.nan)
    return buf, view


def gaps_intact(buf, rows, HD, what):
    mask = torch.ones(buf.shape, dtype=torch.bool, device=dev)
    mask[:, :rows, :HD] = False
    assert torch.equal(buf[mask].view(torch.int16), torch.full_like(buf[mask], SENTINEL).view(torch.int16)), \
        f"{what}: a kernel wrote outside its view"


def inputs(B, heads, L, Lk, dh, d_true, regime, seed):
    """bf16 q, k, v, dO on the device whose logits scale q.k follow `regime` (scale = d_true^-1/2)."""
    g = torch.Generator(device=dev).manual_seed(seed)

    def rn(rows, s=1.0):
        return torch.randn(B, rows, heads, dh, generator=g, device=dev) * s
    q, k, v, dO = rn(L), rn(Lk), rn(Lk), rn(L)
    e = torch.zeros(dh, device=dev)
    e[0] = 1.0
    root = math.sqrt(d_true)                         # scale * root = 1: one logit unit per unit along e
    kpos = torch.arange(Lk, device=dev, dtype=torch.float32).view(1, Lk, 1, 1) / 128
    if regime == "random":
        q = 1.5 * q
    elif regime == "rising":                         # each key block holds a larger maximum: every block rescales
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
        t[..., d_true:] = 0                          # zero-padded head columns, as the UNet produces them
        out.append(t.reshape(B, t.shape[1], heads * dh).bfloat16())
    return out


def run(B, heads, L, Lk, dh, d_true, regime="random", seed=0):
    q, k, v, dO = inputs(B, heads, L, Lk, dh, d_true, regime, seed)
    HD = heads * dh
    scale = d_true ** -0.5
    n_st = B * heads * L
    lse_buf = torch.full((n_st + 64,), SENTINEL, dtype=torch.float32, device=dev)
    lse = lse_buf[:n_st].view(B, heads, L)
    lse.fill_(math.nan)
    ob, o = padded(B, L, HD)
    a = ops._attn_desc(q, k, v, o, lse, heads, dh, scale)
    check(load().fdx_attention_fwd(ctypes.byref(a), stream_ptr()), "attention_fwd")
    (dqb, dq), (dkb, dk), (dvb, dv) = padded(B, L, HD), padded(B, Lk, HD), padded(B, Lk, HD)
    ws = torch.full((n_st,), math.nan, dtype=torch.float32, device=dev)
    a.d_o, a.do_ld, a.do_bs = ptr(dO), dO.stride(1), dO.stride(0)
    a.dvec_ws = ptr(ws)
    a.dq, a.dq_ld, a.dq_bs = ptr(dq), dq.stride(1), dq.stride(0)
    a.dk, a.dk_ld, a.dk_bs = ptr(dk), dk.stride(1), dk.stride(0)
    a.dv, a.dv_ld, a.dv_bs = ptr(dv), dv.stride(1), dv.stride(0)
    check(load().fdx_attention_bwd(ctypes.byref(a), stream_ptr()), "attention_bwd")
    torch.cuda.synchronize()
    for buf, rows, what in ((ob, L, "o"), (dqb, L, "dq"), (dkb, Lk, "dk"), (dvb, Lk, "dv")):
        gaps_intact(buf, rows, HD, what)
    assert torch.equal(lse_buf[n_st:].view(torch.int32), torch.full_like(lse_buf[n_st:], SENTINEL).view(torch.int32)), \
        "lse: a kernel wrote past its end"
    ref = R.attention_ref(*(t.to(F64) for t in (q, k, v)), heads, dh, scale, dO.to(F64))
    tag = f"dh={dh} B={B} heads={heads} L={L} Lk={Lk} d={d_true} {regime}"
    got = {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}
    for n, t in got.items():
        val, d = ref[n]
        bound = R.f32_bound(val, d) if n == "lse" else R.bf16_bound(val, d)
        w = R.assert_elementwise(t, val, bound, f"{tag}: {n}")
        WORST[(dh, n)] = max(WORST.get((dh, n), 0.0), w)
    if d_true < dh:                                  # padded head columns come out exactly zero
        for n, rows in (("o", L), ("dq", L), ("dk", Lk), ("dv", Lk)):
            assert (got[n].reshape(B, rows, heads, dh)[..., d_true:] == 0).all(), f"{tag}: padded {n}"


EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257]
# every edge value once as L and once as Lk (Lk rotated by three places), plus 1024 / 1025 keys
EDGE_PAIRS = list(zip(EDGES, EDGES[3:] + EDGES[:3])) + [(257, 1024), (129, 1025)]
# (stored width, true width, head counts that are legal for it: heads * dh % 64 == 0)
FAMILIES = [(32, 16, (2, 6)), (32, 8, (6,)), (64, 64, (1, 3)), (64, 48, (6,)), (128, 128, (1, 3)), (128, 80, (6,)),
            (128, 96, (1,))]


def edge_cases():
    out = []
    for i, (L, Lk) in enumerate(EDGE_PAIRS):
        dh, d_true, hs = FAMILIES[i % len(FAMILIES)]
        for dh_, dt_ in ((dh, d_true), (32, 32), (64, 64), (128, 128)) if i % 3 == 0 else ((dh, d_true),):
            hs_ = hs if dh_ == dh else ((2,) if dh_ == 32 else (1,))
            out.append((1 + i % 2, hs_[i % len(hs_)], L, Lk, dh_, dt_))
    return sorted(set(out))


@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", edge_cases())
def test_attention_tile_edges_elementwise(B, heads, L, Lk, dh, d_true):
    run(B, heads, L, Lk, dh, d_true, seed=L * 7 + Lk)


@pytest.mark.parametrize("B,heads,L,Lk,dh,d_true", [
    (2, 8, 1024, 1024, 64, 64),        # C3 self-attention at the 32 x 32 level
    (1, 8, 16384, 77, 32, 16),         # C4 text cross-attention at 128 x 128 (d = 16 stored as 32)
    (1, 8, 4096, 77, 32, 32),          # C4 at 64 x 64
    (64, 8, 1024, 77, 64, 64),         # C4 at 32 x 32 with the doubled CFG batch (grid z = 64)
    (2, 8, 256, 256, 128, 128),        # the gallery UNet's 128-wide heads at 16 x 16: self-attention
    (2, 8, 256, 77, 128, 128),         # ... and its text cross-attention
])
def test_attention_unet_shapes_elementwise(B, heads, L, Lk, dh, d_true):
    run(B, heads, L, Lk, dh, d_true, seed=B + L + Lk)


@pytest.mark.parametrize("regime", ["rising", "first_max", "one_hot", "negative", "constant"])
@pytest.mark.parametrize("dh", [32, 64, 128])
def test_attention_logit_regimes_elementwise(dh, regime):
    heads = 2 if dh == 32 else 1
    run(1, heads, 257, 1024, dh, dh, regime, seed=dh)            # eight key blocks: the online softmax
    run(1, heads, 200, 77, dh, dh, regime, seed=dh + 1)          # 51 zero-filled tail keys in the one block
