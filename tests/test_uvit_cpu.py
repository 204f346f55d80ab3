"""UViT host logic (no GPU): parameter names and shapes, the constructor's and the call's refusals, the config round
trip, the Hilbert orders against the reference's own indices, the oracle against a closed form and gradcheck, and a
ptxas guard for fdx_uvit.cu.

Parameter names: UViT.setup (simple_vit.py:42-170) names patch_embed, hilbert_projection (only under use_hilbert),
pos_encoding, time_embed, text_proj, down_block_{i}, mid_block, up_dense_{i}, up_block_{i}, final_norm, final_proj and,
with add_residualblock_output, final_conv1, final_norm_conv and final_conv2.  Modules built in setup() get parameters
only when called: patch_embed has none under use_hilbert, text_proj none without a text context and final_conv_direct
none at all.  Inside a block, TransformerBlock's compact names apply (RMSNorm_0, project_in / project_out, Attention
with Attention1 / Attention2, ff, norm1-3).  No UViT checkpoint exists in the reference tree, so the names are derived
from flax's naming rules, not pinned against a file flax wrote."""
import json
import os

import numpy as np
import pytest
import torch

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.uvit import UViT
from oracle import uvit_ref
from oracle.dit_ref import layernorm
from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scan_orders.json")


def _names(F, h, p, layers, ctx, proj=False, both=False, norm_in=False, hilbert=False, head=False, out=3):
    d = F // h
    want = {"pos_encoding": (1, (512 // p) ** 2, F),
            "time_embed/layers_1/DenseGeneral_0/kernel": (F, F), "time_embed/layers_1/DenseGeneral_0/bias": (F,),
            "time_embed/layers_1/DenseGeneral_1/kernel": (F, F), "time_embed/layers_1/DenseGeneral_1/bias": (F,),
            "final_norm/scale": (F,), "final_norm/bias": (F,), "final_proj/kernel": (F, p * p * out),
            "final_proj/bias": (p * p * out,)}
    if ctx:
        want.update({"text_proj/kernel": (ctx, F), "text_proj/bias": (F,)})
    if hilbert:
        want.update({"hilbert_projection/kernel": (p * p * 3, F), "hilbert_projection/bias": (F,)})
    else:
        want.update({"patch_embed/Conv_0/kernel": (p, p, 3, F), "patch_embed/Conv_0/bias": (F,)})
    if head:
        want.update({"final_conv1/conv/kernel": (3, 3, 3 + out, 64), "final_conv1/conv/bias": (64,),
                     "final_norm_conv/scale": (64,), "final_norm_conv/bias": (64,),
                     "final_conv2/conv/kernel": (3, 3, 64, out), "final_conv2/conv/bias": (out,)})
    half = layers // 2
    for b in [f"down_block_{i}" for i in range(half)] + ["mid_block"] + [f"up_block_{i}" for i in range(half)]:
        a = f"{b}/Attention"
        if norm_in:
            want[f"{b}/RMSNorm_0/scale"] = (F,)
        if proj:
            want[f"{b}/project_in/kernel"] = (F, F)
            want[f"{b}/project_out/kernel"] = (F, F)
        for m in (["Attention1", "Attention2"] if both else ["Attention2"]):
            for k in ("to_q", "to_k", "to_v"):
                want[f"{a}/{m}/{k}/kernel"] = (F, h, d)
            want[f"{a}/{m}/to_out_0/kernel"] = (h, d, F)
        want.update({f"{a}/ff/net_0/proj/kernel": (F, 8 * F), f"{a}/ff/net_0/proj/bias": (8 * F,),
                     f"{a}/ff/net_2/kernel": (4 * F, F), f"{a}/ff/net_2/bias": (F,),
                     f"{a}/norm2/scale": (F,), f"{a}/norm3/scale": (F,)})
        if both:
            want[f"{a}/norm1/scale"] = (F,)
    for i in range(half):
        want[f"up_dense_{i}/kernel"] = (2 * F, F)
        want[f"up_dense_{i}/bias"] = (F,)
    return want


SMALL = dict(patch_size=4, emb_features=64, num_layers=2, num_heads=2)


@pytest.mark.parametrize("kw,names", [
    ({}, {}),
    (dict(context_dim=32), dict(ctx=32)),
    (dict(use_projection=True), dict(proj=True)),
    (dict(use_self_and_cross=True, context_dim=16), dict(both=True, ctx=16)),
    (dict(norm_inputs=True), dict(norm_in=True)),
    (dict(use_hilbert=True), dict(hilbert=True)),
    (dict(add_residualblock_output=True, context_dim=8), dict(head=True, ctx=8)),
])
def test_parameter_names_and_shapes(kw, names):
    m = UViT(**SMALL, **kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(64, 2, 4, 2, names.pop("ctx", None), **names)
    order = list(m.layout().table)       # the layout follows the forward order
    assert order.index("up_dense_0/bias") + 1 == order.index(m._ada_leaf("up_block_0"))


@pytest.mark.parametrize("p", [2, 16])
def test_training_py_configuration(p):
    """training.py's `uvit` entry: the default emb_features (768), 12 layers, 12 heads; p = 2 and 16."""
    m = UViT(patch_size=p, num_layers=12, num_heads=12, dropout_rate=0.1, add_residualblock_output=False,
             use_flash_attention=False, use_self_and_cross=False, use_hilbert=False, context_dim=768)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(768, 12, p, 12, 768)
    assert got["pos_encoding"] == (1, (512 // p) ** 2, 768)


def test_init_and_config_round_trip():
    m = UViT(**SMALL, context_dim=16, add_residualblock_output=True, activation="mish", use_hilbert=True)
    fp = m.init(0, device="cpu")
    assert fp.named["pos_encoding"].std().item() == pytest.approx(0.02, rel=0.05)
    assert fp.named["final_proj/kernel"].abs().max().item() == 0
    assert fp.named["up_dense_0/kernel"].std().item() == pytest.approx((1 / 128) ** 0.5, rel=0.2)   # lecun, fan-in 2F
    assert fp.named["final_conv1/conv/kernel"].std().item() == pytest.approx((1 / 54) ** 0.5, rel=0.2)
    assert fp.named["final_norm_conv/scale"].min().item() == 1
    m2 = UViT(**m.config())
    assert m2.layout().table == m.layout().table and m2.config() == m.config()


@pytest.mark.parametrize("kw,msg", [
    (dict(num_layers=3), "num_layers=3 must be even"),
    (dict(use_flash_attention=True), "use_flash_attention"),
    (dict(dtype=torch.float32), "dtype"),
    (dict(emb_features=768, num_heads=7), "not a multiple of num_heads"),
    (dict(emb_features=1024, num_heads=2), "head width 512 > 256"),
    (dict(emb_features=96, num_heads=2), "multiple of 64, at most 1024"),
    (dict(emb_features=1536, num_heads=12), "multiple of 64, at most 1024"),
    (dict(add_residualblock_output=True, activation="relu"), "activation 'relu'"),
    (dict(add_residualblock_output=True, output_channels=4), "output_channels=3"),
])
def test_constructor_refusals_name_the_class(kw, msg):
    args = dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12)
    args.update(kw)
    with pytest.raises(FdxError, match="UViT") as e:
        UViT(**args)
    assert msg in str(e.value)


@pytest.mark.parametrize("shape,ctx,msg", [
    ((1, 18, 16, 3), None, "not divisible by the patch size"),
    ((1, 16, 16, 4), None, "3 channels"),
    ((1, 16, 16, 3), (1, 8), "must be [B, T, D]"),
])
def test_call_refusals(shape, ctx, msg):
    """Refused before anything reaches the device (the inputs are CPU tensors)."""
    m = UViT(**SMALL, context_dim=8 if ctx else None)
    fp = m.init(0, device="cpu")
    c = torch.zeros(*ctx) if ctx else None
    with pytest.raises(FdxError) as e:
        m.forward(fp, torch.zeros(*shape), torch.zeros(1), c)
    assert msg in str(e.value)


def test_more_patches_than_the_position_table_is_refused():
    m = UViT(patch_size=16, emb_features=64, num_layers=2, num_heads=2)     # (512 / 16)^2 = 1024 rows
    fp = m.init(0, device="cpu")
    with pytest.raises(FdxError, match="1089 patches exceed pos_encoding's 1024 rows"):
        m.forward(fp, torch.zeros(1, 528, 528, 3), torch.zeros(1))


def test_ignored_arguments_are_accepted():
    UViT(**SMALL, dropout_rate=0.3, norm_groups=0, force_fp32_for_softmax=False, use_remat=True, precision="high")


# ------------------------------------------------------------------------------------------------------ Hilbert
@pytest.mark.parametrize("grid", ["4x4", "8x8", "6x4", "3x5"])
def test_hilbert_orders_follow_the_reference(grid):
    """Sequence position s holds row-major patch idx[idx[s]] (hilbert_patchify's gather, then __call__'s), and the
    output returns through inv_idx once: row-major k <- sequence inv_idx[k]."""
    HP, WP = (int(v) for v in grid.split("x"))
    idx = np.asarray(json.load(open(GOLDEN))[grid]["hilbert"])
    m = UViT(**SMALL, use_hilbert=True)
    gather_in, gather_out, inv_of_out = (t.numpy() for t in m._order(HP, WP, "cpu"))
    assert np.array_equal(gather_in, idx[idx])
    inv = np.empty_like(idx)
    inv[idx] = np.arange(len(idx))
    assert np.array_equal(gather_out, inv)
    assert np.array_equal(inv_of_out[gather_out], np.arange(len(idx)))
    assert UViT(**SMALL)._order(HP, WP, "cpu") is None


# ------------------------------------------------------------------------------------------------------ oracle
def _params(m, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    fp = m.init(seed, device="cpu")
    return {k: (v.to(dtype) + 0.2 * torch.randn(v.shape, generator=g, dtype=dtype)) for k, v in fp.named.items()}


def test_oracle_closed_form_pins_the_skip_pairing_and_the_double_residual():
    """Zero to_out_0 kernels and zero ff/net_2 kernels and biases make every block out = x + (x + 0 + 0) = 2x.  The
    output is then a hand-computable chain: up layer i reads [x, skip of down_block_{half-1-i}]."""
    m = UViT(patch_size=2, emb_features=64, num_layers=6, num_heads=2, context_dim=8)
    P = _params(m, 1)
    for k in P:
        if k.endswith("to_out_0/kernel") or "/ff/net_2/" in k:
            P[k].zero_()
    B, H, W, p, F, half = 2, 8, 8, 2, 64, 3
    x = torch.randn(B, H, W, 3, dtype=torch.float64)
    t = torch.rand(B, dtype=torch.float64)
    ctx = torch.randn(B, 5, 8, dtype=torch.float64)
    freqs = m._fourier_freqs("cpu").double()
    got = uvit_ref.uvit_forward(P, x, t, freqs, patch_size=p, num_layers=6, num_heads=2, textcontext=ctx)

    N = (H // p) * (W // p)
    patches = x.reshape(B, H // p, p, W // p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(B, N, -1)
    tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(-1, F) + P["patch_embed/Conv_0/bias"] + \
        P["pos_encoding"][:, :N]
    seq = torch.cat([tok, uvit_ref.time_token(P, t, freqs)[:, None], ctx @ P["text_proj/kernel"] + P["text_proj/bias"]],
                    1)
    skips = []
    for i in range(half):
        seq = 2 * seq
        skips.append(seq)
    seq = 2 * seq
    for i in range(half):
        k = P[f"up_dense_{i}/kernel"]
        seq = 2 * (seq @ k[:F] + skips[half - 1 - i] @ k[F:] + P[f"up_dense_{i}/bias"])
    y = layernorm(seq, 1e-5, P["final_norm/scale"], P["final_norm/bias"])[:, :N] @ P["final_proj/kernel"] + \
        P["final_proj/bias"]
    want = y.reshape(B, H // p, W // p, p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, 3)
    torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)
    assert not torch.allclose(skips[0] @ P["up_dense_0/kernel"][F:], skips[2] @ P["up_dense_0/kernel"][F:])


@pytest.mark.parametrize("kw", [dict(), dict(use_projection=True, use_self_and_cross=True, norm_inputs=True),
                                dict(add_residualblock_output=True, activation="mish", use_hilbert=True)])
def test_oracle_gradcheck(kw):
    m = UViT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=4, **kw)
    P = _params(m, 4)
    x = torch.randn(1, 4, 4, 3, dtype=torch.float64)
    t = torch.rand(1, dtype=torch.float64)
    ctx = torch.randn(1, 3, 4, dtype=torch.float64)
    freqs = m._fourier_freqs("cpu").double()
    names = ["up_dense_0/kernel", "pos_encoding", "final_proj/kernel", "text_proj/kernel",
             "mid_block/Attention/ff/net_0/proj/bias", "down_block_0/Attention/norm2/scale"]
    if kw.get("add_residualblock_output"):
        names += ["final_conv1/conv/bias", "final_norm_conv/scale", "final_conv2/conv/bias"]
    leaves = [P[n].reshape(-1)[:4].clone().requires_grad_(True) for n in names]
    opts = {k: getattr(m, k) for k in ("use_projection", "use_self_and_cross", "norm_inputs",
                                        "explicitly_add_residual", "add_residualblock_output", "activation")}

    def f(*vals):
        Q = dict(P)
        for n, v in zip(names, vals):
            w = P[n].clone().reshape(-1)
            w = torch.cat([v, w[4:]])
            Q[n] = w.reshape(P[n].shape)
        return uvit_ref.uvit_forward(Q, x, t, freqs, patch_size=2, num_layers=2, num_heads=2, textcontext=ctx,
                                     order=m._scan_indices(2, 2), **opts)
    assert torch.autograd.gradcheck(f, leaves, eps=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------------ ptxas
@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_uvit_kernels_have_no_spills_and_no_frames():
    frames, _ = _report("fdx_uvit.cu")
    uvit = {k: v for k, v in frames.items() if "uvit_" in k}
    assert len(uvit) == 13, sorted(frames)   # assembly, split, 2 position passes, 2 x 2 norm + finish, 4 im2col
    assert all(v == (0, 0, 0) for v in uvit.values()), uvit
