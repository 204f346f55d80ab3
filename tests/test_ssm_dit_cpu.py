"""HybridSSMAttentionDiT host logic (no GPU): parameter names and shapes, the block pattern, the S5 initialisation, the
constructor's refusals and a config round trip, the Hilbert / zigzag patch orders against the reference's own functions,
the oracle against a closed form and against finite differences, and a ptxas guard for fdx_ssm.cu.

Parameter names follow flax's rules for the reference's modules (no hybrid checkpoint exists in the reference tree):
SSMDiTBlock names ada_params_module, ssm and mlp; BidirectionalS5Layer names its two S5Layers s5_forward / s5_backward
and its Dense out_proj; S5Layer's leaves are self.param names.  Block indices are positions in the pattern."""
import json
import math
import os

import numpy as np
import pytest
import torch

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.simple_dit import SimpleDiT
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT, build_block_pattern, hilbert_indices, zigzag_indices
from oracle import ssm_dit_ref
from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scan_orders.json")


def _s5(base, N, F):
    return {f"{base}/log_A_real": (N,), f"{base}/A_imag": (N,), f"{base}/B_re": (N, F), f"{base}/B_im": (N, F),
            f"{base}/C_re": (F, N), f"{base}/C_im": (F, N), f"{base}/D": (F,), f"{base}/log_dt": (N,)}


def _names(F, h, p, E, pattern, N, bidir=True, scan=False, ctx=None, sigma=False):
    d = F // h
    n = p * p * 3 * (2 if sigma else 1)
    want = {"time_embed/layers_1/DenseGeneral_0/kernel": (F, E), "time_embed/layers_1/DenseGeneral_0/bias": (E,),
            "time_embed/layers_1/DenseGeneral_1/kernel": (E, E), "time_embed/layers_1/DenseGeneral_1/bias": (E,),
            "time_embed/layers_2/kernel": (E, F), "time_embed/layers_2/bias": (F,),
            "final_norm/scale": (F,), "final_norm/bias": (F,), "final_proj/kernel": (F, n), "final_proj/bias": (n,)}
    if scan:
        want.update({"hilbert_projection/kernel": (p * p * 3, F), "hilbert_projection/bias": (F,)})
    else:
        want.update({"patch_embed/Conv_0/kernel": (p, p, 3, F), "patch_embed/Conv_0/bias": (F,)})
    if ctx:
        want.update({"text_context_proj/kernel": (ctx, F), "text_context_proj/bias": (F,)})
    for i, kind in enumerate(pattern):
        b = f"{'ssm' if kind == 'ssm' else 'dit'}_block_{i}"
        want[f"{b}/ada_params_module/ada_proj/kernel"] = (F, 6 * F)
        want[f"{b}/ada_params_module/ada_proj/bias"] = (6 * F,)
        if kind == "ssm":
            if bidir:
                want.update(_s5(f"{b}/ssm/s5_forward", N, F))
                want.update(_s5(f"{b}/ssm/s5_backward", N, F))
                want[f"{b}/ssm/out_proj/kernel"] = (2 * F, F)
                want[f"{b}/ssm/out_proj/bias"] = (F,)
            else:
                want.update(_s5(f"{b}/ssm", N, F))
        else:
            for m in ("to_q", "to_k", "to_v"):
                want[f"{b}/attention/{m}/kernel"] = (F, h, d)
                want[f"{b}/attention/{m}/bias"] = (h, d)
            want[f"{b}/attention/to_out_0/kernel"] = (h, d, F)
            want[f"{b}/attention/to_out_0/bias"] = (F,)
        want[f"{b}/mlp/layers_0/kernel"] = (F, E)
        want[f"{b}/mlp/layers_0/bias"] = (E,)
        want[f"{b}/mlp/layers_2/kernel"] = (E, F)
        want[f"{b}/mlp/layers_2/bias"] = (F,)
    return want


S31 = ["ssm", "ssm", "ssm", "attn"]


@pytest.mark.parametrize("kw,want", [
    (dict(patch_size=2, emb_features=64, num_layers=4, num_heads=2, ssm_state_dim=16),
     dict(F=64, h=2, p=2, E=256, pattern=S31, N=16)),
    (dict(patch_size=2, emb_features=64, num_layers=4, num_heads=2, ssm_state_dim=32, bidirectional_ssm=False),
     dict(F=64, h=2, p=2, E=256, pattern=S31, N=32, bidir=False)),
    (dict(patch_size=4, emb_features=128, num_layers=2, num_heads=4, ssm_state_dim=16, use_hilbert=True,
          ssm_attention_ratio="1:1"),
     dict(F=128, h=4, p=4, E=512, pattern=["ssm", "attn"], N=16, scan=True)),
    (dict(patch_size=2, emb_features=64, num_layers=3, num_heads=2, ssm_state_dim=16, use_zigzag=True,
          context_dim=96, learn_sigma=True),
     dict(F=64, h=2, p=2, E=256, pattern=S31[:3], N=16, scan=True, ctx=96, sigma=True)),
    (dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12), dict(F=768, h=12, p=2, E=3072,
                                                                             pattern=S31 * 3, N=64)),  # hybrid-B/2
])
def test_parameter_names_and_shapes(kw, want):
    m = HybridSSMAttentionDiT(**kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(**want)


def test_all_attn_has_simple_dit_parameters():
    kw = dict(patch_size=2, emb_features=128, num_layers=3, num_heads=4, context_dim=32, learn_sigma=True)
    assert HybridSSMAttentionDiT(ssm_attention_ratio="all-attn", **kw).param_specs() == SimpleDiT(**kw).param_specs()


@pytest.mark.parametrize("layers,ratio,pattern,want", [
    (12, "3:1", None, S31 * 3),
    (7, "2:1", None, ["ssm", "ssm", "attn", "ssm", "ssm", "attn", "ssm"]),
    (5, "1:1", None, ["ssm", "attn", "ssm", "attn", "ssm"]),
    (3, "all-ssm", None, ["ssm"] * 3),
    (3, "all-attn", None, ["attn"] * 3),
    (4, "3:1", ["attn", "ssm", "mamba", "ssm", "ssm"], ["attn", "ssm", "mamba", "ssm", "ssm"]),
    (2, "0:1", None, ["attn", "attn"]),
])
def test_block_pattern(layers, ratio, pattern, want):
    assert build_block_pattern(layers, pattern, ratio) == want
    m = HybridSSMAttentionDiT(emb_features=64, num_heads=2, num_layers=layers, ssm_state_dim=16,
                              ssm_attention_ratio=ratio, block_pattern=pattern)
    names = [n for n, _, _ in m._blocks()]
    assert names == [f"{'ssm' if k == 'ssm' else 'dit'}_block_{i}" for i, k in enumerate(want)]


def test_init_follows_s5_layer():
    F, N = 256, 64
    m = HybridSSMAttentionDiT(patch_size=2, emb_features=F, num_layers=1, num_heads=4, ssm_state_dim=N,
                              ssm_attention_ratio="all-ssm")
    P = m.init(3, device=torch.device("cpu")).named
    n = torch.arange(N, dtype=torch.float32)
    for base in ("ssm_block_0/ssm/s5_forward", "ssm_block_0/ssm/s5_backward"):
        assert torch.allclose(P[f"{base}/log_A_real"], torch.log(n + 0.5))
        assert torch.allclose(P[f"{base}/A_imag"], math.pi * n)
        ld = P[f"{base}/log_dt"]
        assert ld.min() >= math.log(0.001) and ld.max() <= math.log(0.1) and ld.std() > 0.5
        assert abs(P[f"{base}/D"].std().item() - 1.0) < 0.2
        for leaf, fan_in in (("B_re", N), ("B_im", N), ("C_re", F), ("C_im", F)):
            std = P[f"{base}/{leaf}"].std().item()
            assert abs(std * math.sqrt(fan_in) - 1.0) < 0.1, (leaf, std, fan_in)
    std = P["ssm_block_0/ssm/out_proj/kernel"].std().item()
    assert abs(std * math.sqrt(2 * F) - 1.0) < 0.1
    assert not P["ssm_block_0/ssm/s5_forward/B_re"].equal(P["ssm_block_0/ssm/s5_backward/B_re"])


@pytest.mark.parametrize("kw,match", [
    (dict(use_hilbert=True, use_zigzag=True), "mutually exclusive"),
    (dict(use_2d_fusion=True), "use_2d_fusion"),
    (dict(ssm_state_dim=24), "multiple of 16"),
    (dict(ssm_state_dim=0), "multiple of 16"),
    (dict(ssm_attention_ratio="3-1"), "ssm_attention_ratio"),
    (dict(ssm_attention_ratio="a:b"), "ssm_attention_ratio"),
    (dict(ssm_attention_ratio="0:0"), "ssm_attention_ratio"),
    (dict(ssm_attention_ratio="1:2:3"), "ssm_attention_ratio"),
    (dict(use_flash_attention=True), "flash"),
    (dict(dtype=torch.float32), "dtype"),
    (dict(emb_features=768, num_heads=10), "multiple of num_heads"),
    (dict(emb_features=192, num_heads=64), "odd"),
])
def test_constructor_refusals(kw, match):
    with pytest.raises(FdxError, match=match):
        HybridSSMAttentionDiT(**kw)


def test_simple_dit_still_refuses_scan_orders():
    for kw in (dict(use_hilbert=True), dict(use_zigzag=True)):
        with pytest.raises(FdxError, match="Hilbert / zigzag"):
            SimpleDiT(**kw)


def test_config_round_trip():
    m = HybridSSMAttentionDiT(patch_size=4, emb_features=192, num_layers=5, num_heads=3, mlp_ratio=2, learn_sigma=True,
                              context_dim=64, ssm_state_dim=32, ssm_attention_ratio="2:1", bidirectional_ssm=False,
                              use_zigzag=True, block_pattern=("ssm", "attn", "ssm"))
    m2 = HybridSSMAttentionDiT(**m.config())
    assert m2.config() == m.config() and m2.param_specs() == m.param_specs() and m2.pattern == m.pattern


@pytest.mark.parametrize("grid", ["1x1", "2x2", "4x4", "8x8", "16x16", "64x64", "6x4", "3x5", "16x8"])
def test_scan_orders_match_the_reference(grid):
    gold = json.load(open(GOLDEN))[grid]
    HP, WP = (int(v) for v in grid.split("x"))
    for name, fn in (("hilbert", hilbert_indices), ("zigzag", zigzag_indices)):
        got = fn(HP, WP)
        assert got.tolist() == gold[name], name
        assert sorted(got.tolist()) == list(range(HP * WP)), name


def test_scan_order_position_table_and_inverse():
    m = HybridSSMAttentionDiT(emb_features=64, num_heads=2, num_layers=1, ssm_state_dim=16, use_hilbert=True)
    idx = m._scan_indices(6, 4)
    tab = m._const("pos", torch.device("cpu"), 6, 4).float()
    raster = HybridSSMAttentionDiT(emb_features=64, num_heads=2, num_layers=1, ssm_state_dim=16)
    assert torch.equal(tab, raster._const("pos", torch.device("cpu"), 6, 4).float()[torch.from_numpy(idx)])
    fwd, inv = m._order(6, 4, torch.device("cpu"))
    assert torch.equal(fwd[inv.long()], torch.arange(24, dtype=torch.int32))


def _params(N, F, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=dtype)  # noqa: E731
    n = torch.arange(N, dtype=dtype)
    return {"s/log_A_real": torch.log(n + 0.5) + 0.1 * r(N), "s/A_imag": math.pi * n + 0.1 * r(N),
            "s/log_dt": math.log(0.01) + r(N), "s/B_re": r(N, F) / N ** 0.5, "s/B_im": r(N, F) / N ** 0.5,
            "s/C_re": r(F, N) / F ** 0.5, "s/C_im": r(F, N) / F ** 0.5, "s/D": r(F)}


def test_oracle_s5_is_a_geometric_series_for_constant_input():
    """One state, one feature, u = 1: x_k = Bbar (1 - Abar^(k+1)) / (1 - Abar), y_k = Re(C x_k) + D."""
    lar, ai, ldt, br, bi, cr, ci, D = 0.3, 2.0, math.log(0.05), 0.7, -0.4, 1.1, 0.6, 0.25
    P = {"s/log_A_real": torch.tensor([lar]), "s/A_imag": torch.tensor([ai]), "s/log_dt": torch.tensor([ldt]),
         "s/B_re": torch.tensor([[br]]), "s/B_im": torch.tensor([[bi]]), "s/C_re": torch.tensor([[cr]]),
         "s/C_im": torch.tensor([[ci]]), "s/D": torch.tensor([D])}
    P = {k: v.double() for k, v in P.items()}
    L = 50
    y = ssm_dit_ref.s5_layer(P, "s", torch.ones(1, L, 1, dtype=torch.float64))[0, :, 0]
    A = complex(-math.exp(lar), ai)
    dt = math.exp(ldt)
    ab = np.exp(A * dt)
    bb = (ab - 1) / (A + 1e-8) * complex(br, bi)
    k = np.arange(L)
    x = bb * (1 - ab ** (k + 1)) / (1 - ab)
    want = (complex(cr, ci) * x).real + D
    np.testing.assert_allclose(y.numpy(), want, rtol=1e-7, atol=1e-9)


@pytest.mark.parametrize("bidirectional", [True, False])
def test_oracle_s5_gradients_pass_gradcheck(bidirectional):
    N, F, B, L = 3, 4, 2, 5
    P = {}
    for d, base in enumerate(("blk/ssm/s5_forward", "blk/ssm/s5_backward") if bidirectional else ("blk/ssm",)):
        P.update({k.replace("s/", base + "/"): v for k, v in _params(N, F, torch.float64, seed=d).items()})
    g = torch.Generator().manual_seed(9)
    if bidirectional:
        P["blk/ssm/out_proj/kernel"] = torch.randn(2 * F, F, generator=g, dtype=torch.float64) / 3
        P["blk/ssm/out_proj/bias"] = torch.randn(F, generator=g, dtype=torch.float64)
    u = torch.randn(B, L, F, generator=g, dtype=torch.float64)
    names = sorted(P)

    def f(*vals):
        return ssm_dit_ref.ssm(dict(zip(names, vals)), "blk", u, bidirectional)

    assert torch.autograd.gradcheck(f, tuple(P[k].clone().requires_grad_(True) for k in names))


pytestmark_ptxas = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytestmark_ptxas
def test_ssm_kernels_have_no_spills_and_no_frames():
    frames, notes = _report("fdx_ssm.cu")
    ours = {k: v for k, v in frames.items() if "ssm_" in k or "permute_rows" in k}
    assert len(ours) == 7, sorted(frames)
    assert all(v == (0, 0, 0) for v in ours.values()), ours
    assert not notes, notes
