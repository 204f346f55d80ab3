"""SimpleMMDiT host logic (no GPU): parameter names and shapes with and without the Hilbert order, init, the
constructor's refusals, a config round trip, the Hilbert table, the oracle against closed forms and gradcheck, and a
ptxas guard for fdx_mmdit.cu.

Parameter names: SimpleMMDiT.setup (simple_mmdit.py:187-255) names patch_embed, time_embed, hilbert_projection (only
under use_hilbert), text_context_proj, mmdit_block_{i}, final_norm and final_proj.  patch_embed is built in setup but
only called in raster order, so under use_hilbert it has no parameters.  MMDiTBlock names ada_ln_zero (MMAdaLNZero, with
its Dense ada_t_proj / ada_text_proj), attention (RoPEAttention: to_q / to_k / to_v / to_out_0 with biases) and mlp
(nn.Sequential: layers_0, the gelu, layers_2).  No SimpleMMDiT checkpoint exists in the reference tree, so the names
are derived from flax's naming rules, not pinned against a file flax wrote."""
import json
import math
import os

import pytest
import torch

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.mmdit import SimpleMMDiT
from flaxdiff_b200.models.ssm_dit import hilbert_indices
from oracle import mmdit_ref
from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scan_orders.json")


def _names(F, h, p, E, layers, ctx, out=3, sigma=False, hilbert=False):
    d = F // h
    n = p * p * out * (2 if sigma else 1)
    want = {"time_embed/layers_1/DenseGeneral_0/kernel": (F, E), "time_embed/layers_1/DenseGeneral_0/bias": (E,),
            "time_embed/layers_1/DenseGeneral_1/kernel": (E, E), "time_embed/layers_1/DenseGeneral_1/bias": (E,),
            "time_embed/layers_2/kernel": (E, F), "time_embed/layers_2/bias": (F,),
            "text_context_proj/kernel": (ctx, F), "text_context_proj/bias": (F,),
            "final_norm/scale": (F,), "final_norm/bias": (F,), "final_proj/kernel": (F, n), "final_proj/bias": (n,)}
    if hilbert:
        want.update({"hilbert_projection/kernel": (p * p * 3, F), "hilbert_projection/bias": (F,)})
    else:
        want.update({"patch_embed/Conv_0/kernel": (p, p, 3, F), "patch_embed/Conv_0/bias": (F,)})
    for i in range(layers):
        b = f"mmdit_block_{i}"
        for a in ("ada_t_proj", "ada_text_proj"):
            want[f"{b}/ada_ln_zero/{a}/kernel"] = (F, 6 * F)
            want[f"{b}/ada_ln_zero/{a}/bias"] = (6 * F,)
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


@pytest.mark.parametrize("kw,F,h,p,E,layers,ctx,sigma,hilbert", [
    (dict(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=32), 64, 2, 2, 256, 2, 32, False,
     False),
    (dict(patch_size=2, emb_features=128, num_layers=1, num_heads=4, context_dim=768, learn_sigma=True,
          use_hilbert=True), 128, 4, 2, 512, 1, 768, True, True),
    (dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12, context_dim=768), 768, 12, 2, 3072, 12, 768,
     False, False),                                                   # the reference's simple_mmdit config
])
def test_parameter_names_and_shapes(kw, F, h, p, E, layers, ctx, sigma, hilbert):
    m = SimpleMMDiT(**kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(F, h, p, E, layers, ctx, sigma=sigma, hilbert=hilbert)


def test_ada_kernels_are_adjacent_so_their_stack_is_a_view():
    m = SimpleMMDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=32)
    fp = m.init(0, device="cpu")
    for i in range(2):
        st = m._ada_stack(fp.named, f"mmdit_block_{i}")
        assert torch.equal(st[:64], fp.named[f"mmdit_block_{i}/ada_ln_zero/ada_t_proj/kernel"])
        assert torch.equal(st[64:], fp.named[f"mmdit_block_{i}/ada_ln_zero/ada_text_proj/kernel"])


def test_init_follows_flax():
    """ada_t_proj / ada_text_proj / final_proj kernels zero; LayerNorm scales one; biases zero; every other kernel
    lecun-normal (truncated normal, variance 1 / fan-in)."""
    m = SimpleMMDiT(patch_size=2, emb_features=256, num_layers=2, num_heads=4, context_dim=512, use_hilbert=True)
    fp = m.init(7, device="cpu")
    for name, t in fp.named.items():
        leaf = name.rsplit("/", 1)[1]
        if leaf == "bias":
            assert t.abs().max().item() == 0, name
        elif leaf == "scale":
            assert torch.equal(t, torch.ones_like(t)), name
        elif "/ada_ln_zero/" in name or name.startswith("final_proj"):
            assert t.abs().max().item() == 0, name
        else:
            fan_in = t.shape[0] * t.shape[1] if name.endswith("to_out_0/kernel") else t.shape[0]
            std = t.std().item() * math.sqrt(fan_in)
            assert 0.9 < std < 1.1, (name, std)
            assert t.abs().max().item() <= 2 / 0.87962566103423978 / math.sqrt(fan_in) + 1e-6, name


@pytest.mark.parametrize("kw,match", [
    (dict(use_flash_attention=True), "flash"),
    (dict(dtype=torch.float32), "dtype"),
    (dict(emb_features=768, num_heads=10), "multiple of num_heads"),
    (dict(emb_features=192, num_heads=64), "odd"),
    (dict(emb_features=612, num_heads=12), "odd"),          # training.py's hierarchical mapping: 51-wide heads
    (dict(emb_features=512, num_heads=1), "> 256"),
    (dict(emb_features=96, num_heads=2), "multiple of 64"),
    (dict(emb_features=1600, num_heads=25), "at most 1536"),
])
def test_constructor_refusals(kw, match):
    with pytest.raises(FdxError, match=match):
        SimpleMMDiT(**kw)


def test_text_is_required():
    m = SimpleMMDiT(patch_size=2, emb_features=64, num_layers=1, num_heads=2)
    with pytest.raises(FdxError, match="text conditioning is required"):
        m.layout()
    with pytest.raises(FdxError, match="text conditioning is required"):
        m.init(0, device="cpu")
    m = SimpleMMDiT(patch_size=2, emb_features=64, num_layers=1, num_heads=2, context_dim=32)
    with pytest.raises(FdxError, match="textcontext is required"):
        m.forward(None, torch.zeros(1, 8, 8, 3), torch.zeros(1), None)
    with pytest.raises(FdxError, match="must be"):
        m.forward(None, torch.zeros(1, 8, 8, 3), torch.zeros(1), torch.zeros(1, 2, 3, 32))


def test_image_not_divisible_by_patch_is_refused():
    m = SimpleMMDiT(patch_size=4, emb_features=64, num_layers=1, num_heads=2, context_dim=32)
    with pytest.raises(FdxError, match="divisible"):
        m.forward(None, torch.zeros(1, 18, 16, 3), torch.zeros(1), torch.zeros(1, 5, 32))


def test_ignored_arguments_are_accepted():
    a = SimpleMMDiT(emb_features=64, num_heads=2, num_layers=1, context_dim=32, norm_groups=8, dropout_rate=0.1,
                    activation=torch.nn.functional.silu, force_fp32_for_softmax=False)
    b = SimpleMMDiT(emb_features=64, num_heads=2, num_layers=1, context_dim=32)
    assert a.param_specs() == b.param_specs()


def test_config_round_trip():
    m = SimpleMMDiT(patch_size=4, emb_features=192, num_layers=3, num_heads=3, mlp_ratio=2, learn_sigma=True,
                    context_dim=64, use_hilbert=True)
    m2 = SimpleMMDiT(**m.config())
    assert m2.config() == m.config() and m2.param_specs() == m.param_specs()
    assert "use_zigzag" not in m.config()


@pytest.mark.parametrize("grid", ["4x4", "8x8", "6x4", "3x5", "16x8"])
def test_hilbert_order_is_the_reference_table(grid):
    gold = json.load(open(GOLDEN))[grid]
    HP, WP = (int(v) for v in grid.split("x"))
    m = SimpleMMDiT(emb_features=64, num_heads=2, num_layers=1, context_dim=32, use_hilbert=True)
    assert m._scan_indices(HP, WP).tolist() == gold["hilbert"]
    fwd, inv = m._order(HP, WP, torch.device("cpu"))
    assert torch.equal(fwd[inv.long()], torch.arange(HP * WP, dtype=torch.int32))
    assert SimpleMMDiT(emb_features=64, num_heads=2, num_layers=1, context_dim=32)._scan_indices(HP, WP) is None


def test_no_position_table_and_rope_in_both_orders():
    for hilbert in (False, True):
        m = SimpleMMDiT(emb_features=64, num_heads=2, num_layers=1, context_dim=32, use_hilbert=hilbert)
        assert m._pos_table(torch.device("cpu"), 4, 4) is None and m._rope()


# ------------------------------------------------------------------------------------------ the oracle
def _oracle_params(F, h, p, layers, ctx, dtype=torch.float32, seed=0, zero_ada=False):
    g = torch.Generator().manual_seed(seed)
    P = {}
    for name, shape in _names(F, h, p, 4 * F, layers, ctx).items():
        t = torch.randn(shape, generator=g, dtype=dtype) / math.sqrt(shape[0])
        if zero_ada and ("/ada_ln_zero/" in name):
            t.zero_()
        P[name] = t
    P["final_norm/scale"] = 1 + 0.1 * torch.randn(F, generator=g, dtype=dtype)
    return P


def test_oracle_zero_ada_makes_every_block_the_identity():
    torch.manual_seed(0)
    F, h = 32, 2
    P = _oracle_params(F, h, 2, 1, 16, zero_ada=True)
    x = torch.randn(2, 9, F)
    y = mmdit_ref.mmdit_block(P, "mmdit_block_0", x, torch.randn(2, F), torch.randn(2, 5, F), h, 1e-5)
    assert torch.equal(y, x)


def test_oracle_text_pooling_is_linear():
    """Pooling the projected text per block (the reference's order) equals projecting the pooled text."""
    torch.manual_seed(1)
    F, h = 32, 2
    P = _oracle_params(F, h, 2, 1, 16, dtype=torch.float64)
    x, t = torch.randn(2, 9, F, dtype=torch.float64), torch.randn(2, F, dtype=torch.float64)
    ctx = torch.randn(2, 5, 16, dtype=torch.float64)
    per_token = mmdit_ref.mmdit_block(P, "mmdit_block_0", x, t, mmdit_ref.dense(P, "text_context_proj", ctx), h, 1e-5)
    pooled = mmdit_ref.mmdit_block(P, "mmdit_block_0", x, t,
                                   mmdit_ref.dense(P, "text_context_proj", ctx.mean(1)), h, 1e-5)
    torch.testing.assert_close(per_token, pooled, rtol=1e-12, atol=1e-12)


def test_oracle_clip_gradient_mask():
    v = torch.tensor([-12.0, -10.0, -9.5, 0.0, 9.99, 10.0, 11.0], dtype=torch.float64, requires_grad=True)
    y = mmdit_ref.clip10(v)
    assert y.tolist() == [-10.0, -10.0, -9.5, 0.0, 9.99, 10.0, 10.0]
    y.backward(torch.full_like(v, 3.0))
    assert v.grad.tolist() == [0.0, 1.5, 3.0, 3.0, 3.0, 1.5, 0.0]


def test_oracle_hilbert_order_round_trips_the_patches():
    """With the identity at every block and an identity-like patch map, Hilbert-ordered and raster runs agree: the
    order only permutes the tokens and is undone before unpatchify (RoPE aside, which zero ada makes moot)."""
    torch.manual_seed(2)
    F, h, p = 64, 2, 2
    P = _oracle_params(F, h, p, 1, 16, dtype=torch.float64, zero_ada=True)
    PH = dict(P)
    PH["hilbert_projection/kernel"] = P.pop("patch_embed/Conv_0/kernel").reshape(p * p * 3, F)
    PH["hilbert_projection/bias"] = P["patch_embed/Conv_0/bias"]
    del PH["patch_embed/Conv_0/bias"]
    x = torch.randn(2, 12, 8, 3, dtype=torch.float64)
    t, ctx = torch.rand(2), torch.randn(2, 5, 16, dtype=torch.float64)
    P["patch_embed/Conv_0/kernel"] = PH["hilbert_projection/kernel"].reshape(p, p, 3, F)
    kw = dict(patch_size=p, num_layers=1, num_heads=h)
    a = mmdit_ref.simple_mmdit_forward(P, x, t, torch.randn(F // 2), ctx, **kw)
    b = mmdit_ref.simple_mmdit_forward(PH, x, t, torch.randn(F // 2), ctx, order=hilbert_indices(6, 4), **kw)
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("text_dims", [2, 3])
def test_oracle_gradients_pass_gradcheck(text_dims):
    F, h, p = 8, 2, 2
    P = _oracle_params(F, h, p, 1, 6, dtype=torch.float64, seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 4, 6, 3, generator=g, dtype=torch.float64)
    t = torch.rand(1, generator=g, dtype=torch.float64)
    freqs = torch.randn(F // 2, generator=g, dtype=torch.float64)
    ctx = torch.randn(1, *((3, 6) if text_dims == 3 else (6,)), generator=g, dtype=torch.float64)
    names = sorted(P)

    def f(*vals):
        return mmdit_ref.simple_mmdit_forward(dict(zip(names, vals)), x, t, freqs, ctx, patch_size=p, num_layers=1,
                                              num_heads=h)

    assert torch.autograd.gradcheck(f, tuple(P[k].clone().requires_grad_(True) for k in names))


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_mmdit_kernels_have_no_spills_and_no_frames():
    frames, notes = _report("fdx_mmdit.cu")
    ours = {k: v for k, v in frames.items() if "mmdit_" in k}
    assert len(ours) == 10, sorted(ours)
    for name, (frame, stores, loads) in ours.items():
        assert frame == stores == loads == 0, (name, frame, stores, loads)
    assert not any("mmdit_" in k for k in notes), notes


# ------------------------------------------------------------------------------------------ HierarchicalMMDiT
# Names: HierarchicalMMDiT.setup (simple_mmdit.py:457-625) names patch_embed / hilbert_projection, time_embed_base,
# text_context_proj_base, t_emb_proj_stage{s}, text_emb_proj_stage{s}, encoder_block_stage{s}_{i}, patch_merger_{s}
# (PatchMerging: norm, projection), patch_expander_{s} (PatchExpanding: projection, norm), decoder_block_stage{s}_{i},
# final_norm and final_proj.  The fusion LayerNorm / Dense are explicitly named modules constructed inside setup() and
# then wrapped in an nn.Sequential: flax attaches a named module built in setup to the module being set up, so they are
# the top-level fusion_norm_{s} / fusion_dense_{s}, not fusion_layers_{i}/....  Derived from flax's rules; no
# HierarchicalMMDiT checkpoint exists to pin them against.
from flaxdiff_b200.models.mmdit import HierarchicalMMDiT  # noqa: E402


def _hier_names(Fs, hs, Ls, p, ctx, mlp=4, hilbert=False, sigma=False):
    N, FL = len(Fs), Fs[-1]
    E = FL * mlp
    te = "time_embed_base/layers_"
    want = {te + "1/DenseGeneral_0/kernel": (FL, E), te + "1/DenseGeneral_0/bias": (E,),
            te + "1/DenseGeneral_1/kernel": (E, E), te + "1/DenseGeneral_1/bias": (E,),
            te + "2/kernel": (E, FL), te + "2/bias": (FL,),
            "text_context_proj_base/kernel": (ctx, FL), "text_context_proj_base/bias": (FL,)}
    if hilbert:
        want.update({"hilbert_projection/kernel": (p * p * 3, Fs[0]), "hilbert_projection/bias": (Fs[0],)})
    else:
        want.update({"patch_embed/Conv_0/kernel": (p, p, 3, Fs[0]), "patch_embed/Conv_0/bias": (Fs[0],)})
    for s in range(N):
        F = Fs[s]
        for m in ("t_emb_proj", "text_emb_proj"):
            want[f"{m}_stage{s}/kernel"], want[f"{m}_stage{s}/bias"] = (FL, F), (F,)
        blocks = [f"encoder_block_stage{s}_{i}" for i in range(Ls[s])]
        if s < N - 1:
            blocks += [f"decoder_block_stage{s}_{i}" for i in range(Ls[s])]
            want.update({f"patch_merger_{s}/norm/scale": (4 * F,), f"patch_merger_{s}/norm/bias": (4 * F,),
                         f"patch_merger_{s}/projection/kernel": (4 * F, Fs[s + 1]),
                         f"patch_merger_{s}/projection/bias": (Fs[s + 1],),
                         f"patch_expander_{s}/projection/kernel": (Fs[s + 1], 4 * F),
                         f"patch_expander_{s}/projection/bias": (4 * F,),
                         f"patch_expander_{s}/norm/scale": (4 * F,), f"patch_expander_{s}/norm/bias": (4 * F,),
                         f"fusion_norm_{s}/scale": (2 * F,), f"fusion_norm_{s}/bias": (2 * F,),
                         f"fusion_dense_{s}/kernel": (2 * F, F), f"fusion_dense_{s}/bias": (F,)})
        for b in blocks:
            want.update({k.replace("mmdit_block_0", b): v for k, v in _names(F, hs[s], p, F * mlp, 1, ctx).items()
                         if k.startswith("mmdit_block_0/")})
    n = p * p * 3 * (2 if sigma else 1)
    want.update({"final_norm/scale": (Fs[0],), "final_norm/bias": (Fs[0],), "final_proj/kernel": (Fs[0], n),
                 "final_proj/bias": (n,)})
    return want


@pytest.mark.parametrize("kw", [
    dict(context_dim=768),                                                          # the class defaults
    dict(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 2), num_heads=(2, 2), context_dim=32,
         use_hilbert=True, learn_sigma=True),
    dict(base_patch_size=4, emb_features=(64, 128, 192), num_layers=(2, 1, 1), num_heads=(2, 2, 3), context_dim=64),
])
def test_hierarchical_parameter_names_and_shapes(kw):
    m = HierarchicalMMDiT(**kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _hier_names(m.emb_features, m.num_heads, m.num_layers, m.base_patch_size, kw["context_dim"],
                              hilbert=m.use_hilbert, sigma=m.learn_sigma)
    assert not any(k.startswith("fusion_layers") for k in got)


def test_hierarchical_stage_widths_and_block_counts():
    m = HierarchicalMMDiT(context_dim=768)
    names = [n for n, _, _ in m._blocks()]
    assert len(names) == (4 + 4 + 14) + (4 + 4)          # encoder stages 0, 1, 2; decoder stages 1, 0
    assert names[:4] == [f"encoder_block_stage0_{i}" for i in range(4)]
    assert names[22:26] == [f"decoder_block_stage1_{i}" for i in range(4)]
    assert names[-1] == "decoder_block_stage0_3"
    assert m._widths("encoder_block_stage2_13") == (1024, 16) and m._widths("decoder_block_stage1_0") == (768, 12)
    assert m._fourier_freqs(torch.device("cpu")).numel() == 512       # Fourier(F_last), not F_0


@pytest.mark.parametrize("kw,match", [
    (dict(emb_features=(512, 768), num_layers=(4, 4, 14)), "same number of stages"),
    (dict(num_heads=(8, 12)), "same number of stages"),
    (dict(emb_features=(510, 768, 1022), num_heads=(10, 12, 14)), "stage 0: head width 51 is odd"),
    (dict(emb_features=(512, 768, 1022), num_heads=(8, 12, 14)), "stage 2: head width 73 is odd"),
    (dict(emb_features=(512, 768, 1024), num_heads=(8, 12, 2)), "> 256"),
    (dict(emb_features=(512, 96, 1024), num_heads=(8, 2, 16)), "multiple of 64"),
    (dict(use_flash_attention=True), "flash"),
    (dict(dtype=torch.float16), "dtype"),
])
def test_hierarchical_refusals(kw, match):
    with pytest.raises(FdxError, match=match):
        HierarchicalMMDiT(context_dim=32, **kw)


def test_hierarchical_image_divisibility_and_text_are_checked():
    m = HierarchicalMMDiT(base_patch_size=2, emb_features=(64, 128, 192), num_layers=(1, 1, 1), num_heads=(2, 2, 3),
                          context_dim=32)
    with pytest.raises(FdxError, match="coarsest patch size 2 \\* 2\\^2 = 8"):
        m.forward(None, torch.zeros(1, 12, 16, 3), torch.zeros(1), torch.zeros(1, 5, 32))
    with pytest.raises(FdxError, match="textcontext is required"):
        m.forward(None, torch.zeros(1, 16, 16, 3), torch.zeros(1), None)


def test_hierarchical_config_round_trip():
    m = HierarchicalMMDiT(base_patch_size=4, emb_features=(64, 128), num_layers=(1, 3), num_heads=(2, 4), mlp_ratio=2,
                          learn_sigma=True, use_hilbert=True, context_dim=64)
    m2 = HierarchicalMMDiT(**m.config())
    assert m2.config() == m.config() and m2.param_specs() == m.param_specs()


def test_oracle_merge_and_expand_match_loops_and_invert():
    B, HP, WP, C = 2, 6, 4, 3
    x = torch.randn(B, HP * WP, C)
    mg = mmdit_ref.patch_merge(x, HP, WP)
    for b in range(B):
        for h in range(HP // 2):
            for w in range(WP // 2):
                for p1 in range(2):
                    for p2 in range(2):
                        got = mg[b, h * (WP // 2) + w, (p1 * 2 + p2) * C:(p1 * 2 + p2 + 1) * C]
                        assert torch.equal(got, x[b, (2 * h + p1) * WP + 2 * w + p2])
    assert torch.equal(mmdit_ref.patch_expand(mg, HP // 2, WP // 2), x)
    y = torch.randn(B, 6, 4 * C)
    assert torch.equal(mmdit_ref.patch_merge(mmdit_ref.patch_expand(y, 3, 2), 6, 4), y)


def _hier_oracle_params(Fs, hs, Ls, p, ctx, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    P = {}
    for name, shape in _hier_names(Fs, hs, Ls, p, ctx).items():
        P[name] = torch.randn(shape, generator=g, dtype=dtype) / math.sqrt(shape[0])
        if name.endswith("/scale"):
            P[name] = 1 + 0.1 * P[name]
    return P


def test_hierarchical_oracle_gradients_pass_gradcheck():
    Fs, hs, Ls, p = (8, 12), (2, 2), (1, 1), 1
    P = _hier_oracle_params(Fs, hs, Ls, p, 6, torch.float64, 5)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, 4, 2, 3, generator=g, dtype=torch.float64)
    t = torch.rand(1, generator=g, dtype=torch.float64)
    freqs = torch.randn(Fs[-1] // 2, generator=g, dtype=torch.float64)
    ctx = torch.randn(1, 3, 6, generator=g, dtype=torch.float64)
    names = sorted(P)

    def f(*vals):
        return mmdit_ref.hierarchical_mmdit_forward(dict(zip(names, vals)), x, t, freqs, ctx, base_patch_size=p,
                                                    num_layers=Ls, num_heads=hs)

    assert torch.autograd.gradcheck(f, tuple(P[k].clone().requires_grad_(True) for k in names))
