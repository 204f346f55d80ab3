"""SimpleDiT host logic (no GPU): parameter names and shapes, the constructor's refusals, the oracle against closed forms
and a config round trip.

Parameter names: SimpleDiT.setup (simple_dit.py:121-207) names its submodules patch_embed, time_embed,
text_context_proj, dit_block_{i}, final_norm and final_proj.  PatchEmbedding's conv is its first nn.Conv (Conv_0);
time_embed and each block's mlp are nn.Sequential, whose members flax names layers_{index} (the Fourier embedding,
layers_0 of time_embed, and the gelu, layers_1 of mlp, hold no parameters); TimeProjection's two DenseGeneral are
DenseGeneral_0/1; DiTBlock names ada_params_module, attention (to_q / to_k / to_v / to_out_0, NormalAttention with
biases) and AdaLNParams its Dense ada_proj.  No SimpleDiT checkpoint exists in the reference tree, so the names below
are derived from flax's naming rules, not pinned against a file flax wrote."""
import numpy as np
import pytest
import torch

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.simple_dit import SimpleDiT, sincos_2d_table
from oracle import dit_ref


def _names(F, h, p, E, layers, out=3, ctx=None, sigma=False):
    d = F // h
    n = p * p * out * (2 if sigma else 1)
    want = {"patch_embed/Conv_0/kernel": (p, p, 3, F), "patch_embed/Conv_0/bias": (F,),
            "time_embed/layers_1/DenseGeneral_0/kernel": (F, E), "time_embed/layers_1/DenseGeneral_0/bias": (E,),
            "time_embed/layers_1/DenseGeneral_1/kernel": (E, E), "time_embed/layers_1/DenseGeneral_1/bias": (E,),
            "time_embed/layers_2/kernel": (E, F), "time_embed/layers_2/bias": (F,),
            "final_norm/scale": (F,), "final_norm/bias": (F,), "final_proj/kernel": (F, n), "final_proj/bias": (n,)}
    if ctx:
        want.update({"text_context_proj/kernel": (ctx, F), "text_context_proj/bias": (F,)})
    for i in range(layers):
        b = f"dit_block_{i}"
        want[f"{b}/ada_params_module/ada_proj/kernel"] = (F, 6 * F)
        want[f"{b}/ada_params_module/ada_proj/bias"] = (6 * F,)
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


@pytest.mark.parametrize("kw,F,h,p,E,layers,ctx,sigma", [
    (dict(patch_size=2, emb_features=64, num_layers=2, num_heads=2), 64, 2, 2, 256, 2, None, False),
    (dict(patch_size=2, emb_features=128, num_layers=1, num_heads=4, context_dim=768, learn_sigma=True),
     128, 4, 2, 512, 1, 768, True),
    (dict(patch_size=4, emb_features=768, num_layers=12, num_heads=12), 768, 12, 4, 3072, 12, None, False),  # DiT-B/4
])
def test_parameter_names_and_shapes(kw, F, h, p, E, layers, ctx, sigma):
    m = SimpleDiT(**kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(F, h, p, E, layers, ctx=ctx, sigma=sigma)


@pytest.mark.parametrize("kw,match", [
    (dict(use_hilbert=True), "Hilbert"),
    (dict(use_zigzag=True), "zigzag"),
    (dict(use_flash_attention=True), "flash"),
    (dict(dtype=torch.float32), "dtype"),
    (dict(dtype=torch.float16), "dtype"),
    (dict(emb_features=768, num_heads=10), "multiple of num_heads"),
    (dict(emb_features=192, num_heads=64), "odd"),
    (dict(emb_features=512, num_heads=1), "> 256"),
])
def test_constructor_refusals(kw, match):
    with pytest.raises(FdxError, match=match):
        SimpleDiT(**kw)


def test_image_not_divisible_by_patch_is_refused():
    m = SimpleDiT(patch_size=4, emb_features=64, num_layers=1, num_heads=2)
    with pytest.raises(FdxError, match="divisible"):
        m.forward(None, torch.zeros(1, 18, 16, 3), torch.zeros(1))


def test_norm_groups_and_activation_are_accepted_and_ignored():
    a = SimpleDiT(emb_features=64, num_heads=2, num_layers=1, norm_groups=8, activation=torch.nn.functional.silu)
    b = SimpleDiT(emb_features=64, num_heads=2, num_layers=1)
    assert a.param_specs() == b.param_specs()


def test_config_round_trip():
    m = SimpleDiT(patch_size=4, emb_features=192, num_layers=3, num_heads=3, mlp_ratio=2, learn_sigma=True,
                  context_dim=64)
    m2 = SimpleDiT(**m.config())
    assert m2.config() == m.config() and m2.param_specs() == m.param_specs()


def test_rope_at_position_zero_is_identity():
    x = torch.randn(2, 5, 3, 16)
    y = dit_ref.rope(x)
    assert torch.equal(y[:, 0], x[:, 0])
    assert not torch.allclose(y[:, 1:], x[:, 1:])


def test_sincos_table_quarters():
    F, HP, WP = 32, 3, 5
    tab = dit_ref.sincos_2d(F, HP, WP).reshape(HP, WP, F)
    q = F // 4
    om = 1.0 / 10000.0 ** (np.arange(q) / q)
    r, c = np.meshgrid(np.arange(HP), np.arange(WP), indexing="ij")
    np.testing.assert_allclose(tab[..., :q], np.sin(r[..., None] * om), atol=1e-6)
    np.testing.assert_allclose(tab[..., q:2 * q], np.cos(r[..., None] * om), atol=1e-6)
    np.testing.assert_allclose(tab[..., 2 * q:3 * q], np.sin(c[..., None] * om), atol=1e-6)
    np.testing.assert_allclose(tab[..., 3 * q:], np.cos(c[..., None] * om), atol=1e-6)
    assert np.array_equal(sincos_2d_table(F, HP, WP), dit_ref.sincos_2d(F, HP, WP))


def test_zero_initialised_ada_and_final_proj_give_zero_output():
    """ada_proj and final_proj are zero-initialised: every block is the identity and the output is final_proj's zero
    bias, whatever the input."""
    torch.manual_seed(0)
    F, h, p, layers = 64, 2, 2, 2
    P = {}
    for name, shape in _names(F, h, p, 4 * F, layers).items():
        zero = "ada_proj" in name or name.startswith("final_proj") or name.endswith("bias")
        P[name] = torch.zeros(shape) if zero else torch.randn(shape) * 0.1
    P["final_norm/scale"] = torch.ones(F)
    out = dit_ref.simple_dit_forward(P, torch.randn(2, 8, 8, 3), torch.rand(2), torch.randn(F // 2), patch_size=p,
                                     num_layers=layers, num_heads=h)
    assert out.shape == (2, 8, 8, 3) and out.abs().max().item() == 0
