"""The mish activation without a GPU: the oracle's mish and its autograd derivative against known float64 values
(including z = +-100, where the kernels clamp), the Unet's acceptance of mish, and the configuration round trip
of a mish model."""
import pytest
import torch
import torch.nn.functional as F

from flaxdiff_b200 import ops, utils
from flaxdiff_b200.models.simple_unet import FdxError, Unet
from mish_ref import mish as oracle_mish
from mish_ref import mish_oracle
from oracle import unet_ref

KNOWN = [  # (z, mish(z)) and (z, mish'(z)), float64, from z tanh(log1p(e^z)) and its derivative
    (1.0, 0.8650983882673103), (-1.0, -0.30340146137410895), (3.0, 2.9865350049679575)]
KNOWN_GRAD = [(0.5, 0.8864243753577272), (4.0, 1.00443287690375)]


def test_oracle_mish_known_values():
    for z, want in KNOWN:
        got = oracle_mish(torch.tensor(z, dtype=torch.float64)).item()
        assert abs(got - want) <= 1e-15 * max(1.0, abs(want)), (z, got, want)
    for z, want in KNOWN_GRAD:
        t = torch.tensor(z, dtype=torch.float64, requires_grad=True)
        (g,) = torch.autograd.grad(oracle_mish(t), t)
        assert abs(g.item() - want) <= 1e-14, (z, g.item(), want)


def test_oracle_mish_clamp_regions():
    """Where the kernels clamp: mish(z) = z and mish'(z) = 1 for large z, mish -> 0- and mish' -> 0 for very
    negative z, all finite."""
    z = torch.tensor([100.0, -100.0], dtype=torch.float64, requires_grad=True)
    y = oracle_mish(z)
    (g,) = torch.autograd.grad(y.sum(), z)
    assert torch.isfinite(y).all() and torch.isfinite(g).all()
    assert y[0].item() == 100.0 and g[0].item() == 1.0
    assert -1e-40 < y[1].item() < 0.0 and abs(g[1].item()) < 1e-40
    # the same function as torch's (which is not used on the hot path)
    zz = torch.linspace(-30, 30, 601, dtype=torch.float64)
    assert torch.allclose(oracle_mish(zz), F.mish(zz), rtol=1e-14, atol=1e-300)


def mish(x):        # a user-defined function named like jax.nn.mish
    return x * torch.tanh(F.softplus(x))


@pytest.mark.parametrize("activation", ["mish", F.mish, mish], ids=["name", "torch", "named-function"])
def test_unet_accepts_mish_with_the_swish_parameter_tree(activation):
    m = Unet(attention_configs=(None,) * 4, activation=activation)
    s = Unet(attention_configs=(None,) * 4)
    assert m._act == ops.ACT_MISH and s._act == ops.ACT_SILU
    assert m.param_specs() == s.param_specs()


def test_unet_still_refuses_relu():
    with pytest.raises(FdxError, match="activation"):
        Unet(attention_configs=(None,) * 4, activation="relu")


def test_mish_config_round_trip():
    """map_nested_config drops tuple-valued fields as the reference does, so the model keeps its defaults there."""
    model = Unet(activation="mish")
    cfg = utils.map_nested_config(utils.serialize_model(model))
    assert cfg["activation"] == "mish"
    again = Unet(**cfg)
    assert again._act == ops.ACT_MISH and again.param_specs() == model.param_specs()
    # the function object serialises by name as well
    cfg2 = utils.map_nested_config(utils.serialize_model(Unet(activation=F.mish)))
    assert Unet(**cfg2)._act == ops.ACT_MISH


def test_activation_map_holds_the_reference_keys():
    for key in ("swish", "silu", "jax._src.nn.functions.silu"):
        assert utils.ACTIVATION_MAP[key] == "swish"
        assert utils.map_nested_config({"activation": key}) == {"activation": "swish"}
    assert utils.ACTIVATION_MAP["mish"] == "mish"


def test_activation_codes():
    assert [ops._act_code(a) for a in (False, True, ops.ACT_MISH)] == [0, 1, 2]
    with pytest.raises(ValueError):
        ops._act_code(3)


def test_mish_oracle_swaps_the_activation_of_the_residual_block():
    """mish_oracle() makes the oracle's ResidualBlock apply mish after both norms, and restores swish afterwards."""
    g = torch.Generator().manual_seed(0)
    C, E, name = 16, 8, "blk"
    P = {f"{name}/norm1/scale": 1 + 0.1 * torch.randn(C, generator=g), f"{name}/norm1/bias": torch.randn(C, generator=g),
         f"{name}/norm2/scale": 1 + 0.1 * torch.randn(C, generator=g), f"{name}/norm2/bias": torch.randn(C, generator=g),
         f"{name}/conv1/conv/kernel": 0.1 * torch.randn(3, 3, C, C, generator=g),
         f"{name}/conv1/conv/bias": 0.1 * torch.randn(C, generator=g),
         f"{name}/conv2/conv/kernel": 0.1 * torch.randn(3, 3, C, C, generator=g),
         f"{name}/conv2/conv/bias": 0.1 * torch.randn(C, generator=g),
         f"{name}/temb_projection/kernel": 0.1 * torch.randn(E, C, generator=g),
         f"{name}/temb_projection/bias": 0.1 * torch.randn(C, generator=g)}
    x, temb = torch.randn(2, 8, 8, C, generator=g), torch.randn(2, E, generator=g)

    def by_hand(act):
        h = act(unet_ref.group_norm(x, P[f"{name}/norm1/scale"], P[f"{name}/norm1/bias"], 8, 1e-4))
        h = unet_ref.conv_same(h, P[f"{name}/conv1/conv/kernel"], P[f"{name}/conv1/conv/bias"])
        h = h + (temb @ P[f"{name}/temb_projection/kernel"] + P[f"{name}/temb_projection/bias"])[:, None, None, :]
        h = act(unet_ref.group_norm(h, P[f"{name}/norm2/scale"], P[f"{name}/norm2/bias"], 8, 1e-4))
        return unet_ref.conv_same(h, P[f"{name}/conv2/conv/kernel"], P[f"{name}/conv2/conv/bias"]) + x

    with mish_oracle():
        got = unet_ref.residual_block(P, name, x, temb, 8)
    assert torch.allclose(got, by_hand(oracle_mish), atol=1e-5)
    assert not torch.allclose(got, by_hand(unet_ref.swish), atol=1e-3)
    assert torch.allclose(unet_ref.residual_block(P, name, x, temb, 8), by_hand(unet_ref.swish), atol=1e-5)
