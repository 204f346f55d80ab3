"""The README gallery's text-to-image UNet (feature_depths 128 / 256 / 512 / 1024, 8-head attention at the last
three levels) constructs with flax's parameter shapes, and its 128-channel heads are stored 128 wide."""
import math

import pytest

from flaxdiff_b200.models.simple_unet import Unet, _attn_width

DEPTHS = (128, 256, 512, 1024)


@pytest.mark.parametrize("ctxdim", [None, 768])
def test_gallery_unet_parameter_shapes(ctxdim):
    cfg = {"heads": 8}
    m = Unet(feature_depths=DEPTHS, attention_configs=(None, cfg, cfg, cfg), context_dim=ctxdim)
    lay = dict(m.param_specs())
    kv = ctxdim or 1024
    for block in ("middle_attention_0", "up_0_attention_1"):
        base = f"{block}/Attention/Attention2"
        assert lay[f"{base}/to_q/kernel"] == (1024, 8, 128)
        assert lay[f"{base}/to_k/kernel"] == (kv, 8, 128)
        assert lay[f"{base}/to_v/kernel"] == (kv, 8, 128)
        assert lay[f"{base}/to_out_0/kernel"] == (8, 128, 1024)
    # the other attention blocks keep their narrower heads
    for block, shape in (("down_1_attention_1", (128, 8, 16)), ("down_2_attention_1", (256, 8, 32)),
                         ("down_3_attention_1", (512, 8, 64)), ("up_1_attention_1", (512, 8, 64))):
        assert lay[f"{block}/Attention/Attention2/to_q/kernel"] == shape, block
    assert not any(n.startswith("down_0_attention") for n in lay)
    if ctxdim is None:
        assert round(sum(math.prod(s) for s in lay.values()) / 1e6) == 137


def test_full_transformer_block_at_1024_channels_constructs():
    cfg = {"heads": 8, "only_pure_attention": False, "use_projection": True}
    lay = dict(Unet(feature_depths=DEPTHS, attention_configs=(None, None, None, cfg), context_dim=768).param_specs())
    assert lay["middle_attention_0/Attention/Attention1/to_q/kernel"] == (1024, 8, 128)
    assert lay["middle_attention_0/Attention/Attention2/to_k/kernel"] == (768, 8, 128)


def test_stored_head_widths(monkeypatch):
    assert [_attn_width(d) for d in (8, 16, 32, 48, 64, 65, 80, 96, 128)] == [32, 32, 32, 64, 64, 128, 128, 128, 128]
    monkeypatch.setenv("FDX_ATTN_PAD64", "1")
    assert [_attn_width(d) for d in (16, 32, 64, 96, 128)] == [64, 64, 64, 128, 128]
