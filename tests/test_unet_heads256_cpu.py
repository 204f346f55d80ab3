"""UNets whose attention heads are 129 - 256 channels wide (the reference's `--attention_heads 2` on the default
feature_depths, 4 heads at 1024 channels): flax's parameter shapes, the stored head width 256, and the refusal of
heads wider than 256."""
import pytest

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.simple_unet import Unet, _attn_width


def test_stored_head_width_256():
    assert all(_attn_width(d) == 256 for d in range(129, 257))
    assert [_attn_width(d) for d in (32, 64, 65, 128)] == [32, 64, 128, 128]
    with pytest.raises(FdxError, match="head width 257 > 256 is not supported"):
        _attn_width(257)


def test_head_width_512_is_refused():
    with pytest.raises(FdxError, match="head width 512 > 256 is not supported"):
        _attn_width(512)


@pytest.mark.parametrize("ctxdim", [None, 768])
def test_two_head_unet_parameter_shapes(ctxdim):
    cfg = {"heads": 2}
    lay = dict(Unet(attention_configs=(None, cfg, cfg, cfg), context_dim=ctxdim).param_specs())
    kv = ctxdim or 512
    for block in ("middle_attention_0", "up_0_attention_1"):
        base = f"{block}/Attention/Attention2"
        assert lay[f"{base}/to_q/kernel"] == (512, 2, 256)
        assert lay[f"{base}/to_k/kernel"] == (kv, 2, 256)
        assert lay[f"{base}/to_v/kernel"] == (kv, 2, 256)
        assert lay[f"{base}/to_out_0/kernel"] == (2, 256, 512)
    # the other attention blocks keep their narrower heads
    for block, shape in (("down_1_attention_1", (64, 2, 32)), ("down_2_attention_1", (128, 2, 64)),
                         ("down_3_attention_1", (256, 2, 128)), ("up_1_attention_1", (256, 2, 128))):
        assert lay[f"{block}/Attention/Attention2/to_q/kernel"] == shape, block


def test_four_head_wide_unet_parameter_shapes():
    cfg = {"heads": 4, "only_pure_attention": False, "use_projection": True}
    lay = dict(Unet(feature_depths=(128, 256, 512, 1024), attention_configs=(None, cfg, cfg, cfg),
                    context_dim=768).param_specs())
    assert lay["middle_attention_0/Attention/Attention1/to_q/kernel"] == (1024, 4, 256)
    assert lay["middle_attention_0/Attention/Attention2/to_k/kernel"] == (768, 4, 256)
    assert lay["down_3_attention_1/Attention/Attention2/to_q/kernel"] == (512, 4, 128)
