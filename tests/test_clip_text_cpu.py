"""The engine's CLIP text tower without a GPU: the configurations its kernels cannot run are refused at
construction, CLIPTextEncoder(backend="fdx") serialises as such and fails offline like the torch backend, and the
weights are packed in the layout the kernels read."""
import pytest
import torch

from clip_text_ref import Tok, clip_model
from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.inputs import CLIPTextEncoder
from flaxdiff_b200.models.clip_text import CLIPTextTower


def _cfg(**kw):
    from transformers import CLIPTextConfig
    base = dict(vocab_size=1000, hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2,
                max_position_embeddings=77)
    base.update(kw)
    return CLIPTextConfig(**base)


@pytest.mark.parametrize("kw,seq_len,match", [
    (dict(hidden_act="gelu_new"), None, "hidden_act"),
    (dict(hidden_act="relu"), None, "hidden_act"),
    (dict(num_attention_heads=8), None, "head width 8 "),
    (dict(hidden_size=96, num_attention_heads=3), None, "multiple of 64"),
    (dict(hidden_size=1344, num_attention_heads=21), None, "multiple of 64, <= 1280"),
    (dict(intermediate_size=100), None, "intermediate_size"),
    (dict(), 78, "exceeds max_position_embeddings"),
    (dict(max_position_embeddings=16), 77, "exceeds max_position_embeddings"),
])
def test_tower_refuses_configs_outside_the_kernels(kw, seq_len, match):
    with pytest.raises(FdxError, match=match):
        CLIPTextTower(_cfg(**kw), {}, device="cpu", seq_len=seq_len)


def test_tower_accepts_head_widths_32_and_64_and_packs_the_kernel_layout():
    from transformers import CLIPTextModel
    torch.manual_seed(0)
    model = CLIPTextModel(_cfg(num_attention_heads=4))   # test_text_encoder_cpu.py's tiny tower: 4 heads of 16
    with pytest.raises(FdxError, match="head width 16"):
        CLIPTextTower.from_transformers(model, device="cpu")
    torch.manual_seed(0)
    model = CLIPTextModel(_cfg(num_attention_heads=2, num_hidden_layers=2))
    t = CLIPTextTower.from_transformers(model, device="cpu")
    assert (t.dh, t.layers, t.seq_len) == (32, 2, 77)
    sd = model.state_dict()
    p = "text_model.encoder.layers.1."
    wqkv = t.w["1.wqkv"]
    assert wqkv.dtype == torch.bfloat16 and wqkv.shape == (64, 192) and wqkv.is_contiguous()
    assert torch.equal(wqkv[:, 64:128], sd[p + "self_attn.k_proj.weight"].t().to(torch.bfloat16))
    assert torch.equal(t.w["1.bqkv"][128:], sd[p + "self_attn.v_proj.bias"])
    assert torch.equal(t.w["1.w1"], sd[p + "mlp.fc1.weight"].t().to(torch.bfloat16))
    assert t.w["tok"].dtype == torch.float32 and torch.equal(t.w["tok"], sd["text_model.embeddings.token_embedding.weight"])
    assert all(v.untyped_storage().data_ptr() == t.buffer.untyped_storage().data_ptr() for v in t.w.values())
    assert all((v.data_ptr() - t.buffer.data_ptr()) % 256 == 0 for v in t.w.values())


def test_encoder_backend_fdx_serialises_and_fails_offline_like_torch():
    from transformers import CLIPTextModel
    torch.manual_seed(0)
    enc = CLIPTextEncoder(CLIPTextModel(_cfg(num_attention_heads=2)), Tok(1000), modelname="tiny-random",
                          backend="fdx", device="cpu")
    assert enc.serialize() == {"modelname": "tiny-random", "backend": "fdx"}
    with pytest.raises(FdxError, match="local Hugging Face cache"):
        CLIPTextEncoder.deserialize(enc.serialize())
    with pytest.raises(FdxError, match="local Hugging Face cache"):
        CLIPTextEncoder.from_modelname("openai/clip-vit-large-patch14", backend="fdx")
    with pytest.raises(FdxError, match="only the torch backend"):
        CLIPTextEncoder.from_modelname(backend="jax")
    assert CLIPTextEncoder(clip_model("tiny"), Tok(1000)).tower is None          # the default stays torch
