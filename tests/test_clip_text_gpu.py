"""The CLIP text tower on the engine: its kernels element by element against float64 (tests/clip_text_ref.py, the
tolerance model of tests/elementwise_ref.py), the whole tower against transformers' CLIPTextModel, and the
text-conditioned training step that encodes its tokens inside the captured graph."""
import math

import pytest
import torch

from clip_text_ref import (Tok, attention_masked_ref, bias_act_ref, clip_model, layernorm_ref, rel_l2_per_sequence,
                           token_batch, token_embed_ref)
from elementwise_ref import assert_elementwise, bf16_bound
from flaxdiff_b200 import ops
from flaxdiff_b200._lib import ACT_GELU, ACT_QUICK_GELU, FdxError

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def _bf16(shape, std=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * std).to(torch.bfloat16).to(dev)


# ----------------------------------------------------------------------------------------------- kernels
def test_token_embed_elementwise_nan_rows_and_sentinels():
    B, T, D, vocab = 3, 77, 768, 1000
    g = torch.Generator().manual_seed(1)
    tok = torch.randn(vocab, D, generator=g).to(dev)
    pos = torch.randn(T, D, generator=g).to(dev) * 0.1
    ids = torch.randint(0, vocab, (B, T), generator=g, dtype=torch.int32)
    ids[0, 5], ids[1, 0], ids[2, 76], ids[2, 40] = -1, vocab, 2 ** 31 - 1, -2 ** 31
    sentinel = 3.0
    buf = torch.full((B * T * D + 2 * 64,), sentinel, dtype=torch.bfloat16, device=dev)
    out = buf[64:64 + B * T * D].view(B, T, D)
    ops.token_embed(ids.to(dev), tok, pos, out=out)
    ref, delta = token_embed_ref(ids.to(dev).long(), tok.double(), pos.double())
    bad = ~((ids >= 0) & (ids < vocab)).to(dev)
    assert torch.isnan(out[bad].float()).all()
    assert_elementwise(out[~bad], ref[~bad], bf16_bound(ref[~bad], delta[~bad]), "token_embed")
    assert torch.equal(buf[:64], torch.full_like(buf[:64], sentinel))
    assert torch.equal(buf[-64:], torch.full_like(buf[-64:], sentinel))


@pytest.mark.parametrize("C", [512, 768, 1024, 1280])
def test_layernorm_elementwise(C):
    rows = 1003                                          # not a multiple of the 8 rows of a block
    x = _bf16((rows, C), 2.0, seed=C) + 0.5
    gen = torch.Generator().manual_seed(C + 1)
    g = (1 + 0.5 * torch.randn(C, generator=gen)).to(dev)
    b = (0.3 * torch.randn(C, generator=gen)).to(dev)
    y = ops.layernorm_fwd(x, g, b, 1e-5)
    ref, delta = layernorm_ref(x.double(), g.double(), b.double(), 1e-5)
    assert_elementwise(y, ref, bf16_bound(ref, delta), f"layernorm C={C}")


@pytest.mark.parametrize("act", [ACT_QUICK_GELU, ACT_GELU])
@pytest.mark.parametrize("with_bias", [True, False])
def test_bias_act_elementwise(act, with_bias):
    rows, C = 333, 3072
    x = _bf16((rows, C), 3.0, seed=act)
    bias = (torch.randn(C, generator=torch.Generator().manual_seed(7))).to(dev) if with_bias else None
    y = ops.bias_act(x, bias, act)
    ref, delta = bias_act_ref(x.double(), None if bias is None else bias.double(), act)
    assert_elementwise(y, ref, bf16_bound(ref, delta), f"bias_act act={act} bias={with_bias}")
    ops.bias_act(x, bias, act, out=x)                    # in place, as the tower runs it
    assert torch.equal(x, y)


def _key_mask(kind, B, Lk, seed=0):
    if kind is None:
        return None
    g = torch.Generator().manual_seed(seed)
    if kind == "prefix":
        n = torch.randint(1, Lk + 1, (B,), generator=g)
        m = (torch.arange(Lk).view(1, -1) < n.view(-1, 1)).to(torch.int32)
    else:
        m = (torch.rand(B, Lk, generator=g) < 0.6).to(torch.int32)
        m[0, :min(3, Lk)] = 0                            # causal rows 0..2 of image 0 have no allowed key
    if B > 1:
        m[B - 1] = 0                                     # an image with no allowed key at all
    return m.contiguous().to(dev)


def _check_masked(B, L, heads, dh, causal, kind, seed=0):
    HD = heads * dh
    qkv = _bf16((B, L, 3 * HD), 1.0, seed=seed)          # q, k, v: strided views with ld = 3 HD, as in the tower
    q, k, v = qkv[:, :, :HD], qkv[:, :, HD:2 * HD], qkv[:, :, 2 * HD:]
    mask = _key_mask(kind, B, L, seed)
    scale = 1.0 / math.sqrt(dh)
    o = ops.attention_fwd_masked(q, k, v, heads, dh, scale, causal, mask)
    ref, delta = attention_masked_ref(q.double(), k.double(), v.double(), heads, dh, scale, causal, mask)
    assert_elementwise(o, ref, bf16_bound(ref, delta), f"masked attention L={L} h={heads} dh={dh} {causal} {kind}")
    if mask is not None and B > 1:
        assert not o[B - 1].any()                        # rows with no allowed key are zeros


@pytest.mark.parametrize("L", [1, 77, 128, 129])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("kind", [None, "prefix", "arbitrary"])
def test_masked_attention_elementwise(L, causal, kind):
    _check_masked(3, L, 12, 64, causal, kind, seed=L)


@pytest.mark.parametrize("heads,dh", [(8, 64), (16, 64), (8, 32)])
@pytest.mark.parametrize("L", [77, 129])
def test_masked_attention_head_widths(heads, dh, L):
    _check_masked(2, L, heads, dh, True, "arbitrary", seed=heads + dh)


def test_masked_attention_refuses_head_width_128():
    q = _bf16((1, 77, 128))
    with pytest.raises(FdxError, match="status -2"):
        ops.attention_fwd_masked(q, q, q, 1, 128, 128 ** -0.5, True)


def test_unmasked_rows_match_fdx_attention_fwd():
    """No key mask and no causal mask: the masked kernel computes what fdx_attention_fwd computes, bit for bit."""
    for L, dh in ((77, 64), (200, 64), (77, 32)):
        q, k, v = (_bf16((2, L, 8 * dh), seed=i) for i in range(3))
        o_ref, _ = ops.attention_fwd(q, k, v, 8, dh, dh ** -0.5)
        assert torch.equal(ops.attention_fwd_masked(q, k, v, 8, dh, dh ** -0.5, False), o_ref)


# ----------------------------------------------------------------------------------------------- the tower
def _tower(kind):
    from flaxdiff_b200.models.clip_text import CLIPTextTower
    model = clip_model(kind)
    return model, CLIPTextTower.from_transformers(model, dev)


@pytest.mark.parametrize("kind", ["tiny", "clip-l", "openclip"])
def test_tower_matches_transformers(kind):
    """All 77 positions (the padding positions feed cross-attention): the per-sequence relative L2 error against
    transformers in fp32 is at most 1.25x that of the same model run in bf16 on the CPU."""
    model, tower = _tower(kind)
    ids, mask = token_batch(model.config.vocab_size, [5, 75, 0, 17, 40], seed=3)
    got = tower.encode(ids.to(dev), mask.to(dev))
    assert got.dtype == torch.bfloat16 and got.shape == (5, 77, model.config.hidden_size)
    with torch.no_grad():
        ref = model(input_ids=ids, attention_mask=mask).last_hidden_state
        m16 = clip_model(kind).to(torch.bfloat16)
        ref16 = m16(input_ids=ids, attention_mask=mask).last_hidden_state
    e_fdx, e_bf16 = rel_l2_per_sequence(got, ref), rel_l2_per_sequence(ref16, ref)
    print(f"{kind}: engine {['%.3e' % e for e in e_fdx]}  transformers bf16 {['%.3e' % e for e in e_bf16]}")
    for s, (a, b) in enumerate(zip(e_fdx, e_bf16)):
        assert a <= 1.25 * b, (kind, s, a, b)


def test_tower_is_bit_reproducible_across_batch_compositions():
    model, tower = _tower("clip-l")
    ids, mask = token_batch(model.config.vocab_size, [int(n) for n in torch.arange(256) % 76], seed=5)
    ids, mask = ids.to(dev), mask.to(dev)
    full = tower.encode(ids, mask)
    assert torch.equal(full, tower.encode(ids, mask))
    for r in (0, 75, 200):
        assert torch.equal(tower.encode(ids[r:r + 1], mask[r:r + 1])[0], full[r])
    perm = torch.randperm(256, generator=torch.Generator().manual_seed(0)).to(dev)
    assert torch.equal(tower.encode(ids[perm], mask[perm]), full[perm])


def test_encoder_backend_fdx_and_registry_roundtrip(monkeypatch):
    import transformers

    from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig
    model = clip_model("tiny")
    enc = CLIPTextEncoder(model, Tok(1000), modelname="tiny-random", backend="fdx")
    out = enc(["a photo of a cat", "", "a painting of a dog"])
    assert out.is_cuda and out.dtype == torch.bfloat16 and out.shape == (3, 77, 64)
    tokens = enc.tokenize(["a photo of a cat", "", "a painting of a dog"])
    with torch.no_grad():
        ref = model(**tokens).last_hidden_state
    assert max(rel_l2_per_sequence(out, ref)) < 2e-2
    assert enc.serialize() == {"modelname": "tiny-random", "backend": "fdx"}
    monkeypatch.setattr(transformers.CLIPTextModel, "from_pretrained", staticmethod(lambda *a, **k: clip_model("tiny")))
    monkeypatch.setattr(transformers.AutoTokenizer, "from_pretrained", staticmethod(lambda *a, **k: Tok(1000)))
    cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", unconditional_input="")
    back = ConditionalInputConfig.deserialize(cond.serialize())
    assert back.encoder.backend == "fdx" and back.encoder.tower is not None
    assert torch.equal(back.get_unconditional(), cond.get_unconditional())
    assert torch.equal(back.encoder(["a photo of a cat"]), out[:1])


# ----------------------------------------------------------------------------------------------- the trainer
def _text_trainer(graph):
    from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.schedulers import EDMNoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    enc = CLIPTextEncoder(clip_model("tiny"), Tok(1000), modelname="tiny-random", backend="fdx")
    cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True,
                                  unconditional_input="")
    model = Unet(attention_configs=(None, None, None, {"heads": 8}), dtype=torch.bfloat16)
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (16, 16, 3), [cond]), rngs=4, unconditional_prob=0.5,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 use_cuda_graph=graph)
    return tr, cond


def test_train_step_encodes_tokens_inside_the_graph():
    B = 8
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (B, 16, 16, 3), generator=g, dtype=torch.uint8)
    ids, mask = token_batch(1000, [3, 10, 0, 75, 20, 1, 33, 7], seed=1)
    batch = {"image": images, "text": {"input_ids": ids, "attention_mask": mask}}
    tr_g, cond = _text_trainer(True)
    tr_e, _ = _text_trainer(False)
    step_g, step_e = tr_g._define_train_step(), tr_e._define_train_step()
    tower = cond.encoder.tower
    null = cond.get_unconditional()[0]
    rng_g = rng_e = tr_g.rngstate
    seen = set()
    for _ in range(4):
        _, loss_g, rng_g = step_g(tr_g.state, rng_g, batch)
        _, loss_e, rng_e = step_e(tr_e.state, rng_e, batch)
        ids_s, amask_s, umask = tr_g._static[4]
        sel = umask.view(-1, 1)
        null_ids, null_mask = tr_g._null_tokens
        eager = tower.encode(torch.where(sel, null_ids, ids_s), torch.where(sel, null_mask, amask_s))
        ctx = tr_g._step_ctx
        assert torch.equal(ctx, eager)                   # what the graph fed the UNet, bit for bit
        assert torch.equal(tr_e._step_ctx, eager)        # the eager step runs the same code
        for b in range(B):
            if bool(umask[b]):
                assert torch.equal(ctx[b], null)         # masked samples get exactly get_unconditional()
            else:
                assert not torch.equal(ctx[b], null) or int(mask[b].sum()) == 2
            seen.add(bool(umask[b]))
        lg, le = float(loss_g), float(loss_e)
        assert math.isfinite(lg) and abs(lg - le) <= 2e-3 * abs(le), (lg, le)
    assert seen == {True, False}
