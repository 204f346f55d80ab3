"""The CLIP metrics on the engine: the image preprocessing bit for bit against CLIPImageProcessorPil, the embedding,
pooling and cosine kernels element by element against float64 (tests/clip_metric_ref.py, the tolerance model of
tests/elementwise_ref.py), both towers' projected embeddings against transformers, both metrics end to end against a
torch restatement of flaxdiff/metrics/images.py, and a text-conditioned fit that tracks them."""
import copy
import math

import numpy as np
import pytest
import torch

from clip_metric_ref import (clip_pair_model, metric_ref, patchify, pool_rows, processor_u8, quantise_np, save_tiny,
                             similarity_ref, vision_embed_ref)
from clip_text_ref import Tok, layernorm_ref, rel_l2_per_sequence, token_batch
from elementwise_ref import assert_elementwise, bf16_bound, f32_bound, ulp_bf16
from flaxdiff_b200 import ops
from flaxdiff_b200.models.clip_vision import CLIPPair

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
SIZES = [(16, 16), (28, 28), (32, 32), (64, 64), (96, 128), (128, 128), (224, 224), (256, 256), (300, 300),
         (512, 512)]


def _processor():
    from transformers.models.clip import CLIPImageProcessorPil
    return CLIPImageProcessorPil()


_PAIRS = {}


def _pair(kind):
    if kind not in _PAIRS:
        model = clip_pair_model(kind)
        _PAIRS[kind] = (model, CLIPPair.from_transformers(model, _processor(), dev))
    return _PAIRS[kind]


def _samples(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, H, W, 3, generator=g) * 2 - 1


# ----------------------------------------------------------------------------------------------- preprocessing
@pytest.mark.parametrize("H,W", SIZES)
def test_image_prep_matches_clip_image_processor_pil(H, W):
    _, pair = _pair("tiny")
    x = _samples(2, H, W, H * 7 + W)
    u8 = torch.zeros((2, 224, 224, 3), dtype=torch.uint8, device=dev)
    patches = pair.preprocess(x.to(dev), u8_out=u8)
    q = quantise_np(x.numpy())
    pv = _processor()(images=list(q), return_tensors="pt")["pixel_values"]            # [2, 3, 224, 224] f32
    for b in range(2):
        assert np.array_equal(u8[b].cpu().numpy(), processor_u8(q[b])), (H, W, b)
    lut = pair.w["lut"].cpu()
    assert torch.equal(lut[torch.arange(3).view(1, 1, 1, 3), u8.cpu().long()].permute(0, 3, 1, 2), pv)
    ref = patchify(pv, 14)
    assert patches.shape == (2 * 256, 592) and not patches[:, 588:].any()
    err = (patches[:, :588].float().cpu() - ref).abs()
    assert (err <= ulp_bf16(ref).float()).all(), float(err.max())


def test_image_prep_clamps_out_of_range_values_and_nan():
    _, pair = _pair("tiny")
    special = torch.tensor([2.0, -2.0, math.inf, -math.inf, math.nan, 1.0, -1.0, 0.0])
    for H in (224, 64):                                   # no resize pass, and an upscale
        x = _samples(2, H, H, H)
        idx = torch.randint(0, x.numel(), (4000,), generator=torch.Generator().manual_seed(H))
        x.view(-1)[idx] = special[torch.arange(4000) % 8]
        u8 = torch.zeros((2, 224, 224, 3), dtype=torch.uint8, device=dev)
        pair.preprocess(x.to(dev), u8_out=u8)
        q = quantise_np(x.numpy())
        for b in range(2):
            assert np.array_equal(u8[b].cpu().numpy(), processor_u8(q[b]))
    assert quantise_np(special.numpy()).tolist() == [255, 0, 255, 0, 0, 255, 0, 127]


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("D", [128, 768, 1024, 1280])
def test_vision_embed_elementwise(D):
    B, G2 = 3, 256
    g = torch.Generator().manual_seed(D)
    patch = (torch.randn(B * G2, D, generator=g) * 2).to(dev)
    cls, pos = torch.randn(D, generator=g).to(dev), (torch.randn(G2 + 1, D, generator=g) * 0.5).to(dev)
    gm, bt = (1 + 0.5 * torch.randn(D, generator=g)).to(dev), (0.3 * torch.randn(D, generator=g)).to(dev)
    y = ops.clip_vision_embed(patch, B, cls, pos, gm, bt, 1e-5)
    ref, delta = vision_embed_ref(patch.double(), cls.double(), pos.double(), gm.double(), bt.double(), 1e-5)
    assert_elementwise(y, ref, bf16_bound(ref, delta), f"vision_embed D={D}")


@pytest.mark.parametrize("with_ids", [False, True])
@pytest.mark.parametrize("with_ln", [False, True])
@pytest.mark.parametrize("T,D", [(257, 1024), (77, 768), (50, 1280)])
def test_pool_elementwise(with_ids, with_ln, T, D):
    B = 37
    g = torch.Generator().manual_seed(T + D)
    x = (torch.randn(B, T, D, generator=g) * 2 + 0.5).to(torch.bfloat16).to(dev)
    ids = None
    if with_ids:
        ids = torch.randint(0, 1000, (B, T), generator=g, dtype=torch.int32)
        ids[0] = 7                                        # all equal: the first position
        ids[1, 3] = ids[1, T - 5] = 5000                  # a tie: the first of the two
        ids[2, T - 1] = 2 ** 31 - 1
        ids[3] = -5
        ids = ids.to(dev)
    gm = (1 + 0.5 * torch.randn(D, generator=g)).to(dev) if with_ln else None
    bt = (0.3 * torch.randn(D, generator=g)).to(dev) if with_ln else None
    out = ops.clip_pool(x, ids, gm, bt, 1e-5)
    rows = pool_rows(ids, B)
    if with_ids:
        assert rows[0] == 0 and rows[1] == 3 and rows[2] == T - 1 and rows[3] == 0
    sel = x[torch.arange(B), rows.to(dev)]
    if not with_ln:
        assert torch.equal(out, sel)
        return
    ref, delta = layernorm_ref(sel.double(), gm.double(), bt.double(), 1e-5)
    assert_elementwise(out, ref, bf16_bound(ref, delta), f"pool T={T} D={D} ids={with_ids}")


@pytest.mark.parametrize("B,P", [(1, 768), (5, 512), (256, 768), (1000, 64)])
def test_similarity_elementwise(B, P):
    g = torch.Generator().manual_seed(B + P)
    img = torch.randn(B, P, generator=g) * 3
    txt = 0.5 * img + torch.randn(B, P, generator=g)           # cosines spread over both signs
    txt[0] = -img[0]
    cos, out2 = ops.clip_similarity(img.to(dev), txt.to(dev))
    rc, r2, dc, d2 = similarity_ref(img.double(), txt.double())
    assert_elementwise(cos, rc, f32_bound(rc, dc), f"cos B={B} P={P}")
    assert_elementwise(out2, r2, f32_bound(r2, d2), f"clip metrics B={B} P={P}")


# ----------------------------------------------------------------------------------------------- the towers
def _ref_embeds(model, pv, ids, mask, dtype):
    """CLIPVisionModelWithProjection's / CLIPTextModelWithProjection's embeddings, the model run on the GPU."""
    m = copy.deepcopy(model).to(dev, dtype)
    with torch.no_grad():
        img = m.visual_projection(m.vision_model(pixel_values=pv.to(dev, dtype)).pooler_output)
        txt = m.text_projection(m.text_model(input_ids=ids.to(dev), attention_mask=mask.to(dev)).pooler_output)
    return img.float(), txt.float()


@pytest.mark.parametrize("kind", ["tiny", "vit-l"])
def test_embeds_match_transformers(kind):
    """Per-sample relative L2 error of image_embeds and text_embeds against transformers in fp32 is at most 1.25x
    that of the same model run in bf16."""
    model, pair = _pair(kind)
    x = _samples(4, 64, 96, 11)
    pv = _processor()(images=list(quantise_np(x.numpy())), return_tensors="pt")["pixel_values"]
    ids, mask = token_batch(model.config.text_config.vocab_size, [5, 75, 0, 17], seed=3)
    img, txt = pair.image_embeds(x.to(dev)), pair.text_embeds(ids.to(dev), mask.to(dev))
    assert img.dtype == txt.dtype == torch.float32 and img.shape == txt.shape == (4, model.config.projection_dim)
    ref_i, ref_t = _ref_embeds(model, pv, ids, mask, torch.float32)
    b16_i, b16_t = _ref_embeds(model, pv, ids, mask, torch.bfloat16)
    for what, got, ref, b16 in (("image", img, ref_i, b16_i), ("text", txt, ref_t, b16_t)):
        e_fdx, e_bf16 = rel_l2_per_sequence(got, ref), rel_l2_per_sequence(b16, ref)
        print(f"{kind} {what}: engine {['%.3e' % e for e in e_fdx]}  transformers bf16 {['%.3e' % e for e in e_bf16]}")
        for s, (a, b) in enumerate(zip(e_fdx, e_bf16)):
            assert a <= 1.25 * b, (kind, what, s, a, b)


def test_embeds_are_bit_reproducible_across_batch_compositions():
    model, pair = _pair("tiny")
    B = 12
    x = _samples(B, 64, 64, 5).to(dev)
    ids, mask = token_batch(1000, [int(n) for n in torch.arange(B) * 6 % 76], seed=5)
    ids, mask = ids.to(dev), mask.to(dev)
    cos, out2 = pair.similarity(x, ids, mask)
    img, txt = pair.image_embeds(x), pair.text_embeds(ids, mask)
    assert torch.equal(pair.similarity(x, ids, mask)[1], out2)
    for r in (0, 5, 11):
        assert torch.equal(pair.image_embeds(x[r:r + 1])[0], img[r])
        assert torch.equal(pair.text_embeds(ids[r:r + 1], mask[r:r + 1])[0], txt[r])
        assert torch.equal(pair.similarity(x[r:r + 1], ids[r:r + 1], mask[r:r + 1])[0][0], cos[r])
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(0)).to(dev)
    assert torch.equal(pair.similarity(x[perm], ids[perm], mask[perm])[0], cos[perm])


# ----------------------------------------------------------------------------------------------- the metrics
@pytest.fixture(scope="module")
def tiny_dir(tmp_path_factory):
    return save_tiny(tmp_path_factory.mktemp("clip-tiny"))


@pytest.mark.parametrize("res", [64, 128, 256])
def test_metrics_end_to_end_against_torch_restatement(tiny_dir, res):
    """Both metrics against images.py:32-112 in torch fp32 (CLIPImageProcessorPil + CLIPModel + the formula), within
    1.25x the cosine error of the same CLIPModel in bf16 (and 1e-3)."""
    from transformers import CLIPModel
    from transformers.models.clip import CLIPImageProcessorPil

    from flaxdiff_b200.metrics import get_clip_metric, get_clip_score_metric
    sim, score = get_clip_metric(tiny_dir), get_clip_score_metric(tiny_dir)
    B = 6
    x = _samples(B, res, res, res).numpy()
    ids, mask = token_batch(1000, [3, 10, 0, 75, 20, 33], seed=res)
    batch = {"text": {"input_ids": ids.numpy(), "attention_mask": mask.numpy()}}
    got_sim, got_score = sim.function(x, batch), score.function(torch.from_numpy(x).to(dev), batch)
    assert isinstance(got_sim, float) and isinstance(got_score, float)
    model, proc = CLIPModel.from_pretrained(tiny_dir).eval(), CLIPImageProcessorPil.from_pretrained(tiny_dir)
    ref_sim, ref_score, ref_cos = metric_ref(model, proc, x, ids, mask)
    _, _, b16_cos = metric_ref(model.to(torch.bfloat16), proc, x, ids, mask)
    tol = max(1.25 * float((b16_cos.float() - ref_cos).abs().max()), 1e-3)
    print(f"{res}: clip_similarity {got_sim:.6f} vs {ref_sim:.6f}, clip_score {got_score:.4f} vs {ref_score:.4f}, "
          f"tol {tol:.3e}")
    assert abs(got_sim - ref_sim) <= tol
    assert abs(got_score - ref_score) <= 100 * tol


def test_fit_tracks_clip_similarity_as_minimum_and_clip_score_as_maximum(tiny_dir):
    from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig
    from flaxdiff_b200.metrics import EvaluationMetric, get_clip_metric, get_clip_score_metric
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.samplers import EulerSampler
    from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    from clip_text_ref import clip_model
    enc = CLIPTextEncoder(clip_model("tiny"), Tok(1000), modelname="tiny-random", backend="fdx")
    cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True, unconditional_input="")
    torch.manual_seed(0)
    model = Unet(attention_configs=(None, None, None, {"heads": 8}), dtype=torch.bfloat16)
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (16, 16, 3), [cond]), rngs=4, unconditional_prob=0.5,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev)
    seen = {"clip_similarity": [], "clip_score": []}

    def recorded(m):
        def fn(samples, batch):
            v = m.function(samples, batch)
            seen[m.name].append(v)
            return v
        return EvaluationMetric(function=fn, name=m.name, higher_is_better=m.higher_is_better)

    tr.eval_metrics = [recorded(get_clip_metric(tiny_dir)), recorded(get_clip_score_metric(tiny_dir))]
    B = 4

    def gen(seed):
        def it():
            g = torch.Generator().manual_seed(seed)
            k = 0
            while True:
                ids, mask = token_batch(1000, [3 + k % 5, 10, 0, 40], seed=seed + k)
                k += 1
                yield {"image": torch.randint(0, 256, (B, 16, 16, 3), dtype=torch.uint8, generator=g),
                       "text": {"input_ids": ids, "attention_mask": mask}}
        return it

    tr.fit({"train": gen(0), "val": gen(1), "local_batch_size": B}, training_steps_per_epoch=2, epochs=3,
           val_steps_per_epoch=1, sampler_class=EulerSampler,
           sampling_noise_schedule=KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
           verbose=False, val_diffusion_steps=3)
    assert len(seen["clip_similarity"]) == len(seen["clip_score"]) == 4          # sanity validation + 3 epochs
    assert all(math.isfinite(v) for v in seen["clip_similarity"] + seen["clip_score"])
    assert tr.best_val_metrics["val/clip_similarity"] == min(seen["clip_similarity"])
    assert tr.best_val_metrics["val/clip_score"] == max(seen["clip_score"])
