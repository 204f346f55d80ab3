"""The CLIP metrics without a GPU: the engine's resize tables reproduce PIL's bicubic resize bit for bit, the metric
objects carry the reference's names and directions, a model missing from the local cache fails with FdxError, and
the configurations the kernels cannot run are refused at construction."""
import numpy as np
import pytest
import torch

from clip_metric_ref import clip_pair_config, pil_resize_np, processor_u8, quantise_np
from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.metrics import EvaluationMetric
from flaxdiff_b200.models.clip_vision import CLIPPair, CLIPVisionTower, crop_tables, normalise_lut, resize_shape

SIZES = [(16, 16), (28, 28), (32, 32), (64, 64), (96, 128), (128, 128), (224, 224), (256, 256), (300, 300),
         (512, 512), (224, 300), (300, 224)]


def _image(H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("H,W", SIZES)
def test_table_resize_equals_pil_bicubic(H, W):
    from PIL import Image
    u8 = _image(H, W, H * 1000 + W)
    nh, nw = resize_shape(H, W, 224)
    ref = np.asarray(Image.fromarray(u8).resize((nw, nh), Image.BICUBIC))
    assert np.array_equal(pil_resize_np(u8, nh, nw), ref)


@pytest.mark.parametrize("H,W", SIZES)
def test_crop_tables_are_the_processor_window(H, W):
    """The crop tables, applied the way fdx_clip_image_prep applies them (vertical taps of horizontal sums, each
    clipped), give CLIPImageProcessorPil's uint8 crop."""
    from PIL import Image
    u8 = _image(H, W, H + W)
    tab, ky, kx = crop_tables(H, W, 224, 224)
    ty = tab[:224 * (2 + ky)].reshape(224, 2 + ky)
    tx = tab[224 * (2 + ky):].reshape(224, 2 + kx)
    assert tab.size == 224 * (4 + ky + kx)
    src = u8.astype(np.int64)
    hrow = np.zeros((H, 224, 3), np.int64)
    for X in range(224):
        acc = np.full((H, 3), 1 << 21, np.int64)
        for t in range(tx[X, 1]):
            acc += src[:, tx[X, 0] + t] * int(tx[X, 2 + t])
        hrow[:, X] = np.clip(acc >> 22, 0, 255)
    out = np.zeros((224, 224, 3), np.int64)
    for Y in range(224):
        acc = np.full((224, 3), 1 << 21, np.int64)
        for t in range(ty[Y, 1]):
            acc += hrow[ty[Y, 0] + t] * int(ty[Y, 2 + t])
        out[Y] = np.clip(acc >> 22, 0, 255)
    nh, nw = resize_shape(H, W, 224)
    full = np.asarray(Image.fromarray(u8).resize((nw, nh), Image.BICUBIC))
    top, left = (nh - 224) // 2, (nw - 224) // 2
    assert np.array_equal(out, full[top:top + 224, left:left + 224])
    assert np.array_equal(out, processor_u8(u8))


def test_processor_restatement_matches_clip_image_processor_pil():
    from transformers.models.clip import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil()
    lut = normalise_lut(proc.rescale_factor, proc.image_mean, proc.image_std)
    for H, W in ((64, 64), (96, 128)):
        u8 = _image(H, W, 7)
        pv = proc(images=[u8], return_tensors="np")["pixel_values"][0]            # [3, 224, 224] f32
        crop = processor_u8(u8)
        assert np.array_equal(lut[np.arange(3)[None, None, :], crop], pv.transpose(1, 2, 0))


def test_quantise_clamps_and_maps_nan_to_zero():
    x = np.array([-2.0, -1.0, -0.5, 0.0, 0.999, 1.0, 2.0, np.inf, -np.inf, np.nan], np.float32)
    assert quantise_np(x).tolist() == [0, 0, 63, 127, 254, 255, 255, 255, 0, 0]


def test_evaluation_metric_fields_and_defaults():
    import dataclasses
    m = EvaluationMetric(function=len, name="x")
    assert [f.name for f in dataclasses.fields(EvaluationMetric)] == ["function", "name", "higher_is_better"]
    assert m.higher_is_better is False and m.function is len and m.name == "x"
    assert EvaluationMetric(len, "y", True).higher_is_better is True


def test_metric_names_and_directions(monkeypatch):
    from flaxdiff_b200.metrics import images
    monkeypatch.setitem(images._clip_cache, "stub", object())
    sim, score = images.get_clip_metric("stub"), images.get_clip_score_metric("stub")
    assert (sim.name, sim.higher_is_better) == ("clip_similarity", False)
    assert (score.name, score.higher_is_better) == ("clip_score", True)


def test_missing_model_is_an_fdx_error(monkeypatch, tmp_path):
    from flaxdiff_b200.metrics import get_clip_metric, get_clip_score_metric
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    monkeypatch.setenv("HF_HOME", str(tmp_path))
    for fn in (get_clip_metric, get_clip_score_metric):
        with pytest.raises(FdxError, match="'openai/clip-vit-large-patch14' from the local Hugging Face cache"):
            fn()
    with pytest.raises(FdxError, match="local Hugging Face cache"):
        get_clip_metric(str(tmp_path / "no-such-model"))


def _vision(**kw):
    cfg = clip_pair_config("tiny").vision_config
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("kw,match", [
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(hidden_act="relu"), "hidden_act"),
    (dict(num_attention_heads=8), "head width 16 "),
    (dict(hidden_size=96, num_attention_heads=3), "multiple of 64"),
    (dict(hidden_size=1344, num_attention_heads=21), "multiple of 64, <= 1280"),
    (dict(hidden_size=1280, num_attention_heads=16), "head width 80 "),
    (dict(intermediate_size=100), "intermediate_size"),
    (dict(image_size=225), "not a multiple of patch_size"),
    (dict(num_channels=4), "num_channels"),
])
def test_vision_tower_refuses_configs_outside_the_kernels(kw, match):
    with pytest.raises(FdxError, match=match):
        CLIPVisionTower(_vision(**kw), {}, device="cpu")


def test_vision_tower_accepts_head_width_128_and_packs_the_patch_kernel():
    from transformers import CLIPVisionModel
    cfg = _vision(hidden_size=256, num_attention_heads=2)
    torch.manual_seed(0)
    model = CLIPVisionModel(cfg)
    t = CLIPVisionTower(cfg, model.state_dict(), device="cpu")
    assert (t.D // t.heads, t.G, t.K, t.ld) == (128, 16, 588, 592)
    w = model.state_dict()["vision_model.embeddings.patch_embedding.weight"]       # [D, 3, 14, 14]
    assert torch.equal(t.w["wpatch"][1 * 196 + 2 * 14 + 5, 7], w[7, 1, 2, 5].to(torch.bfloat16))   # (c, ky, kx)
    assert torch.equal(t.w["wpatch"], w.reshape(256, 588).t().to(torch.bfloat16))
    assert all((v.data_ptr() - t.buffer.data_ptr()) % 256 == 0 for v in t.w.values())


def _proc(**kw):
    from transformers.models.clip import CLIPImageProcessorPil
    return CLIPImageProcessorPil(**kw)


@pytest.mark.parametrize("proc,cfg_kw,match", [
    (dict(resample=2), {}, "not BICUBIC"),
    (dict(do_center_crop=False), {}, "do_center_crop"),
    (dict(do_resize=False), {}, "do_resize"),
    (dict(crop_size={"height": 224, "width": 196}), {}, "square"),
    (dict(size={"shortest_edge": 196}, crop_size={"height": 196, "width": 196}), {}, "image_size 224"),
    (dict(), dict(projection_dim=48), "projection_dim"),
])
def test_pair_refuses_processors_and_configs_outside_the_kernels(proc, cfg_kw, match):
    cfg = clip_pair_config("tiny")
    for k, v in cfg_kw.items():
        setattr(cfg, k, v)
    with pytest.raises(FdxError, match=match):
        CLIPPair(cfg, {}, _proc(**proc), device="cpu")


def _validate(metrics, values, overrides=None):
    """GeneralDiffusionTrainer.validation_loop over one validation step per value, with stand-in samples."""
    from types import SimpleNamespace

    from flaxdiff_b200.trainer import GeneralDiffusionTrainer
    tr = SimpleNamespace(eval_metrics=metrics, metric_higher_is_better=overrides or {}, best_val_metrics={})
    it = iter(values)
    for _ in values:
        GeneralDiffusionTrainer.validation_loop(tr, None, lambda s, b, n: next(it), None, 1, 0)
    return tr.best_val_metrics


def test_validation_tracks_the_direction_each_metric_declares():
    values = [3.0, 1.0, 2.0]
    up, down = EvaluationMetric(lambda s, b: s, "up", True), EvaluationMetric(lambda s, b: s, "down")

    class Plain:                                          # no higher_is_better attribute: lower is better
        name = "plain"
        function = staticmethod(lambda s, b: s)

    assert _validate([up, down, Plain], values) == {"val/up": 3.0, "val/down": 1.0, "val/plain": 1.0}
    # metric_higher_is_better keeps precedence over the declared direction
    assert _validate([up, down], values, {"val/up": False, "val/down": True}) == {"val/up": 1.0, "val/down": 3.0}
