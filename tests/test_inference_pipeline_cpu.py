"""The inference pipeline's host logic (flaxdiff_b200/inference): run configs as training.py logs them back into
models, schedules and input configs; the refusals; the wandb entry points; checkpoint loading; and how the sampler
splits raw conditioning among its conditions."""
import json
import sys

import numpy as np
import pytest
import torch

from flaxdiff_b200 import checkpoint as ckpt_io
from flaxdiff_b200 import utils
from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.inference import (DiffusionInferencePipeline, get_wandb_run, load_from_checkpoint,
                                     load_from_wandb_registry, load_from_wandb_run, parse_config)
from flaxdiff_b200.inputs import (ConditionalInputConfig, ConditioningEncoder, DiffusionInputConfig,
                                  RandomEmbeddingEncoder)
from flaxdiff_b200.models.mmdit import HierarchicalMMDiT, SimpleMMDiT
from flaxdiff_b200.models.simple_dit import SimpleDiT
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT
from flaxdiff_b200.models.udit import SimpleUDiT
from flaxdiff_b200.models.uvit import UViT
from flaxdiff_b200.predictors import KarrasPredictionTransform, VPredictionTransform
from flaxdiff_b200.samplers import EulerSampler
from flaxdiff_b200.schedulers import CosineNoiseScheduler, KarrasVENoiseScheduler

# training.py's argument defaults (training.py:139-212), with widths and heads the engine's models accept
ARGS = dict(emb_features=256, feature_depths=[64, 128, 256, 512], attention_heads=8, flash_attention=False,
            use_projection=False, use_self_and_cross=True, only_pure_attention=True, norm_groups=8, named_norms=False,
            num_res_blocks=2, num_middle_res_blocks=1, activation="swish", patch_size=4, num_layers=6, num_heads=4,
            mlp_ratio=4, dropout_rate=0.1, add_residualblock_output=False, ssm_attention_ratio="3:1",
            ssm_state_dim=64, image_size=32, noise_schedule="edm", autoencoder=None)


def _training_model_config(architecture: str, dtype, precision, **over):
    """(architecture name as logged, model kwargs) the way training.py:347-491 builds them for `architecture`."""
    a = {**ARGS, **over}
    use_hilbert = use_zigzag = use_2d_fusion = False
    name = architecture
    if "+2d" in name:
        name, use_2d_fusion = name.replace("+2d", ""), True
    if "hilbert" in name:
        name, use_hilbert = name.split("+")[0], True
    elif "zigzag" in name:
        name, use_zigzag = name.split("+")[0], True
    attn = [None]
    if a["attention_heads"] > 0:
        attn += [{"heads": a["attention_heads"], "dtype": dtype, "flash_attention": a["flash_attention"],
                  "use_projection": a["use_projection"], "use_self_and_cross": a["use_self_and_cross"],
                  "only_pure_attention": a["only_pure_attention"]}] * (len(a["feature_depths"]) - 2)
        attn += [{"heads": a["attention_heads"], "dtype": dtype, "flash_attention": False, "use_projection": False,
                  "use_self_and_cross": a["use_self_and_cross"], "only_pure_attention": a["only_pure_attention"]}]
    else:
        attn += [None] * (len(a["feature_depths"]) - 1)
    cfg = {"emb_features": a["emb_features"], "dtype": dtype, "precision": precision, "activation": a["activation"],
           "output_channels": 3, "norm_groups": a["norm_groups"]}
    common = {"patch_size": a["patch_size"], "num_layers": a["num_layers"], "num_heads": a["num_heads"],
              "dropout_rate": a["dropout_rate"], "use_flash_attention": a["flash_attention"]}
    kwargs = {
        "unet": {"feature_depths": a["feature_depths"], "attention_configs": attn,
                 "num_res_blocks": a["num_res_blocks"], "num_middle_res_blocks": a["num_middle_res_blocks"],
                 "named_norms": a["named_norms"]},
        "uvit": {**common, "add_residualblock_output": a["add_residualblock_output"],
                 "use_self_and_cross": a["use_self_and_cross"], "use_hilbert": use_hilbert},
        "simple_udit": {**common, "mlp_ratio": a["mlp_ratio"], "use_hilbert": use_hilbert},
        "simple_dit": {**common, "mlp_ratio": a["mlp_ratio"], "use_hilbert": use_hilbert, "use_zigzag": use_zigzag},
        "simple_mmdit": {**common, "mlp_ratio": a["mlp_ratio"], "use_hilbert": use_hilbert},
        "hierarchical_mmdit": {
            "base_patch_size": a["patch_size"] // 2,
            "emb_features": (a["emb_features"] - 256, a["emb_features"], a["emb_features"] + 256),
            "num_layers": (a["num_layers"] // 3, a["num_layers"] // 2, a["num_layers"]),
            "num_heads": (a["num_heads"] - 2, a["num_heads"], a["num_heads"] + 2),
            "dropout_rate": a["dropout_rate"], "use_flash_attention": a["flash_attention"],
            "mlp_ratio": a["mlp_ratio"], "use_hilbert": use_hilbert},
        "hybrid_dit": {**common, "mlp_ratio": a["mlp_ratio"], "use_hilbert": use_hilbert, "use_zigzag": use_zigzag,
                       "use_2d_fusion": use_2d_fusion, "ssm_state_dim": a["ssm_state_dim"],
                       "ssm_attention_ratio": a["ssm_attention_ratio"]},
    }[name]
    cfg.update(kwargs)
    if name == "uvit":
        cfg["emb_features"] = 768
    return name, cfg


def _logged(cfg):
    """What a wandb run config holds: JSON, with jax dtypes and precisions written as strings."""
    def enc(o):
        if isinstance(o, torch.dtype):
            return "bfloat16"
        raise TypeError(o)
    return json.loads(json.dumps(cfg, default=enc))


def _run_config(architecture, input_config, *, dtype_name="bfloat16", precision_name="DEFAULT", **over):
    name, model = _training_model_config(architecture, torch.bfloat16, None, **over)
    logged = _logged(model)
    logged["dtype"] = dtype_name
    logged["precision"] = precision_name
    if "attention_configs" in logged:
        for c in logged["attention_configs"]:
            if c is not None:
                c["dtype"] = dtype_name
    args = {**ARGS, **over, "architecture": architecture}
    return {"model": logged, "architecture": name, "dataset": {"name": "x", "length": 1, "batches": 1},
            "input_config": input_config, "arguments": args, "autoencoder": None, "autoencoder_opts": "{}"}


CLASSES = {"unet": Unet, "uvit": UViT, "simple_udit": SimpleUDiT, "simple_dit": SimpleDiT, "simple_mmdit": SimpleMMDiT,
           "hierarchical_mmdit": HierarchicalMMDiT, "hybrid_dit": HybridSSMAttentionDiT}


def _text_config(features=768):
    return DiffusionInputConfig("image", (32, 32, 3), [ConditionalInputConfig(
        RandomEmbeddingEncoder(seq_len=77, features=features), conditioning_data_key="text", unconditional_input="",
        model_key_override="textcontext")])


def _state(model):
    if isinstance(model, Unet):
        return utils.serialize_model(model)
    return model.config()


@pytest.mark.parametrize("architecture,over,names", [
    ("unet", {}, ("bfloat16", "DEFAULT")),
    ("unet", {"activation": "mish", "named_norms": True}, ("jax.numpy.bfloat16", "Precision.DEFAULT")),
    ("uvit", {"num_heads": 12}, ("bfloat16", "HIGHEST")),
    ("simple_udit", {}, ("jax.numpy.bfloat16", "None")),
    ("simple_dit", {}, ("bfloat16", "default")),
    ("simple_mmdit", {"activation": "jax._src.nn.functions.silu"}, ("bfloat16", "DEFAULT")),
    ("hierarchical_mmdit", {"emb_features": 512}, ("bfloat16", "DEFAULT")),
    ("hybrid_dit", {}, ("bfloat16", "high")),
    ("hybrid_dit+hilbert", {}, ("bfloat16", "DEFAULT")),
    ("hybrid_dit+zigzag", {"ssm_attention_ratio": "1:1"}, ("bfloat16", "DEFAULT")),
])
def test_parse_config_builds_the_model_training_built(architecture, over, names, capsys):
    """Every architecture of training.py the engine builds: the logged config gives the model a direct
    construction with training.py's kwargs gives, with the text width of the input config as context_dim."""
    name, kwargs = _training_model_config(architecture, torch.bfloat16, None, **over)
    ic = _text_config()
    out = parse_config(_run_config(architecture, ic, dtype_name=names[0], precision_name=names[1], **over))
    if kwargs.get("activation") == "jax._src.nn.functions.silu":
        kwargs["activation"] = "swish"
    direct = CLASSES[name](**kwargs, context_dim=768)
    assert type(out["model"]) is CLASSES[name] and out["architecture"] == name
    assert _state(out["model"]) == _state(direct)
    assert out["model"].param_specs() == direct.param_specs()
    assert out["model_config"]["context_dim"] == 768 and out["model_config"]["dtype"] is torch.bfloat16
    assert out["input_config"] is ic and out["autoencoder"] is None
    if "." in names[1]:
        assert "Ignoring key precision with value Precision.DEFAULT as it contains a dot." in capsys.readouterr().out
        assert "precision" not in out["model_config"]


def test_parse_config_unconditioned_input_config_is_deserialised():
    ic = DiffusionInputConfig("image", (32, 32, 3), [])
    out = parse_config(_run_config("hybrid_dit+zigzag", _logged(ic.serialize())))
    _, kwargs = _training_model_config("hybrid_dit+zigzag", torch.bfloat16, None)
    assert out["model"].config() == HybridSSMAttentionDiT(**kwargs).config()
    assert out["model"].context_dim is None and out["model"].use_zigzag
    assert out["input_config"].conditions == [] and out["input_config"].sample_data_shape == (32, 32, 3)


@pytest.mark.parametrize("architecture,over,exc,needle", [
    ("simple_dit+hilbert", {}, FdxError, "Hilbert / zigzag"),
    ("hybrid_dit+2d", {}, FdxError, "use_2d_fusion"),
])
def test_parse_config_passes_model_refusals_through(architecture, over, exc, needle):
    with pytest.raises(exc, match=needle):
        parse_config(_run_config(architecture, _text_config(), **over))


def test_parse_config_refuses_architectures_autoencoders_and_schedules():
    base = _run_config("unet", _text_config())
    with pytest.raises(FdxError, match="diffusers_unet_simple"):
        parse_config({**base, "architecture": "diffusers_unet_simple", "model": {}})
    with pytest.raises(FdxError, match="no_such_net"):
        parse_config({**base, "architecture": "no_such_net"})
    with pytest.raises(FdxError, match="latent diffusion \\(autoencoder\\) is outside the supported hot path"):
        parse_config({**base, "autoencoder": "stable_diffusion"})
    with pytest.raises(ValueError, match="Unknown noise schedule: linear"):
        parse_config({**base, "noise_schedule": "linear"})


def test_parse_config_without_input_config_needs_the_local_clip_model():
    """inference/utils.py:203-224: an old run config means CLIP text conditioning; nothing is downloaded."""
    cfg = _run_config("unet", None)
    del cfg["input_config"]
    with pytest.raises(FdxError, match="local Hugging Face cache"):
        parse_config(cfg)


@pytest.mark.parametrize("schedule", ["edm", "karras", "cosine"])
def test_noise_schedule_mapping(schedule):
    out = parse_config({**_run_config("simple_dit", _text_config()), "noise_schedule": schedule})
    ns, tr = out["noise_schedule"], out["prediction_transform"]
    if schedule == "cosine":
        assert type(ns) is CosineNoiseScheduler and ns.max_timesteps == 1000 and type(tr) is VPredictionTransform
        ref = CosineNoiseScheduler(1000, beta_end=1)
        assert torch.equal(torch.as_tensor(ns.betas), torch.as_tensor(ref.betas))
    else:
        assert type(ns) is KarrasVENoiseScheduler and type(tr) is KarrasPredictionTransform
        assert (ns.max_timesteps, ns.sigma_max, ns.rho, ns.sigma_data, tr.sigma_data) == (1, 80, 7, 0.5, 0.5)


def test_noise_schedule_falls_back_to_arguments_then_edm():
    cfg = _run_config("simple_dit", _text_config())
    cfg["arguments"]["noise_schedule"] = "cosine"
    assert type(parse_config(cfg)["noise_schedule"]) is CosineNoiseScheduler
    del cfg["arguments"]["noise_schedule"]
    assert type(parse_config(cfg)["noise_schedule"]) is KarrasVENoiseScheduler


def test_overrides_merge_into_arguments_and_top_level_keys():
    cfg = {**_run_config("simple_dit", _text_config()), "noise_schedule": "edm"}
    out = parse_config(cfg, overrides={"noise_schedule": "cosine", "image_size": 64})
    assert type(out["noise_schedule"]) is CosineNoiseScheduler
    raw = out["raw_config"]
    assert raw["arguments"]["noise_schedule"] == "cosine" and raw["arguments"]["image_size"] == 64
    assert raw["noise_schedule"] == "cosine" and "image_size" not in raw      # only keys already at the top level
    assert cfg["noise_schedule"] == "edm" and cfg["arguments"]["image_size"] == 32     # the caller's dict is kept
    # as in the reference, a config without `arguments` takes no overrides
    bare = {k: v for k, v in cfg.items() if k != "arguments"}
    assert type(parse_config(bare, overrides={"noise_schedule": "cosine"})["noise_schedule"]) is KarrasVENoiseScheduler


def test_wandb_entry_points_raise_without_importing_wandb():
    sys.modules.pop("wandb", None)
    calls = [lambda: get_wandb_run("run", "proj", "me"), lambda: load_from_wandb_run("run", "proj", "me"),
             lambda: load_from_wandb_registry("model", "proj"),
             lambda: DiffusionInferencePipeline.from_wandb_run("run", "proj", "me"),
             lambda: DiffusionInferencePipeline.from_wandb_registry("model", "proj")]
    for call in calls:
        with pytest.raises(FdxError, match="wandb is not a dependency"):
            call()
    assert "wandb" not in sys.modules


def test_load_from_checkpoint(tmp_path, capsys):
    assert load_from_checkpoint(str(tmp_path / "missing")) == (None, None)
    assert "Warning: Failed to load checkpoint" in capsys.readouterr().out
    st = {"step": np.asarray(3, np.int32), "params": {"params": {"a": {"kernel": np.ones((2, 3), np.float32)}}},
          "ema_params": {"params": {"a": {"kernel": np.zeros((2, 3), np.float32)}}}}
    ckpt_io.save_tree(str(tmp_path), 3, {"state": st, "best_state": st, "best_loss": np.asarray(1.0)})
    ckpt_io.save_tree(str(tmp_path), 7, {"state": {**st, "step": np.asarray(7, np.int32)}, "best_state": st})
    state, best = load_from_checkpoint(str(tmp_path))
    assert int(state["step"]) == 7 and int(best["step"]) == 3                # the latest step
    assert np.array_equal(state["params"]["params"]["a"]["kernel"], np.ones((2, 3), np.float32))


def test_pipeline_defaults_and_sampler_cache():
    """pipeline.py:149-215: PRNGKey(42) unless a state is given; one sampler per (class, guidance scale)."""
    ic = DiffusionInputConfig("image", (32, 32, 3), [])
    parsed = parse_config(_run_config("simple_dit", ic.serialize()))
    pipe = DiffusionInferencePipeline.create(parsed, state={"params": None, "ema_params": None})
    assert pipe.rngstate.rng == utils.PRNGKey(42) and pipe.name is None
    a = pipe.get_sampler(0.0, EulerSampler)
    assert pipe.get_sampler(0.0, EulerSampler) is a and pipe.get_sampler(2.0, EulerSampler) is not a
    assert a.model is parsed["model"] and a.input_config is parsed["input_config"] and a.guidance_scale == 0.0


# ----------------------------------------------------------------------------------------------- raw conditioning
class _Recorder(EulerSampler):
    """Runs generate_samples' argument handling on the host: no initial noise, one evaluation that records the
    conditioning inputs it is handed, no post-processing."""

    def _get_initial_samples(self, resolution, batch_size, rngs, start_step, device):
        return torch.zeros(batch_size, resolution, resolution, 3)

    def _flat_for(self, params, device):
        return params

    def sample_model(self, params, x_t, t, *conditioning_inputs):
        self.seen = conditioning_inputs
        return x_t, x_t, x_t

    def post_process(self, samples):
        return samples


class _Enc(ConditioningEncoder):
    """Records each call; embeds item i of a call as a row of value hash(item) % 97."""

    def __init__(self, key):
        self.key, self.calls = key, []

    def __call__(self, data):
        self.calls.append(list(data))
        return torch.tensor([[float(hash(str(d)) % 97)] for d in data])


def _recorder(*keys):
    encs = [_Enc(k) for k in keys]
    ic = DiffusionInputConfig("image", (8, 8, 3), [ConditionalInputConfig(e, unconditional_input="") for e in encs])
    for e in encs:
        e.calls.clear()                         # drop the null-embedding calls of ConditionalInputConfig
    smp = _Recorder(None, KarrasVENoiseScheduler(1), KarrasPredictionTransform(0.5), ic)
    return smp, encs


def _run(smp, **kw):
    smp.generate_samples(None, 2, 8, steps_override=[1], device="cpu", **kw)
    return smp.seen


def test_raw_conditioning_scalar_entries_go_to_every_condition():
    smp, (a, b) = _recorder("text", "style")
    seen = _run(smp, conditioning=["a fox", "a cat"])
    assert a.calls == [["a fox", "a cat"]] and b.calls == [["a fox", "a cat"]]     # one encode per condition
    assert len(seen) == 2 and torch.equal(seen[0], a(["a fox", "a cat"]))


def test_raw_conditioning_tuples_match_conditions_by_position():
    smp, (a, b) = _recorder("text", "style")
    seen = _run(smp, conditioning=[("a fox", "oil"), ["a cat", "ink"]])
    assert a.calls == [["a fox", "a cat"]] and b.calls == [["oil", "ink"]]
    assert torch.equal(seen[1], b(["oil", "ink"]))


def test_raw_conditioning_dicts_match_conditions_by_encoder_key():
    smp, (a, b) = _recorder("text", "style")
    _run(smp, conditioning=[{"style": "oil", "text": "a fox"}, {"text": "a cat", "style": "ink", "extra": 1}])
    assert a.calls == [["a fox", "a cat"]] and b.calls == [["oil", "ink"]]
    with pytest.raises(ValueError, match="Conditioning input style not found in provided dictionary"):
        _run(smp, conditioning=[{"text": "a fox", "style": "oil"}, {"text": "a cat"}])


def test_raw_conditioning_with_embeddings_or_without_conditions_raises():
    smp, (a,) = _recorder("text")
    emb = (torch.zeros(2, 1),)
    with pytest.raises(ValueError, match="Cannot provide both conditioning and model_conditioning_inputs"):
        _run(smp, conditioning=["a fox", "a cat"], model_conditioning_inputs=emb)
    assert a.calls == []
    assert _run(smp, model_conditioning_inputs=emb) == emb                   # the embeddings path is unchanged
    bare = _Recorder(None, KarrasVENoiseScheduler(1), KarrasPredictionTransform(0.5), None)
    with pytest.raises(FdxError, match="conditioning"):
        _run(bare, conditioning=["a fox"])


def test_conditioning_batch_must_match_the_samples():
    """The models read one conditioning row per sample (two with guidance) and broadcast only a batch of 1: any
    other batch is refused on the host, before a launch could read past the rows it was given."""
    smp, (a,) = _recorder("text")
    with pytest.raises(ValueError, match="conditioning has 1 entries for 2 samples"):
        _run(smp, conditioning=["a red fox in snow"])
    with pytest.raises(ValueError, match="conditioning has 3 entries for 2 samples"):
        _run(smp, conditioning=["a", "b", "c"])
    assert a.calls == []                                       # refused before anything is encoded
    with pytest.raises(ValueError, match="batch 3 for 2 samples"):
        _run(smp, model_conditioning_inputs=(torch.zeros(3, 1),))
    assert _run(smp, model_conditioning_inputs=(torch.zeros(1, 1),))[0].shape == (1, 1)   # broadcast, no guidance
    # with priors the batch is theirs, whatever num_samples says
    smp.generate_samples(None, 5, 8, steps_override=[1], device="cpu", priors=torch.zeros(2, 8, 8, 3),
                         conditioning=["a", "b"])
    assert smp.seen[0].shape[0] == 2
    smp.guidance_scale = 3.0                                   # a batch of 1 would meet a single null row
    with pytest.raises(ValueError, match="batch 1 for 2 samples: its batch must be the number of samples$"):
        _run(smp, model_conditioning_inputs=(torch.zeros(1, 1),))
    assert _run(smp, conditioning=["a", "b"])[0].shape == (2, 1)
