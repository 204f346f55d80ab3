"""Run-config parsing and checkpoint loading for inference (API of flaxdiff/inference/utils.py).

`parse_config` turns the config a training run logs (training.py's `CONFIG`: model kwargs, architecture, input
config, arguments, autoencoder) back into a model, a noise schedule, a prediction transform and an input config.
There is no wandb here: the wandb entry points raise, and the caller hands over the config and a local checkpoint
directory instead.
"""
from __future__ import annotations

import torch

from .. import checkpoint as ckpt_io
from .._lib import FdxError
from ..inputs import ConditionalInputConfig, DiffusionInputConfig
from ..predictors import KarrasPredictionTransform, VPredictionTransform
from ..schedulers import CosineNoiseScheduler, KarrasVENoiseScheduler
from ..utils import ACTIVATION_MAP, DTYPE_MAP, PRECISION_MAP, defaultTextEncodeModel

# the dtype names of inference/utils.py:92-99, which also spell out the jax module path
_DTYPE_MAP = {**DTYPE_MAP, "jax.numpy.float32": torch.float32, "jax.numpy.bfloat16": torch.bfloat16}

_NO_WANDB = ("wandb is not a dependency of flaxdiff_b200: download the run's checkpoint directory and config yourself "
             "and use DiffusionInferencePipeline.from_checkpoint(checkpoint_dir, config)")


def _model_classes():
    from ..models.mmdit import HierarchicalMMDiT, SimpleMMDiT
    from ..models.simple_dit import SimpleDiT
    from ..models.simple_unet import Unet
    from ..models.ssm_dit import HybridSSMAttentionDiT
    from ..models.udit import SimpleUDiT
    from ..models.uvit import UViT
    return {"unet": Unet, "uvit": UViT, "simple_dit": SimpleDiT, "simple_mmdit": SimpleMMDiT,
            "simple_udit": SimpleUDiT, "hierarchical_mmdit": HierarchicalMMDiT, "hybrid_dit": HybridSSMAttentionDiT}


def _map_nested_config(config: dict) -> dict:
    """inference/utils.py:137-160: like `utils.map_nested_config`, but every other value is kept, lists are mapped
    item by item, and a string that names none of the maps is kept unless it contains a dot."""
    out = {}
    for key, value in config.items():
        if isinstance(value, dict):
            out[key] = _map_nested_config(value)
        elif isinstance(value, list):
            out[key] = [_map_nested_config(v) if isinstance(v, dict) else v for v in value]
        elif isinstance(value, str):
            if value in _DTYPE_MAP:
                out[key] = _DTYPE_MAP[value]
            elif value in PRECISION_MAP:
                out[key] = PRECISION_MAP[value]
            elif value in ACTIVATION_MAP:
                out[key] = ACTIVATION_MAP[value]
            elif "." in value:
                print(f"Ignoring key {key} with value {value} as it contains a dot.")
            else:
                out[key] = value
        else:
            out[key] = value
    return out


def get_wandb_run(wandb_run: str, project, entity):
    raise FdxError(_NO_WANDB)


def load_from_wandb_run(run, project: str, entity: str = None):
    raise FdxError(_NO_WANDB)


def load_from_wandb_registry(modelname: str, project: str, entity: str = None, version: str = 'latest',
                             registry: str = 'wandb-registry-model'):
    raise FdxError(_NO_WANDB)


def parse_config(config, overrides=None):
    """inference/utils.py:61-268 -> {model, model_config, architecture, autoencoder, noise_schedule,
    prediction_transform, input_config, raw_config}.

    `config` has the shape training.py logs.  `overrides` merge into `arguments` and into the top-level keys they
    name.  `config["input_config"]` is a serialised `DiffusionInputConfig` (its encoders are rebuilt through the
    registry), or a `DiffusionInputConfig` object, which is used as is; when it is missing, the reference's default
    text condition is built from the CLIP model in the local Hugging Face cache.  The model is built with the mapped
    model kwargs; when they give no `context_dim` and the input config has a condition, the model's context width is
    that condition's embedding width, as the trainer's `init` infers it."""
    if overrides is not None:
        conf = dict(config)
        if 'arguments' in conf:
            conf['arguments'] = {**conf['arguments'], **overrides}
            for key in overrides:
                if key in conf:
                    conf[key] = overrides[key]
    else:
        conf = config
    args = conf.get('arguments', {})

    architecture = conf.get('architecture', args.get('architecture', 'unet'))
    if isinstance(architecture, str):
        # the suffix flags (use_2d_fusion, use_hilbert, use_zigzag) are already in the model config
        for suffix in ('+2d', '+hilbert', '+zigzag'):
            architecture = architecture.replace(suffix, '')
    classes = _model_classes()
    if architecture not in classes:
        raise FdxError(f"architecture {architecture!r} is not supported; supported: {', '.join(classes)}")

    if conf.get('autoencoder', args.get('autoencoder')):
        raise FdxError("latent diffusion (autoencoder) is outside the supported hot path")

    input_config = conf.get('input_config', None)
    if input_config is None:
        # inference/utils.py:203-224: runs logged before input_config existed were text-conditioned on CLIP
        image_size = args.get('image_size', 128)
        text = ConditionalInputConfig(encoder=defaultTextEncodeModel(backend="fdx"), conditioning_data_key='text',
                                      pretokenized=True, unconditional_input="", model_key_override="textcontext")
        input_config = DiffusionInputConfig(sample_data_key='image', sample_data_shape=(image_size, image_size, 3),
                                            conditions=[text])
    elif not isinstance(input_config, DiffusionInputConfig):
        input_config = DiffusionInputConfig.deserialize(input_config)

    model_kwargs = _map_nested_config(conf['model'])
    if model_kwargs.get('context_dim') is None and input_config.conditions:
        model_kwargs['context_dim'] = int(input_config.conditions[0].get_unconditional().shape[-1])
    model = classes[architecture](**model_kwargs)

    schedule = conf.get('noise_schedule', args.get('noise_schedule', 'edm'))
    if schedule in ('edm', 'karras'):
        noise_schedule = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5)
        prediction_transform = KarrasPredictionTransform(sigma_data=noise_schedule.sigma_data)
    elif schedule == 'cosine':
        noise_schedule = CosineNoiseScheduler(1000, beta_end=1)
        prediction_transform = VPredictionTransform()
    else:
        raise ValueError(f"Unknown noise schedule: {schedule}")

    return {'model': model, 'model_config': model_kwargs, 'architecture': architecture, 'autoencoder': None,
            'noise_schedule': noise_schedule, 'prediction_transform': prediction_transform,
            'input_config': input_config, 'raw_config': conf}


def load_from_checkpoint(checkpoint_dir: str):
    """inference/utils.py:270-290: (state, best_state) of the latest step under `checkpoint_dir`, as the nested
    numpy trees `checkpoint.load_tree` returns; (None, None) and a warning when there is nothing readable."""
    try:
        _, ckpt = ckpt_io.load_tree(checkpoint_dir)
        state, best_state = ckpt.get('state'), ckpt.get('best_state')
        print(f"Loaded checkpoint from local dir {checkpoint_dir}")
        return state, best_state
    except Exception as e:  # noqa: BLE001  (the reference's contract: any failure is a warning)
        print(f"Warning: Failed to load checkpoint from local dir: {e}")
        return None, None
