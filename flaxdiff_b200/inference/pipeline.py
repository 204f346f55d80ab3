"""`DiffusionInferencePipeline`: from a trained run to images (API of flaxdiff/inference/pipeline.py).

A pipeline holds the model that `parse_config` built from a run config, the run's `state` / `best_state`
(`{"step", "params", "ema_params"}`), the noise schedule, the prediction transform and the input config.  A parameter
tree is packed into `FlatParams` on the GPU the first time a call samples from it, and the packed copy is kept for
later calls; trees no call uses stay on the host.  `generate_samples` hands prompts (or embeddings) to a
cached sampler: the prompts are encoded by the input config's encoders - with `CLIPTextEncoder(backend="fdx")` by
the engine's text tower - and the denoiser and the update steps run on the engine as in any sampler call.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Tuple, Type, Union

import torch

from .. import checkpoint as ckpt_io
from .. import utils
from ..inputs import DiffusionInputConfig
from ..predictors import DiffusionPredictionTransform
from ..samplers import DiffusionSampler, EulerAncestralSampler
from ..schedulers import NoiseScheduler
from ..utils import RandomMarkovState
from .utils import load_from_wandb_registry, load_from_wandb_run, parse_config


@dataclass
class InferencePipeline:
    """Inference pipeline for a general model."""
    name: str = None
    model: Any = None
    state: Any = None
    best_state: Any = None

    def from_wandb(self, wandb_run: str, wandb_project: str, wandb_entity: str):
        raise NotImplementedError("InferencePipeline does not support from_wandb.")


@dataclass
class DiffusionInferencePipeline(InferencePipeline):
    """Inference pipeline for diffusion models (pipeline.py:41-271).

    Seeds: `create` always sets `rngstate` to `RandomMarkovState(PRNGKey(42))`, and `generate_samples` draws from
    `self.rngstate or RandomMarkovState(PRNGKey(seed or 0))`, so - as in the reference - `seed` only takes effect
    once the caller sets `pipeline.rngstate = None`, and every call with the same arguments returns the same
    images."""
    artifact: Any = None
    state: Dict[str, Any] = None
    best_state: Dict[str, Any] = None
    rngstate: Optional[RandomMarkovState] = None
    noise_schedule: NoiseScheduler = None
    model_output_transform: DiffusionPredictionTransform = None
    autoencoder: Any = None
    input_config: DiffusionInputConfig = None
    samplers: Dict[Type[DiffusionSampler], Dict[float, DiffusionSampler]] = field(default_factory=dict)
    config: Dict[str, Any] = field(default_factory=dict)
    # id(tree) -> (tree, its FlatParams); the tree is kept so that its id cannot be reused by another object
    _packed: Dict[int, Tuple[Any, Any]] = field(default_factory=dict, repr=False)

    @classmethod
    def from_wandb_run(cls, wandb_run: str, project: str, entity: str):
        """Raises `FdxError`: wandb is not a dependency here; use `from_checkpoint`."""
        load_from_wandb_run(wandb_run, project=project, entity=entity)

    @classmethod
    def from_wandb_registry(cls, modelname: str, project: str, entity: str = None, version: str = 'latest',
                            registry: str = 'wandb-registry-model'):
        """Raises `FdxError`: wandb is not a dependency here; use `from_checkpoint`."""
        load_from_wandb_registry(modelname=modelname, project=project, entity=entity, version=version,
                                 registry=registry)

    @classmethod
    def from_checkpoint(cls, checkpoint_dir: str, config, step: Optional[int] = None,
                        input_config: Optional[DiffusionInputConfig] = None):
        """A pipeline from a local checkpoint directory and the run's config - the stand-in for `from_wandb_run`.

        `checkpoint_dir` holds `<step>/default/checkpoint` as `GeneralDiffusionTrainer.save` and the reference's
        trainer write it; `step=None` takes the latest.  `config` is the run config (training.py's `CONFIG`) as a
        dict or the path of a JSON file.  A non-None `input_config` replaces `config["input_config"]` and is used as
        is: it is the way to hand over encoders that cannot be rebuilt from a model name, such as an injected text
        tower.  The parameter trees stay on the host until a call samples from them."""
        if not isinstance(config, dict):
            with open(config) as f:
                config = json.load(f)
        _, tree = ckpt_io.load_tree(checkpoint_dir, step)
        if input_config is not None:
            config = {**config, "input_config": input_config}
        parsed = parse_config(config)

        def unwrap(st):
            # {step, params: {params: tree}, ema_params, opt_state, ...} -> the two trees generate_samples reads
            if st is None:
                return None
            return {"step": st.get("step"), "params": st["params"], "ema_params": st["ema_params"]}
        return cls.create(config=parsed, state=unwrap(tree["state"]), best_state=unwrap(tree.get("best_state")))

    @classmethod
    def create(cls, config: Dict[str, Any], state: Dict[str, Any], best_state: Optional[Dict[str, Any]] = None,
               rngstate: Optional[RandomMarkovState] = None, run=None, artifact=None):
        if rngstate is None:
            rngstate = RandomMarkovState(utils.PRNGKey(42))
        return cls(name=run.name if run else None, artifact=artifact, model=config['model'], state=state,
                   best_state=best_state, rngstate=rngstate, noise_schedule=config['noise_schedule'],
                   model_output_transform=config['prediction_transform'], autoencoder=config['autoencoder'],
                   input_config=config['input_config'], config=config)

    def get_sampler(self, guidance_scale: float = 3.0, sampler_class=EulerAncestralSampler) -> DiffusionSampler:
        """The sampler for (sampler_class, guidance_scale), built on first use and cached: its captured graphs
        and packed parameters are reused by later calls."""
        by_scale = self.samplers.setdefault(sampler_class, {})
        if guidance_scale not in by_scale:
            by_scale[guidance_scale] = sampler_class(model=self.model, noise_schedule=self.noise_schedule,
                                                     model_output_transform=self.model_output_transform,
                                                     guidance_scale=guidance_scale, input_config=self.input_config,
                                                     autoencoder=self.autoencoder)
        return by_scale[guidance_scale]

    def _flat(self, tree):
        """`tree` packed into FlatParams on the GPU, once per tree: every sampler of the pipeline then reads the same
        buffers, and its captured graphs stay valid from call to call."""
        hit = self._packed.get(id(tree))
        if hit is None or hit[0] is not tree:
            hit = (tree, self.model._as_flat(tree, torch.device("cuda")))
            self._packed[id(tree)] = hit
        return hit[1]

    def generate_samples(self, num_samples: int, resolution: int,
                         conditioning_data: List[Union[Tuple, Dict]] = None, conditioning_data_tokens: Tuple = None,
                         sequence_length: Optional[int] = None, diffusion_steps: int = 50,
                         guidance_scale: float = 1.0, sampler_class=EulerAncestralSampler,
                         timestep_spacing: str = 'linear', seed: Optional[int] = None, start_step: Optional[int] = None,
                         end_step: int = 0, steps_override=None, priors=None, use_best_params: bool = False,
                         use_ema: bool = False):
        """Images (num_samples, resolution, resolution, 3) in [-1, 1].  `conditioning_data`: raw inputs, one per
        sample (prompts; tuples / dicts for several conditions), encoded by the input config's encoders;
        `conditioning_data_tokens`: the embeddings themselves (the sampler's `model_conditioning_inputs`)."""
        rngstate = self.rngstate or RandomMarkovState(utils.PRNGKey(seed or 0))
        sampler = self.get_sampler(guidance_scale=guidance_scale, sampler_class=sampler_class)
        if hasattr(sampler, 'timestep_spacing'):
            sampler.timestep_spacing = timestep_spacing
        state = self.best_state if use_best_params else self.state
        params = self._flat(state['ema_params'] if use_ema else state['params'])
        return sampler.generate_samples(params=params, num_samples=num_samples, resolution=resolution,
                                        sequence_length=sequence_length, diffusion_steps=diffusion_steps,
                                        start_step=start_step, end_step=end_step, steps_override=steps_override,
                                        priors=priors, rngstate=rngstate, conditioning=conditioning_data,
                                        model_conditioning_inputs=conditioning_data_tokens)
