"""`DiffusionSampler` - the iterative denoising loop (API of flaxdiff/samplers/common.py:23-439).

What is kept from the reference: constructor and `generate_samples` / `sample_step` /
`take_next_step` / `get_steps` / `scale_steps` signatures, the timestep spacing rules (integer,
bit-exact), classifier-free-guidance batching, the "last step returns x0" rule, the initial-noise
scaling and the final clip.

What is different (GPU-first): the reference jits only `sample_model` and runs every update
rule as dozens of un-jitted XLA dispatches (SURVEY.md $3.2).  Here one denoise evaluation
(rates -> c_in scaling -> UNet -> x0/eps recovery) is captured ONCE in a CUDA graph per
(shape, params) and replayed per step, and every update rule is a single `fdx_affine_combine`
launch with per-sample coefficients computed from the schedule.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Tuple

import numpy as np
import torch

from .. import ops, utils
from .._lib import FdxError
from ..predictors import DiffusionPredictionTransform, _affine, _vec
from ..schedulers import NoiseScheduler
from ..utils import RandomMarkovState


def linspace_int16(start, stop, num: int) -> np.ndarray:
    """jnp.linspace(start, stop, num, dtype=int16): float32 lerp a*(1-s)+b*s with s=i/(num-1),
    exact endpoint, floor, cast (SURVEY.md Appendix B)."""
    start, stop = np.float32(start), np.float32(stop)
    if num == 1:
        out = np.asarray([start], dtype=np.float32)
    else:
        div = np.float32(num - 1)
        s = np.arange(num - 1, dtype=np.float32) / div
        body = (start * (np.float32(1.0) - s) + stop * s).astype(np.float32)
        out = np.concatenate([body, np.asarray([stop], dtype=np.float32)])
    return np.floor(out).astype(np.int16)


class _GraphedEval:
    """Capture `fn(*tensors) -> tuple(tensors)` once, replay with copied-in inputs."""

    def __init__(self, fn, example_inputs):
        self.static_in = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):                      # warm-up (lazy inits, func attributes)
                fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        # thread-local capture mode: a data-loading / prefetch thread may call the CUDA API meanwhile
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.static_out = fn(*self.static_in)

    def __call__(self, *inputs, clone: bool = True):
        for s, t in zip(self.static_in, inputs):
            if s.data_ptr() != t.data_ptr():
                s.copy_(t)
        self.graph.replay()
        if not clone:                        # valid until the next replay (stream-ordered consumers only)
            return self.static_out if isinstance(self.static_out, tuple) else (self.static_out,)
        outs = self.static_out if isinstance(self.static_out, tuple) else (self.static_out,)
        return tuple(o.clone() for o in outs)


class _DeviceKeyState:
    """The RandomMarkovState a whole-step capture hands to `take_next_step`: every subkey it gives out is the key
    held in `words` (a (2,) int32 device tensor) at replay time.  One draw per step (see _noise_per_step)."""

    def __init__(self, words: torch.Tensor):
        self.words = words

    def get_random_key(self):
        return self, utils.DeviceKey(self.words)


class DiffusionSampler:
    def __init__(self, model, noise_schedule: NoiseScheduler,
                 model_output_transform: DiffusionPredictionTransform, input_config=None,
                 guidance_scale: float = 0.0, autoencoder=None, timestep_spacing: str = 'linear',
                 use_cuda_graph: bool = True):
        self.model = model
        self.noise_schedule = noise_schedule
        self.model_output_transform = model_output_transform
        self.guidance_scale = guidance_scale
        self.autoencoder = autoencoder
        self.timestep_spacing = timestep_spacing
        self.input_config = input_config
        self.use_cuda_graph = use_cuda_graph
        if autoencoder is not None:
            raise FdxError("latent diffusion (autoencoder) is outside the supported hot path")
        self._unconditionals = input_config.get_unconditionals() if input_config is not None else []
        if hasattr(noise_schedule, 'min_inv_rho') and hasattr(noise_schedule, 'max_inv_rho'):
            self.min_inv_rho = noise_schedule.min_inv_rho
            self.max_inv_rho = noise_schedule.max_inv_rho
        # bounded caches (LRU): captured denoise-evaluation graphs and flax-tree -> FlatParams conversions
        self._graphs: "OrderedDict[tuple, _GraphedEval]" = OrderedDict()
        self._trees: "OrderedDict[int, tuple]" = OrderedDict()

    # ------------------------------------------------------------------ one model evaluation
    def _eval(self, fp, x_t: torch.Tensor, t: torch.Tensor, *conditioning):
        """(x0, eps, model_output) for samples x_t at per-sample steps t (samplers/common.py:70-109)."""
        sched, tr = self.noise_schedule, self.model_output_transform
        B = x_t.shape[0]
        g = float(self.guidance_scale)
        rates = sched.get_rates(t)
        c_in = tr.get_input_scale(rates)
        cvec = _vec(c_in.reshape(-1) if isinstance(c_in, torch.Tensor) else c_in, B, x_t.device)
        _, t_model = sched.transform_inputs(None, t)
        ones = torch.ones((1, B), dtype=torch.float32, device=x_t.device)
        _, _, xin = ops.affine_combine([x_t], ones, want_out1=False, bf16_scale=cvec, want_bf16=True)
        p, q, r, u = tr.x0_eps_coeffs(rates)
        if g > 0:
            conds = []
            for c, unc in zip(conditioning, self._unconditionals):
                conds.append(torch.cat([c, unc.to(c.device).expand_as(c)], dim=0))
            xin2 = torch.cat([xin, xin], dim=0)
            t2 = torch.cat([t_model, t_model], dim=0)
            F2, _ = self.model.forward(fp, xin2, t2, *(conds or [None]), save=False)
            Fc, Fu = F2[:B].contiguous(), F2[B:].contiguous()
            # model_output = Fu + g (Fc - Fu); x0 = p x + q F ; eps = r x + u F  -> one pass
            z = torch.zeros_like(p)
            (x0, eps) = _affine([x_t, Fc, Fu], [p, q * g, q * (1 - g)], [r, u * g, u * (1 - g)])
            Fm = _affine([x_t, Fc, Fu], [z, z + g, z + (1 - g)])
            return x0, eps, Fm
        ctx = conditioning[0] if conditioning else None
        Fm, _ = self.model.forward(fp, xin, t_model, ctx, save=False)
        x0, eps = _affine([x_t, Fm], [p, q], [r, u])
        return x0, eps, Fm

    # Deterministic single-launch update rules (Euler, Heun, DDIM eta=0, ...) set this: generate_samples then
    # captures the WHOLE step - model evaluation(s) + the (B,)-sized coefficient algebra + the update kernel -
    # in one CUDA graph with (x, current_step, next_step) as inputs, so a denoise step is one replay instead
    # of a replay plus ~30 tiny un-graphed launches (the reference runs them as un-jitted XLA dispatches,
    # SURVEY.md $3.2).  Samplers that keep Python-side history use the per-evaluation graph.
    _whole_step_graph = False
    # Update rules that draw exactly one noise tensor per step (EulerAncestral, DDPM, SimpleDDPM, DDIM eta>0) set
    # this.  With a `utils.ThreefryKey` in the RandomMarkovState they take the whole-step graph too: the noise is
    # an fdx_random_normal launch inside the graph that reads its key from 8 bytes of device memory; the host runs
    # the `split` chain of the eager steps ahead of the loop and each replay is handed its subkey.  A plain
    # tuple key draws from a torch.Generator, which a graph cannot re-seed: per-evaluation graph, as before.
    _noise_per_step = False
    MAX_GRAPHS = 4      # captured graphs kept per sampler (each owns a private memory pool)
    MAX_TREES = 2       # flax-tree -> FlatParams conversions kept per sampler

    def _flat_for(self, params, device):
        """FlatParams for `params`.  A plain flax tree is packed ONCE and remembered by identity (the tree is
        kept alive so its id cannot be recycled; flax trees are immutable by convention): calling
        sample_model / generate_samples repeatedly with the same tree neither re-packs nor re-captures."""
        from ..models.params import FlatParams
        if isinstance(params, FlatParams):
            return params
        hit = self._trees.get(id(params))
        if hit is not None and hit[0] is params:
            self._trees.move_to_end(id(params))
            return hit[1]
        fp = self.model._as_flat(params, device)
        self._trees[id(params)] = (params, fp)
        while len(self._trees) > self.MAX_TREES:
            self._trees.popitem(last=False)
        return fp

    def sample_model(self, params, x_t, t, *conditioning_inputs):
        fp = self._flat_for(params, x_t.device)
        t = torch.as_tensor(t, device=x_t.device)
        if t.dim() == 0:
            t = t.expand(x_t.shape[0])
        t = t.contiguous()
        if not self.use_cuda_graph or torch.cuda.is_current_stream_capturing():
            return self._eval(fp, x_t, t, *conditioning_inputs)      # (inside a whole-step capture: inline)
        # The graph reads the parameters through fp's bf16 shadow / f32 buffers BY POINTER, so new parameter
        # VALUES (training steps, EMA updates, checkpoint loads) need no re-capture: the shadow is re-cast
        # here when fp's generation moved (FlatParams.gen - torch's version counter does not see libfdx
        # writes).  Conditioning tensors are copied into static graph inputs, so fresh tensors of the same
        # shape reuse the graph.
        key = (id(fp), tuple(x_t.shape), t.dtype, tuple((tuple(c.shape), c.dtype) for c in conditioning_inputs))
        ge = self._graphs.get(key)
        fp.shadow()
        if ge is None:
            ge = _GraphedEval(lambda a, b, *conds: self._eval(fp, a, b, *conds), [x_t, t, *conditioning_inputs])
            self._graphs[key] = ge
            while len(self._graphs) > self.MAX_GRAPHS:
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(key)
        return ge(x_t, t, *conditioning_inputs)

    def _graphed_step(self, fp, x, cur, nxt, conds, key_words=None):
        """One full sampler step through a captured graph (see _whole_step_graph).  `key_words`: the subkey this
        step's noise is drawn from, as a (2,) int32 device tensor (see _noise_per_step); None for a deterministic
        update rule."""
        keyed = [] if key_words is None else [key_words]
        key = ("step", id(fp), tuple(x.shape), len(keyed), tuple((tuple(c.shape), c.dtype) for c in conds))
        ge = self._graphs.get(key)
        fp.shadow()
        if ge is None:
            def fn(a, c, n, *rest):
                def smf(x_t, t, *add):
                    return self.sample_model(fp, x_t, t, *add)
                state, cc = (_DeviceKeyState(rest[0]), rest[1:]) if keyed else (None, rest)
                out, _ = self.sample_step(smf, a, c, list(cc), next_step=n, state=state)
                return out
            ge = _GraphedEval(fn, [x, cur, nxt, *keyed, *conds])
            self._graphs[key] = ge
            while len(self._graphs) > self.MAX_GRAPHS:
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(key)
        return ge(x, cur, nxt, *keyed, *conds, clone=False)[0]

    def post_process(self, samples: torch.Tensor) -> torch.Tensor:
        ones = torch.ones((1, samples.shape[0]), dtype=torch.float32, device=samples.device)
        out, _, _ = ops.affine_combine([samples.contiguous()], ones, clip=(-1.0, 1.0))
        return out

    # ------------------------------------------------------------------ stepping
    def sample_step(self, sample_model_fn, current_samples, current_step, model_conditioning_inputs,
                    next_step=None, state: RandomMarkovState = None):
        B = current_samples.shape[0]
        dev = current_samples.device
        cur = torch.as_tensor(current_step, device=dev).expand(B) if not (
            isinstance(current_step, torch.Tensor) and current_step.dim() == 1) else current_step
        nxt = torch.as_tensor(next_step, device=dev).expand(B) if not (
            isinstance(next_step, torch.Tensor) and next_step.dim() == 1) else next_step
        pred_images, pred_noise, _ = sample_model_fn(current_samples, cur, *model_conditioning_inputs)
        return self.take_next_step(current_samples=current_samples, reconstructed_samples=pred_images,
                                   pred_noise=pred_noise, current_step=cur, next_step=nxt, state=state,
                                   model_conditioning_inputs=model_conditioning_inputs,
                                   sample_model_fn=sample_model_fn)

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        raise NotImplementedError("Subclasses must implement take_next_step method")

    def scale_steps(self, steps):
        return steps * (self.noise_schedule.max_timesteps / 1000)

    def get_steps(self, start_step, end_step, diffusion_steps) -> np.ndarray:
        """Integer timestep sequence (samplers/common.py:190-251); int16, bit-exact."""
        step_range = start_step - end_step
        if diffusion_steps is None or diffusion_steps == 0:
            diffusion_steps = step_range
        diffusion_steps = int(min(diffusion_steps, step_range))
        spacing = getattr(self, 'timestep_spacing', 'linear')
        f32 = np.float32
        if spacing == 'quadratic':
            u = (np.linspace(0, 1, diffusion_steps, dtype=f32) ** 2).astype(f32)
            steps = (f32(start_step - end_step) * u + f32(end_step)).astype(f32)
            return steps.astype(np.int16)[::-1].copy()
        if spacing == 'karras':
            rho = 7.0
            # end_step = 0 makes sigma_min = 0 and log(0) = -inf: the reference's sequence degenerates to NaN ->
            # int16 0 for every entry but the first product (samplers/common.py:213-228); reproduced as is
            with np.errstate(invalid='ignore', divide='ignore'):
                sig = np.exp(np.linspace(np.log(f32(1.0)), np.log(f32(end_step / start_step)) if end_step > 0
                                         else f32(-np.inf), diffusion_steps, dtype=f32)).astype(f32)
                steps = np.clip((sig ** f32(1 / rho) - f32(self.min_inv_rho)) /
                                f32(self.max_inv_rho - self.min_inv_rho), 0, 1) * f32(start_step)
                steps = np.where(np.isfinite(steps), steps, f32(0.0))
            return steps.astype(np.int16)
        if spacing == 'exponential':
            u = np.linspace(0, 1, diffusion_steps, dtype=f32)
            steps = np.exp(u * np.log(f32((start_step + 1) / (end_step + 1)))) * f32(end_step + 1) - 1
            steps = np.clip(steps, end_step, start_step)
            return steps.astype(np.int16)[::-1].copy()
        return linspace_int16(end_step, start_step, diffusion_steps)[::-1].copy()

    # ------------------------------------------------------------------ the loop
    def generate_samples(self, params, num_samples: int, resolution: int, sequence_length: int = None,
                         diffusion_steps: int = 1000, start_step: int = None, end_step: int = 0,
                         steps_override=None, priors=None, rngstate: RandomMarkovState = None,
                         conditioning=None, model_conditioning_inputs: Tuple = None, device=None):
        """`conditioning`: raw inputs (e.g. prompts), one entry per sample, encoded here by the encoders of
        `input_config` (see _encode_conditioning); `model_conditioning_inputs`: the embeddings themselves.  At most
        one of the two may be given."""
        if sequence_length is not None:
            raise FdxError("video sampling (sequence_length) is outside the supported hot path")
        B = num_samples if priors is None else int(priors.shape[0])
        if conditioning is not None:
            if self.input_config is None or not self.input_config.conditions:
                raise FdxError("raw conditioning needs an encoder: this sampler's input_config has no conditions; "
                               "pass model_conditioning_inputs (embeddings)")
            if model_conditioning_inputs is not None:
                raise ValueError("Cannot provide both conditioning and model_conditioning_inputs")
            if len(conditioning) != B:
                raise ValueError(f"conditioning has {len(conditioning)} entries for {B} samples: pass one entry per "
                                 "sample")
        device = torch.device(device) if device is not None else torch.device("cuda")
        if conditioning is not None:
            model_conditioning_inputs = self._encode_conditioning(conditioning, device)
        # The models read B (2 B with guidance) rows of every conditioning tensor, broadcasting only a batch of 1;
        # with guidance a batch of 1 would be paired with one null row, so there it must be B as well.
        for c in model_conditioning_inputs or ():
            if not (int(c.shape[0]) == B or (int(c.shape[0]) == 1 and self.guidance_scale <= 0)):
                raise ValueError(f"a conditioning input of batch {int(c.shape[0])} for {B} samples: its batch must be "
                                 f"the number of samples{'' if self.guidance_scale > 0 else ' or 1'}")
        if rngstate is None:
            rngstate = RandomMarkovState(utils.PRNGKey(42))
        if start_step is None:
            start_step = self.noise_schedule.max_timesteps
        if priors is None:
            rngstate, newrngs = rngstate.get_random_key()
            samples = self._get_initial_samples(resolution, num_samples, newrngs, start_step, device)
        else:
            samples = priors.to(device=device, dtype=torch.float32).contiguous()
        if model_conditioning_inputs is None:
            model_conditioning_inputs = []

        params = self._flat_for(params, device)        # a flax tree is packed once per call, not per step

        def sample_model_fn(x_t, t, *additional_inputs):
            return self.sample_model(params, x_t, t, *additional_inputs)

        steps = steps_override if steps_override is not None else self.get_steps(start_step, end_step, diffusion_steps)
        steps = [float(s) for s in np.asarray(steps).tolist()]
        n = len(steps)
        keyed = self._noise_per_step and isinstance(getattr(rngstate, "rng", None), utils.ThreefryKey)
        whole = self.use_cuda_graph and (self._whole_step_graph or keyed) and n > 1
        if whole:
            # per-step (B,) step tensors, built once: rows are views, no per-step fill kernels
            tab = torch.tensor([self.scale_steps(s) for s in steps] + [self.scale_steps(0)], dtype=torch.float32,
                               device=device).unsqueeze(1).expand(n + 1, samples.shape[0]).contiguous()
        if whole and keyed:
            # the subkeys of all steps, in one upload: row i is what step i's take_next_step would split off
            subkeys = []
            for _ in range(n - 1):
                rngstate, subkey = rngstate.get_random_key()
                subkeys.append(subkey)
            keytab = torch.from_numpy(np.asarray(subkeys, dtype=np.uint32).view(np.int32)).to(device)
        for i in range(n):
            current_step = self.scale_steps(steps[i])
            next_step = self.scale_steps(steps[i + 1] if i + 1 < n else 0)
            if i != n - 1 and whole:
                samples = self._graphed_step(params, samples, tab[i], tab[i + 1], tuple(model_conditioning_inputs),
                                             keytab[i] if keyed else None)
            elif i != n - 1:
                samples, rngstate = self.sample_step(sample_model_fn, samples, current_step,
                                                     model_conditioning_inputs, next_step=next_step, state=rngstate)
            else:
                cur = torch.full((samples.shape[0],), current_step, device=device)
                samples, _, _ = sample_model_fn(samples, cur, *model_conditioning_inputs)
        return self.post_process(samples)

    def _encode_conditioning(self, conditioning, device) -> tuple:
        """Raw conditioning -> one embedding per condition of `input_config` (samplers/common.py:315-349).  An entry
        that is a tuple or list is matched to the conditions by position, a dict by encoder key, anything else goes
        to every condition; each condition's encoder then encodes its whole list in one call."""
        conds = self.input_config.conditions
        separated = {c.encoder.key: [] for c in conds}
        for vals in conditioning:
            if isinstance(vals, (tuple, list)):
                for c, v in zip(conds, vals):
                    separated[c.encoder.key].append(v)
            elif isinstance(vals, dict):
                for c in conds:
                    if c.encoder.key not in vals:
                        raise ValueError(f"Conditioning input {c.encoder.key} not found in provided dictionary")
                    separated[c.encoder.key].append(vals[c.encoder.key])
            else:
                for c in conds:
                    separated[c.encoder.key].append(vals)
        # the engine's text tower returns bf16 on the device already; .to() is then the same tensor
        return tuple(c.encoder(separated[c.encoder.key]).to(device) for c in conds)

    def _get_noise_parameters(self, resolution, start_step, device):
        a, s = self.noise_schedule.get_rates(torch.as_tensor(self.scale_steps(start_step), device=device))
        return torch.sqrt(a ** 2 + s ** 2), resolution, 3

    def _get_initial_samples(self, resolution, batch_size, rngs, start_step, device):
        variance, size, ch = self._get_noise_parameters(resolution, start_step, device)
        noise = utils.device_normal(rngs, (batch_size, size, size, ch), device)
        return _affine([noise], [variance.reshape(-1)])

    generate_images = generate_samples
