"""Per-step update rules of the reference samplers, each as ONE affine-combine kernel launch.

  EulerSampler / SimplifiedEulerSampler / EulerAncestralSampler   flaxdiff/samplers/euler.py:6-56
  HeunSampler                                                      flaxdiff/samplers/heun_sampler.py:6-27
  DDIMSampler                                                      flaxdiff/samplers/ddim.py:7-49
  DDPMSampler / SimpleDDPMSampler                                  flaxdiff/samplers/ddpm.py:5-37
  RK4Sampler / MultiStepDPM                                        flaxdiff/samplers/{rk4_sampler,multistep_dpm}.py

The (B,)-sized coefficient algebra follows the reference expressions term by term; the
image-sized arithmetic is the libfdx kernel.
"""
from __future__ import annotations

import torch

from .. import utils
from .._lib import FdxError
from ..predictors import _affine
from ..schedulers import GeneralizedNoiseScheduler
from ..utils import RandomMarkovState
from .base import DiffusionSampler


def _rates(schedule, step):
    a, s = schedule.get_rates(step, shape=(-1,))
    return a.to(torch.float32), s.to(torch.float32)


class EulerSampler(DiffusionSampler):
    _whole_step_graph = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        ca, cs = _rates(self.noise_schedule, current_step)
        na, ns = _rates(self.noise_schedule, next_step)
        dt = ns - cs
        k = (ca * ns - na * cs) / dt
        # x + (x - k x0) / cs * dt
        g = dt / cs
        return _affine([current_samples, reconstructed_samples], [1 + g, -k * g]), state


class SimplifiedEulerSampler(DiffusionSampler):
    _whole_step_graph = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        _, cs = _rates(self.noise_schedule, current_step)
        _, ns = _rates(self.noise_schedule, next_step)
        g = (ns - cs) / cs
        return _affine([current_samples, reconstructed_samples], [1 + g, -g]), state


class EulerAncestralSampler(DiffusionSampler):
    _noise_per_step = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        ca, cs = _rates(self.noise_schedule, current_step)
        na, ns = _rates(self.noise_schedule, next_step)
        sigma_up = (ns ** 2 * (cs ** 2 - ns ** 2) / cs ** 2) ** 0.5
        sigma_down = (ns ** 2 - sigma_up ** 2) ** 0.5
        dt = sigma_down - cs
        k = (ca * ns - na * cs) / (ns - cs)
        state, subkey = state.get_random_key()
        noise = utils.device_normal(subkey, tuple(current_samples.shape), current_samples.device)
        g = dt / cs
        return _affine([current_samples, reconstructed_samples, noise], [1 + g, -k * g, sigma_up]), state


class HeunSampler(DiffusionSampler):
    _whole_step_graph = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        ca, cs = _rates(self.noise_schedule, current_step)
        na, ns = _rates(self.noise_schedule, next_step)
        dt = ns - cs
        k = (ca * ns - na * cs) / dt
        g0 = dt / cs
        x_pred = _affine([current_samples, reconstructed_samples], [1 + g0, -k * g0])
        est_x0, _, _ = sample_model_fn(x_pred, next_step, *model_conditioning_inputs)
        # x + 0.5 (dx0 + dx1) dt ; dx0 = (x - k x0)/cs ; dx1 = (x' - k x0')/ns
        h0, h1 = 0.5 * dt / cs, 0.5 * dt / ns
        out = _affine([current_samples, reconstructed_samples, x_pred, est_x0], [1 + h0, -k * h0, h1, -k * h1])
        return out, state


class DDIMSampler(DiffusionSampler):
    def __init__(self, *args, eta=0.0, **kwargs):
        super().__init__(*args, **kwargs)
        self.eta = eta
        self._whole_step_graph = (eta == 0)
        self._noise_per_step = (eta > 0)

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        at, st = _rates(self.noise_schedule, current_step)
        an, sn = _rates(self.noise_schedule, next_step)
        if self.eta > 0:
            # the reference calls .sqrt() on a jnp array here and would raise (SURVEY.md A.7);
            # the evident DDIM formula is implemented
            sigma_tilde = self.eta * sn * torch.sqrt(1 - at ** 2 / an ** 2) / torch.sqrt(1 - at ** 2)
            state, key = state.get_random_key()
            noise = utils.device_normal(key, tuple(current_samples.shape), current_samples.device)
            return _affine([reconstructed_samples, pred_noise, noise], [an, sn, sigma_tilde]), state
        return _affine([reconstructed_samples, pred_noise], [an, sn]), state


class DDPMSampler(DiffusionSampler):
    _noise_per_step = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        c0, ct = self.noise_schedule.get_posterior_coeffs(current_step)
        std = self.noise_schedule.get_posterior_variance(steps=current_step, shape=(-1,))
        state, rng = state.get_random_key()
        noise = utils.device_normal(rng, tuple(reconstructed_samples.shape), reconstructed_samples.device)
        return _affine([reconstructed_samples, current_samples, noise], [c0, ct, std]), state

    def generate_images(self, num_images=16, diffusion_steps=1000, start_step: int = None, *args, **kwargs):
        # reference forwards a `num_images` kwarg the base does not accept (SURVEY.md A.6): alias it
        return super().generate_samples(*args, num_samples=num_images, diffusion_steps=diffusion_steps,
                                        start_step=start_step, **kwargs)


class SimpleDDPMSampler(DiffusionSampler):
    _noise_per_step = True

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        state, rng = state.get_random_key()
        noise = utils.device_normal(rng, tuple(reconstructed_samples.shape), reconstructed_samples.device)
        ca, cs = _rates(self.noise_schedule, current_step)
        na, ns = _rates(self.noise_schedule, next_step)
        pred_noise_coeff = ((ns ** 2) * ca) / (cs * na)
        gamma = torch.sqrt(((ns ** 2) / (cs ** 2)) * (1 - (ca ** 2) / (na ** 2)))
        return _affine([reconstructed_samples, pred_noise, noise], [na, pred_noise_coeff, gamma]), state


class RK4Sampler(DiffusionSampler):
    """4th-order Runge-Kutta on d x / d sigma = eps (rk4_sampler.py:7-33).  The reference jits a
    function taking a Python callable and is broken as written (SURVEY.md A.8); the evident
    algorithm is implemented."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if not isinstance(self.noise_schedule, GeneralizedNoiseScheduler):
            raise FdxError("Noise schedule must be a GeneralizedNoiseScheduler")

    def _deriv(self, sample_model_fn, x_t, sigma, conds):
        t = self.noise_schedule.get_timesteps(sigma)
        _, eps, _ = sample_model_fn(x_t, t, *conds)
        return eps

    def sample_step(self, sample_model_fn, current_samples, current_step, model_conditioning_inputs,
                    next_step=None, state=None):
        B, dev = current_samples.shape[0], current_samples.device
        cur = torch.as_tensor(current_step, device=dev, dtype=torch.float32).expand(B)
        nxt = torch.as_tensor(next_step, device=dev, dtype=torch.float32).expand(B)
        _, cs = _rates(self.noise_schedule, cur)
        _, ns = _rates(self.noise_schedule, nxt)
        dt = ns - cs
        x = current_samples
        k1 = self._deriv(sample_model_fn, x, cs, model_conditioning_inputs)
        k2 = self._deriv(sample_model_fn, _affine([x, k1], [1.0, 0.5 * dt]), cs + 0.5 * dt, model_conditioning_inputs)
        k3 = self._deriv(sample_model_fn, _affine([x, k2], [1.0, 0.5 * dt]), cs + 0.5 * dt, model_conditioning_inputs)
        k4 = self._deriv(sample_model_fn, _affine([x, k3], [1.0, dt]), cs + dt, model_conditioning_inputs)
        return _affine([x, k1, k2, k3, k4], [1.0, dt / 6, dt / 3, dt / 3, dt / 6]), state


class MultiStepDPM(DiffusionSampler):
    """Finite-difference multistep on eps history (multistep_dpm.py:6-58)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.history = []

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state: RandomMarkovState, sample_model_fn, next_step=1):
        _, cs = _rates(self.noise_schedule, current_step)
        _, ns = _rates(self.noise_schedule, next_step)
        dt = ns - cs
        hist = self.history
        if len(hist) == 0:
            out = _affine([current_samples, pred_noise], [1.0, dt])
        elif len(hist) == 1:
            l = hist[-1]
            c2 = 0.5 * dt ** 2 / (cs - l['sigma'])
            out = _affine([current_samples, pred_noise, l['eps']], [1.0, dt + c2, -c2])
        else:
            l, m = hist[-1], hist[-2]
            d1, d0 = cs - l['sigma'], l['sigma'] - m['sigma']
            c2 = 0.5 * dt ** 2
            c3 = (1 / 6) * dt ** 3 / (0.5 * ((cs + l['sigma']) - (l['sigma'] + m['sigma'])))
            # dx2 = (e - el)/d1 ; dx2_last = (el - em)/d0 ; dx3 = (dx2 - dx2_last)/(...)
            ce = dt + c2 / d1 + c3 / d1
            cl = -c2 / d1 - c3 / d1 - c3 / d0
            cm = c3 / d0
            out = _affine([current_samples, pred_noise, l['eps'], m['eps']], [1.0, ce, cl, cm])
        self.history.append({"eps": pred_noise, "sigma": cs})
        return out, state
