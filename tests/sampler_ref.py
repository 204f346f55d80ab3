"""Float64 restatement of the reference's sampler update rules and prediction transforms, unfused, with a
per-element error bound; and an analytic stand-in denoiser the samplers accept in place of a UNet.

The rules are written the way flaxdiff/samplers/{euler,heun_sampler,ddim,ddpm,rk4_sampler,multistep_dpm}.py and
flaxdiff/predictors/__init__.py state them (dx, dx_2, dx_3, x_0_coeff, sigma_up / sigma_down, posterior mean and
std, the RK4 stages, x0 / eps recovery after pred_transform, CFG as Fu + g (Fc - Fu)), not in the fused
coefficients of flaxdiff_b200/samplers/steps.py: the two paths are independent.

Every quantity is a `V`: its float64 value `v` and two bounds that build the per-element tolerance.
  * `m`, the rounding magnitude: the same expression evaluated on absolute values with every subtraction turned
    into an addition.  The device computes each rule as one `fdx_affine_combine` launch whose coefficients are
    the reference expression with its products distributed over its sums; that has the same monomials, so each
    monomial carries at most n roundings (n = every f32 operation on the device's path: the (B,)-sized
    coefficient algebra in torch plus the kernel's multiply-adds) and the rounding error is at most gamma(n) m
    (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Lemma 3.3).  A quotient by a computed
    quantity b adds b's relative rounding, m_b / |b| (first order): this is what makes the cancellation in
    dt = ns - cs, in k = (ca ns - na cs) / dt and in MultiStepDPM's differences visible.
  * `e`, the propagated error of inexact inputs (the stand-in's f32 output, the device's threefry normal draws),
    first order.
  bound = gamma(n) m + e.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from elementwise_ref import U32, assert_elementwise, gamma
from flaxdiff_b200.samplers import HeunSampler, MultiStepDPM
from flaxdiff_b200.samplers import steps as _steps
from flaxdiff_b200.schedulers import KarrasVENoiseScheduler

F64 = torch.float64
# the device's threefry normal draw and the host restatement `utils.normal_f32` are each within 6 ulp (uniform in
# [-0.9, 0.9]) or 98 ulp (tails) of float64 sqrt(2) erfinv of the same uniform (tests/test_prng_streams_gpu.py)
NORMAL_ULP_CENTRAL, NORMAL_ULP_TAIL = 6.0, 98.0


class V:
    __slots__ = ("v", "m", "e")

    def __init__(self, v, m=None, e=None):
        self.v = torch.as_tensor(v, dtype=F64)
        self.m = self.v.abs() if m is None else m
        self.e = torch.zeros_like(self.v) if e is None else e

    @staticmethod
    def of(x):
        return x if isinstance(x, V) else V(x)

    def __add__(self, o):
        o = V.of(o)
        return V(self.v + o.v, self.m + o.m, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = V.of(o)
        return V(self.v - o.v, self.m + o.m, self.e + o.e)

    def __rsub__(self, o):
        return V.of(o) - self

    def __neg__(self):
        return V(-self.v, self.m, self.e)

    def __mul__(self, o):
        o = V.of(o)
        return V(self.v * o.v, self.m * o.m, self.e * o.v.abs() + self.v.abs() * o.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = V.of(o)
        q = self.v / o.v
        b = o.v.abs()
        return V(q, self.m / b + q.abs() * o.m / b, self.e / b + q.abs() * o.e / b)

    def __rtruediv__(self, o):
        return V.of(o) / self

    def sq(self):
        return self * self

    def sqrt(self):
        r = torch.sqrt(self.v)
        pos = r > 0                     # an exact zero (ns = 0 at sigma(0) = 0) stays an exact zero
        return V(r, r + torch.where(pos, self.m / (2 * r), 0.0), torch.where(pos, self.e / (2 * r), 0.0))

    def exp(self):
        r = torch.exp(self.v)
        return V(r, r * (2 + self.m), r * self.e)          # expf: 2 ulp, counted as 2 of the n roundings

    def bound(self, n):
        return gamma(n) * self.m + self.e


def t64(x, shape=(-1, 1, 1, 1)):
    return torch.as_tensor(x).detach().to("cpu", F64).reshape(shape)


# ------------------------------------------------------------------------------------------ prediction transforms
TRANSFORMS = ("eps", "x0", "v", "karras")


def input_scale(kind, s, sigma_data=0.5):
    """get_input_scale (predictors/__init__.py:93-96 for Karras, 1 otherwise)."""
    if kind != "karras":
        return V(torch.ones_like(V.of(s).v))
    return 1 / ((sigma_data ** 2 + V.of(s).sq()).sqrt() + 1e-8)


def x0_eps(kind, x, F, a, s, sigma_data=0.5):
    """pred_transform then backward_diffusion (predictors/__init__.py:13-17), term by term."""
    x, F, a, s = V.of(x), V.of(F), V.of(a), V.of(s)
    if kind == "karras":
        c_out = s * sigma_data / ((sigma_data ** 2 + s.sq()).sqrt() + 1e-8)
        c_skip = sigma_data ** 2 / (sigma_data ** 2 + s.sq() + 1e-8)
        F = c_out * F + c_skip * x
    if kind == "eps":
        return (x - F * s) / a, F
    if kind in ("x0", "karras"):
        return F, (x - F * a) / s
    variance = a.sq() + s.sq()
    vv = F * variance.sqrt()
    return (a * x - s * vv) / variance, (a * vv + s * x) / variance


def guided(Fc, Fu, g):
    """Classifier-free guidance (samplers/common.py:87-88)."""
    return Fu + g * (Fc - Fu)


# ------------------------------------------------------------------------------------------------- update rules
def euler(x, x0, ca, cs, na, ns):
    dt = ns - cs
    x_0_coeff = (ca * ns - na * cs) / dt
    dx = (x - x_0_coeff * x0) / cs
    return x + dx * dt


def simplified_euler(x, x0, cs, ns):
    dt = ns - cs
    dx = (x - x0) / cs
    return x + dx * dt


def euler_ancestral(x, x0, z, ca, cs, na, ns):
    sigma_up = (ns.sq() * (cs.sq() - ns.sq()) / cs.sq()).sqrt()
    sigma_down = (ns.sq() - sigma_up.sq()).sqrt()
    dt = sigma_down - cs
    x_0_coeff = (ca * ns - na * cs) / (ns - cs)
    dx = (x - x_0_coeff * x0) / cs
    return x + dx * dt + z * sigma_up


def heun_predict(x, x0, ca, cs, na, ns):
    """next_samples_0, the first estimate Heun evaluates the model at."""
    return euler(x, x0, ca, cs, na, ns)


def heun(x, x0, x_pred, x0_pred, ca, cs, na, ns):
    dt = ns - cs
    x_0_coeff = (ca * ns - na * cs) / dt
    dx_0 = (x - x_0_coeff * x0) / cs
    dx_1 = (x_pred - x_0_coeff * x0_pred) / ns
    return x + 0.5 * (dx_0 + dx_1) * dt


def ddim(x0, eps, at, an, sn, eta=0.0, z=None):
    out = an * x0 + sn * eps
    if eta > 0:
        # the reference calls .sqrt() on a jnp array here (ddim.py:38); its evident formula
        sigma_tilde = eta * sn * (1 - at.sq() / an.sq()).sqrt() / (1 - at.sq()).sqrt()
        out = out + sigma_tilde * z
    return out


def ddpm(x0, x, z, coef1, coef2, log_var):
    """posterior mean + noise * exp(0.5 log_var) (ddpm.py:8-15, discrete.py get_posterior_*)."""
    mean = coef1 * x0 + coef2 * x
    return mean + z * (0.5 * log_var).exp()


def simple_ddpm(x0, eps, z, ca, cs, na, ns):
    pred_noise_coeff = (ns.sq() * ca) / (cs * na)
    noise_ratio_squared = ns.sq() / cs.sq()
    signal_ratio_squared = ca.sq() / na.sq()
    gamma_ = (noise_ratio_squared * (1 - signal_ratio_squared)).sqrt()
    return na * x0 + pred_noise_coeff * eps + z * gamma_


def rk4_stage(x, k, dt, frac):
    """current_samples + frac * k * dt (frac = 0.5, 0.5, 1), evaluated at sigma = current_sigma + frac * dt."""
    return x + frac * k * dt


def rk4(x, k1, k2, k3, k4, dt):
    return x + (((k1 + 2 * k2 + 2 * k3 + k4) * dt) / 6)


def multistep_dpm(x, eps, cs, ns, history):
    """history: [{"eps": V, "sigma": V}, ...] of the earlier steps, oldest first (multistep_dpm.py:35-58)."""
    dt = ns - cs

    def second_order(e, s, le, ls):
        return (e - le) / (s - ls)

    if len(history) == 0:
        out = x + eps * dt
    elif len(history) == 1:
        last = history[-1]
        dx_2 = second_order(eps, cs, last["eps"], last["sigma"])
        out = x + eps * dt + 0.5 * dx_2 * dt.sq()
    else:
        last, second_last = history[-1], history[-2]
        dx_2 = second_order(eps, cs, last["eps"], last["sigma"])
        dx_2_last = second_order(last["eps"], last["sigma"], second_last["eps"], second_last["sigma"])
        dx_3 = (dx_2 - dx_2_last) / (0.5 * ((cs + last["sigma"]) - (last["sigma"] + second_last["sigma"])))
        out = x + (eps * dt) + (0.5 * dx_2 * dt.sq()) + ((1 / 6) * dx_3 * dt.sq() * dt)
    history.append({"eps": eps, "sigma": cs})
    return out


def initial_sample(z, a, s):
    """x_T = sqrt(alpha^2 + sigma^2) * noise (samplers/common.py _get_noise_parameters)."""
    return (a.sq() + s.sq()).sqrt() * z


def clip(x):
    """clip_images: clip to [-1, 1] (utils.py:101-112)."""
    return torch.clamp(torch.as_tensor(x, dtype=F64), -1.0, 1.0)


def noise_ref(key, shape):
    """The host restatement of jax.random.normal for `key` and its error against the device's draw."""
    from flaxdiff_b200 import utils
    n = int(np.prod(shape))
    z = torch.from_numpy(utils.normal_f32(key, n).astype(np.float64)).reshape(shape)
    uni = torch.from_numpy(utils.uniform(key, n, utils._NORMAL_LO, 1.0).astype(np.float64)).reshape(shape)
    ulps = torch.where(uni.abs() <= 0.9, 2 * NORMAL_ULP_CENTRAL, 2 * NORMAL_ULP_TAIL)
    return V(z, z.abs(), ulps * 2.0 ** -23 * z.abs())


# ---------------------------------------------------------------------------------- the analytic stand-in denoiser
def schedule_family(sched) -> str:
    from flaxdiff_b200 import schedulers as sc
    if isinstance(sched, sc.GeneralizedNoiseScheduler):
        return "ve"
    if isinstance(sched, sc.DiscreteNoiseScheduler):
        return "discrete"
    return "cosine_continuous"


def recovered_rates(family, t_model, tables=None):
    """(alpha, sigma) in float64 from the model time `transform_inputs` hands the model: sigma = exp(4 t) for the
    Karras / EDM model time log(sigma) / 4; the f32 tables at int16(t) (clamped as JAX gathers) for discrete
    schedules; cos / sin (pi t / 2) for the continuous cosine schedule."""
    t = t_model.to(F64)
    if family == "ve":
        return torch.ones_like(t), torch.exp(4 * t)
    if family == "discrete":
        sa, so = tables
        T = sa.shape[0]
        idx = torch.trunc(t).to(torch.int64)
        idx = torch.where(idx < 0, idx + T, idx).clamp(0, T - 1)
        return sa.to(t.device)[idx], so.to(t.device)[idx]
    return torch.cos(math.pi * t / 2), torch.sin(math.pi * t / 2)


def denoiser_output(kind, family, xin, t_model, mu, ctx=None, s_data=0.5, tables=None, sigma_data=0.5):
    """The raw model output F that prediction transform `kind` expects from the exact denoiser for Gaussian data
    x0 ~ N(mu, s_data^2) per element: D = E[x0 | x] = mu + alpha s^2 (x - alpha mu) / (alpha^2 s^2 + sigma^2),
    eps = E[eps | x] = sigma (x - alpha mu) / (alpha^2 s^2 + sigma^2).  x = xin / c_in, with (alpha, sigma)
    recovered from the model time.  A context shifts mu per sample.  Float64 throughout; returns (F, M), M a
    magnitude of the terms F is formed from (its float64 rounding error is far below 2^-40 M)."""
    B = xin.shape[0]
    a, s = (r.reshape(B, 1, 1, 1) for r in recovered_rates(family, t_model, tables))
    x = xin.to(F64)
    if kind == "karras":
        x = x * (torch.sqrt(sigma_data ** 2 + s * s) + 1e-8)
    m = mu.to(device=x.device, dtype=F64).expand_as(x)
    if ctx is not None:
        m = m + 0.25 * torch.tanh(ctx.to(F64).reshape(B, -1).mean(1)).reshape(B, 1, 1, 1)
    var = a * a * s_data ** 2 + s * s
    r = x - a * m
    D = m + a * s_data ** 2 * r / var
    E = s * r / var
    if kind == "x0":
        return D, m.abs() + D.abs()
    if kind == "eps":
        return E, E.abs()
    if kind == "v":
        n = torch.sqrt(a * a + s * s)
        return (a * E - s * D) / n, (a * E.abs() + s * D.abs()) / n
    c_skip = sigma_data ** 2 / (sigma_data ** 2 + s * s + 1e-8)
    c_out = s * sigma_data / (torch.sqrt(sigma_data ** 2 + s * s) + 1e-8)
    return (D - c_skip * x) / c_out, (D.abs() + (c_skip * x).abs()) / c_out


def model_output_ref(F, M):
    """The stand-in's f32 output as an inexact input: f32 rounding of F plus its float64 evaluation on either
    side (device and host)."""
    return V(F, F.abs(), U32 * F.abs() + 2.0 ** -40 * M)


class _Shadow:
    def shadow(self):
        return None


class GaussianDenoiser:
    """What `DiffusionSampler` asks of a model: `forward(fp, x_bf16, t_model, ctx, save=False) -> (F, None)` and
    `_as_flat(params, device)` with `shadow()`.  Pure torch on the device (float64, then f32), so both the
    per-evaluation and the whole-step CUDA graphs capture it.  Records each bf16 input, model time and context
    when `record` is set and no capture is running."""

    def __init__(self, kind, sched, mu, s_data=0.5, sigma_data=0.5):
        self.kind, self.family = kind, schedule_family(sched)
        self.mu, self.s_data, self.sigma_data = mu, s_data, sigma_data
        self.tables = None
        if self.family == "discrete":
            self.tables = tuple(torch.from_numpy(sched._np[n].astype(np.float64))
                                for n in ("sqrt_alpha_cumprod", "sqrt_one_minus_alpha_cumprod"))
        self.params = _Shadow()
        self.record = True
        self.log = []
        self._dev = {}

    def _as_flat(self, params, device):
        return self.params

    def _on(self, device):
        key = str(device)
        if key not in self._dev:
            self._dev[key] = (self.mu.to(device), None if self.tables is None else
                              tuple(t.to(device) for t in self.tables))
        return self._dev[key]

    def forward(self, fp, x, t, ctx=None, save=False):
        assert x.dtype == torch.bfloat16
        mu, tables = self._on(x.device)
        F, _ = denoiser_output(self.kind, self.family, x, t, mu, ctx, self.s_data, tables, self.sigma_data)
        if self.record and not (x.is_cuda and torch.cuda.is_current_stream_capturing()):
            self.log.append((x.clone(), t.clone(), None if ctx is None else ctx.clone()))
        return F.to(torch.float32).contiguous(), None

    def reference(self, xin, t_model, ctx):
        """F and M on the host for a recorded input."""
        return denoiser_output(self.kind, self.family, xin.cpu(), t_model.cpu(), self.mu.cpu(),
                               None if ctx is None else ctx.cpu(), self.s_data, self.tables, self.sigma_data)


# ----------------------------------------------------------------------------------------------- the step checker
RULES = ("euler", "simplified_euler", "euler_ancestral", "heun", "ddim", "ddim_eta", "ddpm", "simple_ddpm", "rk4",
         "multistep_dpm")
STOCHASTIC = ("euler_ancestral", "ddim_eta", "ddpm", "simple_ddpm")
# n for one model evaluation: the transform's (B,)-sized coefficients (Karras, the longest: c_out and c_skip, 10
# operations, composed into p, q, r, u, 6 more), the guidance fold q g, q (1 - g) (3) and the kernel's three
# multiply-adds, each counted as a product and a sum (6); rounded up
N_EVAL = 32
# n added by each update rule: its coefficient algebra plus two per kernel term, counted in steps.py; rounded up
N_RULE = {"euler": 16, "simplified_euler": 8, "euler_ancestral": 32, "heun": 24, "ddim": 4, "ddim_eta": 16,
          "ddpm": 12, "simple_ddpm": 20, "rk4": 16, "multistep_dpm": 32}
N_STAGE = 8


def _rows(v: V, sl):
    return V(v.v[sl], v.m[sl], v.e[sl])


class StepChecker:
    """Drives a sampler one step at a time through its public `sample_step` (eager, no CUDA graph) with a
    `GaussianDenoiser` as its model, and checks every model input, every intermediate stage and the step's
    output element by element against the float64 restatement, fed the device's own state."""

    def __init__(self, smp, model, rule, fp=None):
        assert not smp.use_cuda_graph
        self.smp, self.model, self.rule = smp, model, rule
        self.kind = model.kind
        self.fp = model.params if fp is None else fp
        self.g = float(smp.guidance_scale)
        self.history = []
        self.evals = []
        self.worst = 0.0
        inner = smp._eval

        def recording(fp_, x_t, t, *conds):
            self.evals.append((x_t.clone(), t.clone()))
            return inner(fp_, x_t, t, *conds)
        smp._eval = recording

    def _smf(self, x_t, t, *conds):
        return self.smp.sample_model(self.fp, x_t, t, *conds)

    def _rates(self, t):
        a, s = self.smp.noise_schedule.get_rates(t, shape=(-1,))
        return V(t64(a)), V(t64(s))

    def _check(self, got, ref: V, n, what):
        r = assert_elementwise(got.cpu(), ref.v, ref.bound(n), what)
        self.worst = max(self.worst, r)
        return r

    def _eval_ref(self, j):
        """(x0, eps) of evaluation j in float64, from the bf16 input the stand-in recorded; asserts that input is
        bf16(f32(x) f32(c_in)) of the x the sampler evaluated, bit for bit."""
        x_t, t = self.evals[j]
        xin, t_model, ctx = self.model.log[j]
        B = x_t.shape[0]
        sched, tr = self.smp.noise_schedule, self.smp.model_output_transform
        a32, s32 = sched.get_rates(t, shape=(-1,))
        c_in = tr.get_input_scale((a32, s32))
        c_in = torch.as_tensor(c_in, dtype=torch.float32).reshape(-1).expand(B).cpu()
        want = (x_t.cpu() * c_in.view(-1, 1, 1, 1)).to(torch.bfloat16)
        if self.g > 0:
            want = torch.cat([want, want])
        assert torch.equal(xin.cpu(), want), f"{self.rule}: evaluation {j}: the model input is not bf16(x c_in)"
        cref = input_scale(self.kind, V(t64(s32)))
        assert ((t64(c_in) - cref.v).abs() <= cref.bound(8)).all(), "c_in"
        F, M = self.model.reference(xin, t_model, ctx)
        Fv = model_output_ref(F, M)
        if self.g > 0:
            Fv = guided(_rows(Fv, slice(0, B)), _rows(Fv, slice(B, 2 * B)), self.g)
        x = V(t64(x_t, tuple(x_t.shape)))
        x0, eps = x0_eps(self.kind, x, Fv, V(t64(a32)), V(t64(s32)))
        return x, x0, eps, t

    def step(self, x, cur, nxt, conds=(), state=None):
        """One sampler step from the device state x; returns (x_next, state)."""
        B, dev = x.shape[0], x.device
        self.evals.clear()
        self.model.log.clear()
        cur_t = torch.full((B,), float(cur), device=dev)
        nxt_t = torch.full((B,), float(nxt), device=dev)
        z = None
        if self.rule in STOCHASTIC:
            _, subkey = state.get_random_key()
            z = noise_ref(subkey, tuple(x.shape))
        out, state = self.smp.sample_step(self._smf, x, cur_t, list(conds), next_step=nxt_t, state=state)
        assert len(self.model.log) == len(self.evals)
        ev = [self._eval_ref(j) for j in range(len(self.evals))]
        xv, x0, eps, _ = ev[0]
        ca, cs = self._rates(cur_t)
        na, ns = self._rates(nxt_t)
        r, n = self.rule, N_EVAL + N_RULE[self.rule]
        if r == "euler":
            ref = euler(xv, x0, ca, cs, na, ns)
        elif r == "simplified_euler":
            ref = simplified_euler(xv, x0, cs, ns)
        elif r == "euler_ancestral":
            ref = euler_ancestral(xv, x0, z, ca, cs, na, ns)
        elif r == "heun":
            assert len(ev) == 2 and torch.equal(ev[1][3], nxt_t)
            self._check(self.evals[1][0], heun_predict(xv, x0, ca, cs, na, ns), n, "heun: next_samples_0")
            ref = heun(xv, x0, ev[1][0], ev[1][1], ca, cs, na, ns)
        elif r in ("ddim", "ddim_eta"):
            ref = ddim(x0, eps, ca, na, ns, self.smp.eta, z)
        elif r == "ddpm":
            sched = self.smp.noise_schedule
            c1, c2 = (V(t64(c)) for c in sched.get_posterior_coeffs(cur_t))
            lv = V(t64(sched._gather("posterior_log_variance_clipped", cur_t)))
            ref = ddpm(x0, xv, z, c1, c2, lv)
        elif r == "simple_ddpm":
            ref = simple_ddpm(x0, eps, z, ca, cs, na, ns)
        elif r == "rk4":
            assert len(ev) == 4
            dt = ns - cs
            ks = [eps]
            for j, frac in ((1, 0.5), (2, 0.5), (3, 1)):
                self._check(self.evals[j][0], rk4_stage(xv, ks[-1], dt, frac), N_EVAL + N_STAGE, f"rk4: stage {j + 1}")
                sig = cs + frac * dt
                s_j = self._rates(self.evals[j][1])[1]
                # the stage's sigma goes through get_timesteps and get_rates (a pow round trip) before the model.
                # EDMNoiseScheduler inherits the Karras get_timesteps, as the reference's does (karras.py:65-77),
                # so there the model sees another sigma: pinned as is
                if type(self.smp.noise_schedule).get_sigmas is KarrasVENoiseScheduler.get_sigmas:
                    assert ((s_j.v - sig.v).abs() <= 2.0 ** -14 * sig.v.abs()).all(), f"rk4: stage {j + 1} sigma"
                ks.append(ev[j][2])
            ref = rk4(xv, *ks, dt)
        elif r == "multistep_dpm":
            ref = multistep_dpm(xv, eps, cs, ns, self.history)
        else:
            raise ValueError(r)
        self._check(out, ref, n, f"{r}: step {float(cur)} -> {float(nxt)}")
        return out, state

    def final(self, x, cur, conds=()):
        """The last step: x0 of the evaluation at `cur`, then post_process's clip."""
        B, dev = x.shape[0], x.device
        self.evals.clear()
        self.model.log.clear()
        x0_dev, _, _ = self._smf(x, torch.full((B,), float(cur), device=dev), *conds)
        _, x0, _, _ = self._eval_ref(0)
        self._check(x0_dev, x0, N_EVAL, f"x0 at the last step {float(cur)}")
        out = self.smp.post_process(x0_dev)
        assert torch.equal(out.cpu().to(F64), clip(x0_dev.cpu())), "post_process: not the clip of x0"
        return out


def run_checked(smp, model, rule, steps, x, conds=(), state=None):
    """The generate_samples loop over `steps` (already scaled), one checked step at a time, from x."""
    chk = StepChecker(smp, model, rule)
    for i in range(len(steps) - 1):
        x, state = chk.step(x, steps[i], steps[i + 1], conds, state)
    return chk.final(x, steps[-1], conds), chk


# ------------------------------------------------------------------- mutants: one fused coefficient off
class HeunH1UsesCs(HeunSampler):
    """HeunSampler with h1 = dt / (2 cs) where steps.py has dt / (2 ns)."""

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state, sample_model_fn, next_step=1):
        ca, cs = _steps._rates(self.noise_schedule, current_step)
        na, ns = _steps._rates(self.noise_schedule, next_step)
        dt = ns - cs
        k = (ca * ns - na * cs) / dt
        g0 = dt / cs
        x_pred = _steps._affine([current_samples, reconstructed_samples], [1 + g0, -k * g0])
        est_x0, _, _ = sample_model_fn(x_pred, next_step, *model_conditioning_inputs)
        h0, h1 = 0.5 * dt / cs, 0.5 * dt / cs                                  # mutated: cs where ns belongs
        return _steps._affine([current_samples, reconstructed_samples, x_pred, est_x0],
                                 [1 + h0, -k * h0, h1, -k * h1]), state


class MultiStepSwappedCm(MultiStepDPM):
    """MultiStepDPM with cm = c3 / d1 where steps.py has c3 / d0."""

    def take_next_step(self, current_samples, reconstructed_samples, model_conditioning_inputs, pred_noise,
                       current_step, state, sample_model_fn, next_step=1):
        _, cs = _steps._rates(self.noise_schedule, current_step)
        _, ns = _steps._rates(self.noise_schedule, next_step)
        dt = ns - cs
        hist = self.history
        if len(hist) < 2:
            return super().take_next_step(current_samples, reconstructed_samples, model_conditioning_inputs,
                                          pred_noise, current_step, state, sample_model_fn, next_step)
        l, m = hist[-1], hist[-2]
        d1, d0 = cs - l['sigma'], l['sigma'] - m['sigma']
        c2 = 0.5 * dt ** 2
        c3 = (1 / 6) * dt ** 3 / (0.5 * ((cs + l['sigma']) - (l['sigma'] + m['sigma'])))
        ce = dt + c2 / d1 + c3 / d1
        cl = -c2 / d1 - c3 / d1 - c3 / d0
        cm = c3 / d1                                                            # mutated: d1 where d0 belongs
        out = _steps._affine([current_samples, pred_noise, l['eps'], m['eps']], [1.0, ce, cl, cm])
        self.history.append({"eps": pred_noise, "sigma": cs})
        return out, state
