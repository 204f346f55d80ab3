"""The float64 restatement of tests/sampler_ref.py is right, and its element-wise comparison discriminates.

* Against closed forms: the order of convergence of Euler, Heun, RK4 and MultiStepDPM on the probability-flow ODE of
  Gaussian data, and each prediction transform's x0 / eps recovery from the stand-in denoiser's output.
* An f32 emulation of the fused rules of flaxdiff_b200/samplers/steps.py (the product's own code, with
  `fdx_affine_combine` written out in f32 torch on the CPU) stays inside the bound, and one mutated coefficient
  at a time does not."""
import math

import numpy as np
import pytest
import torch

import sampler_ref as S
from flaxdiff_b200 import ops, predictors, utils
from flaxdiff_b200 import samplers as smp_mod
from flaxdiff_b200 import schedulers as sc
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.samplers import steps as steps_mod

CPU = torch.device("cpu")
MU, SD = 0.3, 0.5


# ------------------------------------------------------------------------------------- order of convergence
def _x0(x, sigma):
    return MU + SD ** 2 * (x - MU) / (SD ** 2 + sigma ** 2)


def _eps(x, sigma):
    return sigma * (x - MU) / (SD ** 2 + sigma ** 2)


def _solve(rule, N, xT):
    """Integrate from sigma = 10 to 0.5 on a uniform float64 grid of N steps with the restated rule."""
    sig = np.linspace(10.0, 0.5, N + 1)
    x, hist, one = S.V(xT), [], S.V(torch.ones(()))
    for i in range(N):
        cs, ns = S.V(torch.tensor(sig[i])), S.V(torch.tensor(sig[i + 1]))
        if rule == "euler":
            x = S.euler(x, S.V(_x0(x.v, cs.v)), one, cs, one, ns)
        elif rule == "heun":
            xp = S.heun_predict(x, S.V(_x0(x.v, cs.v)), one, cs, one, ns)
            x = S.heun(x, S.V(_x0(x.v, cs.v)), xp, S.V(_x0(xp.v, ns.v)), one, cs, one, ns)
        elif rule == "rk4":
            dt = ns - cs
            k1 = S.V(_eps(x.v, cs.v))
            k2 = S.V(_eps(S.rk4_stage(x, k1, dt, 0.5).v, (cs + 0.5 * dt).v))
            k3 = S.V(_eps(S.rk4_stage(x, k2, dt, 0.5).v, (cs + 0.5 * dt).v))
            k4 = S.V(_eps(S.rk4_stage(x, k3, dt, 1).v, ns.v))
            x = S.rk4(x, k1, k2, k3, k4, dt)
        else:
            x = S.multistep_dpm(x, S.V(_eps(x.v, cs.v)), cs, ns, hist)
    return x.v


def test_order_of_convergence_against_the_closed_form():
    """x(sigma) = mu + (x_T - mu) sqrt((s^2 + sigma^2) / (s^2 + sigma_T^2)) solves dx/dsigma = eps(x, sigma) for
    x0 ~ N(mu, s^2).  Euler is order 1, Heun 2, RK4 4.

    MultiStepDPM: with e(sigma) the exact eps along the solution and h = dt, its third-order step adds
    dx_2 dt^2 / 2 + dx_3 dt^3 / 6 where dx_2 = (e_n - e_{n-1}) / h is a backward difference: dx_2 = e' - h e'' / 2
    + O(h^2).  The step's Taylor expansion needs e' h^2 / 2, so the local error keeps -(1/2)(h e''/2) h^2 =
    -h^3 e'' / 4 (the `-1/4 dt^2 d1 e''` term with d1 = dt); dx_3's own term is O(h^3) too but cannot cancel it
    for every e.  A local error of O(h^3) sums over N = O(1/h) steps to a global O(h^2): order 2."""
    xT = torch.tensor([-25.0, -3.0, 7.0, 40.0], dtype=torch.float64)
    exact = MU + (xT - MU) * math.sqrt((SD ** 2 + 0.5 ** 2) / (SD ** 2 + 10.0 ** 2))
    want = {"euler": 1.0, "heun": 2.0, "rk4": 4.0, "multistep_dpm": 2.0}
    for rule, p in want.items():
        e1 = (_solve(rule, 40, xT) - exact).abs().max().item()
        e2 = (_solve(rule, 80, xT) - exact).abs().max().item()
        order = math.log2(e1 / e2)
        print(f"{rule}: error {e1:.3e} at 40 steps, {e2:.3e} at 80, observed order {order:.2f} (derived {p:g})")
        assert e2 > 1e-11 and abs(order - p) <= 0.3, (rule, order)


# ------------------------------------------------------------------------------- transforms vs the closed form
SCHEDULES = {
    "karras_ve": lambda: sc.KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
    "edm": lambda: sc.EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
    "linear": lambda: sc.LinearNoiseSchedule(1000),
    "cosine": lambda: sc.CosineNoiseScheduler(1000),
    "cosine_continuous": lambda: sc.CosineContinuousNoiseScheduler(),
}
TRANSFORMS = {"eps": predictors.EpsilonPredictionTransform, "x0": predictors.DirectPredictionTransform,
              "v": predictors.VPredictionTransform, "karras": lambda: predictors.KarrasPredictionTransform(0.5)}


def _mu(H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(H, W, 3, generator=g, dtype=torch.float64) * 1.6 - 0.8)


@pytest.mark.parametrize("kind", list(TRANSFORMS))
@pytest.mark.parametrize("sched_name", list(SCHEDULES))
def test_transform_recovery_matches_the_closed_form(kind, sched_name):
    sched = SCHEDULES[sched_name]().to(CPU)
    fam = S.schedule_family(sched)
    model = S.GaussianDenoiser(kind, sched, _mu(4, 4))
    steps = torch.tensor([0.999, 0.5, 0.02] if fam != "discrete" else [999.0, 500.0, 3.0], dtype=torch.float32)
    a32, s32 = sched.get_rates(steps, shape=(-1,))
    _, t_model = sched.transform_inputs(None, steps)
    a, s = (r.reshape(-1, 1, 1, 1) for r in S.recovered_rates(fam, t_model, model.tables))
    x = torch.randn(3, 4, 4, 3, dtype=torch.float64) * (a ** 2 + s ** 2).sqrt()
    xin = x * S.input_scale(kind, S.V(s)).v
    F, _ = S.denoiser_output(kind, fam, xin, t_model, model.mu, tables=model.tables)
    x0, eps = S.x0_eps(kind, S.V(x), S.V(F), S.V(a), S.V(s))
    D = model.mu + a * SD ** 2 * (x - a * model.mu) / (a ** 2 * SD ** 2 + s ** 2)
    # float64 rounding, amplified by 1 / alpha (eps: x0 = (x - sigma F) / alpha) or 1 / sigma (x0, Karras)
    tol = 1e-13 * (1 + x.abs() + D.abs()) / torch.minimum(a, s)
    assert ((x0.v - D).abs() <= tol).all() and ((eps.v - (x - a * D) / s).abs() <= tol / torch.minimum(a, s)).all()
    # the f32 rates the sampler uses and the ones the stand-in recovers from the model time agree to f32 accuracy
    torch.testing.assert_close(s.reshape(-1), s32.to(torch.float64), rtol=2e-6, atol=0)
    torch.testing.assert_close(a.reshape(-1), a32.to(torch.float64), rtol=2e-6, atol=0)


# ------------------------------------------------------------------------------- f32 emulation of the kernels
def _affine_f32(inputs, coef1, coef2=None, want_out1=True, bf16_scale=None, want_bf16=False, clip=None):
    """fdx_affine_combine in f32 torch: a product and a sum, each rounded, per term (the kernel fuses them)."""
    B = inputs[0].shape[0]

    def comb(coef):
        o = torch.zeros_like(inputs[0])
        for k, t in enumerate(inputs):
            o = o + coef[k].view(B, *([1] * (t.dim() - 1))) * t
        return o
    o1 = comb(coef1.to(torch.float32))
    o2 = comb(coef2.to(torch.float32)) if coef2 is not None else None
    if clip is not None:
        o1 = torch.clamp(o1, clip[0], clip[1])
    ob = None
    if want_bf16:
        sc_ = bf16_scale if bf16_scale is not None else torch.ones(B)
        ob = (o1 * sc_.view(B, *([1] * (o1.dim() - 1)))).to(torch.bfloat16)
    return (o1 if want_out1 else None), o2, ob


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(ops, "affine_combine", _affine_f32)
    monkeypatch.setattr(ops, "random_normal", lambda words, shape, device=None: torch.from_numpy(
        utils.normal_f32(tuple(int(w) for w in words), int(np.prod(shape)))).reshape(shape))


CLASSES = {"euler": smp_mod.EulerSampler, "simplified_euler": smp_mod.SimplifiedEulerSampler,
           "euler_ancestral": smp_mod.EulerAncestralSampler, "heun": smp_mod.HeunSampler,
           "ddim": smp_mod.DDIMSampler, "ddim_eta": smp_mod.DDIMSampler, "ddpm": smp_mod.DDPMSampler,
           "simple_ddpm": smp_mod.SimpleDDPMSampler, "rk4": smp_mod.RK4Sampler,
           "multistep_dpm": smp_mod.MultiStepDPM}


def make(rule, sched_name, kind, g=0.0, H=8, cls=None, tr=None, spacing="linear", device=CPU):
    sched = SCHEDULES[sched_name]().to(device)
    model = S.GaussianDenoiser(kind, sched, _mu(H, H, 1))
    kw = {"eta": 0.5} if rule == "ddim_eta" else {}
    conds = []
    if g > 0:
        enc = RandomEmbeddingEncoder(7, 16, device=device)
        conds = [ConditionalInputConfig(enc)]
    cfg = DiffusionInputConfig("image", (H, H, 3), conds)
    smp = (cls or CLASSES[rule])(model, sched, tr or TRANSFORMS[kind](), cfg, guidance_scale=g,
                                 timestep_spacing=spacing, use_cuda_graph=False, **kw)
    return smp, model, conds


def _run(rule, sched_name, kind, g=0.0, cls=None, tr=None, n=5, B=2, H=8):
    smp, model, conds = make(rule, sched_name, kind, g, H, cls, tr)
    mci = ()
    if g > 0:
        mci = (conds[0].encoder([f"p{i}" for i in range(B)]),)
    start = 999 if S.schedule_family(smp.noise_schedule) == "discrete" else (990 if sched_name == "cosine_continuous"
                                                                                else 1000)
    steps = [smp.scale_steps(float(s)) for s in smp.get_steps(start, 0, n)]
    a, s = smp.noise_schedule.get_rates(torch.tensor(steps[0]), shape=(-1,))
    x = (torch.randn(B, H, H, 3, generator=torch.Generator().manual_seed(3)) * torch.sqrt(a ** 2 + s ** 2)).float()
    state = utils.RandomMarkovState(utils.jax_key(5))
    _, chk = S.run_checked(smp, model, rule, steps, x, mci, state)
    return chk.worst


EMULATED = [("euler", "karras_ve", "karras"), ("simplified_euler", "edm", "karras"), ("heun", "linear", "v"),
            ("euler_ancestral", "cosine", "eps"), ("ddim", "cosine_continuous", "x0"), ("ddim_eta", "linear", "eps"),
            ("ddpm", "cosine", "v"), ("simple_ddpm", "linear", "x0"), ("rk4", "karras_ve", "eps"),
            ("multistep_dpm", "edm", "v")]


@pytest.mark.parametrize("rule,sched_name,kind", EMULATED)
@pytest.mark.parametrize("g", [0.0, 3.0])
def test_f32_emulation_of_the_fused_rules_is_within_the_bound(emulated, rule, sched_name, kind, g):
    worst = _run(rule, sched_name, kind, g)
    print(f"{rule} / {sched_name} / {kind} / g={g:g}: worst |err|/bound {worst:.3f}")
    assert worst <= 1.0


# ----------------------------------------------------------------------------------------------- mutations
class _RK4QuarterWeights(smp_mod.RK4Sampler):
    def sample_step(self, sample_model_fn, current_samples, current_step, model_conditioning_inputs,
                    next_step=None, state=None):
        B, dev = current_samples.shape[0], current_samples.device
        cur = torch.as_tensor(current_step, device=dev, dtype=torch.float32).expand(B)
        nxt = torch.as_tensor(next_step, device=dev, dtype=torch.float32).expand(B)
        _, cs = steps_mod._rates(self.noise_schedule, cur)
        _, ns = steps_mod._rates(self.noise_schedule, nxt)
        dt = ns - cs
        x, c = current_samples, model_conditioning_inputs
        k1 = self._deriv(sample_model_fn, x, cs, c)
        k2 = self._deriv(sample_model_fn, steps_mod._affine([x, k1], [1.0, 0.5 * dt]), cs + 0.5 * dt, c)
        k3 = self._deriv(sample_model_fn, steps_mod._affine([x, k2], [1.0, 0.5 * dt]), cs + 0.5 * dt, c)
        k4 = self._deriv(sample_model_fn, steps_mod._affine([x, k3], [1.0, dt]), cs + dt, c)
        return steps_mod._affine([x, k1, k2, k3, k4], [1.0, dt / 6, dt / 4, dt / 4, dt / 6]), state   # mutated


class _VSignFlippedOnVP(predictors.VPredictionTransform):
    def backward_coeffs(self, rates):
        p, q, r, u = super().backward_coeffs(rates)
        a, _ = predictors._flat_rates(rates)
        return p, q, r, torch.where(a < 1, -u, u)                               # mutated for VP (alpha < 1) only


def _cfg_swapped_eval(self, fp, x_t, t, *conditioning):
    """DiffusionSampler._eval with the guidance fold as g Fc + (1 - g) Fu computed with g and 1 - g swapped."""
    sched, tr = self.noise_schedule, self.model_output_transform
    B, g = x_t.shape[0], float(self.guidance_scale)
    rates = sched.get_rates(t)
    c_in = tr.get_input_scale(rates)
    cvec = predictors._vec(c_in.reshape(-1) if isinstance(c_in, torch.Tensor) else c_in, B, x_t.device)
    _, t_model = sched.transform_inputs(None, t)
    _, _, xin = ops.affine_combine([x_t], torch.ones((1, B)), want_out1=False, bf16_scale=cvec, want_bf16=True)
    p, q, r, u = tr.x0_eps_coeffs(rates)
    conds = [torch.cat([c, unc.expand_as(c)]) for c, unc in zip(conditioning, self._unconditionals)]
    F2, _ = self.model.forward(fp, torch.cat([xin, xin]), torch.cat([t_model, t_model]), *(conds or [None]))
    Fc, Fu = F2[:B].contiguous(), F2[B:].contiguous()
    x0, eps = predictors._affine([x_t, Fc, Fu], [p, q * (1 - g), q * g], [r, u * (1 - g), u * g])    # mutated
    return x0, eps, Fu


MUTATIONS = {
    "multistep_cm_d0_d1_swapped": dict(rule="multistep_dpm", sched_name="karras_ve", kind="karras",
                                       cls=S.MultiStepSwappedCm),
    "heun_h1_uses_cs": dict(rule="heun", sched_name="karras_ve", kind="karras", cls=S.HeunH1UsesCs),
    "rk4_middle_weights_dt_over_4": dict(rule="rk4", sched_name="edm", kind="eps", cls=_RK4QuarterWeights),
    "v_u_sign_flipped_on_vp": dict(rule="ddim", sched_name="linear", kind="v", tr=_VSignFlippedOnVP()),
    "cfg_g_and_1_minus_g_swapped": dict(rule="euler", sched_name="karras_ve", kind="karras", g=3.0),
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_comparator_rejects_each_mutated_coefficient(emulated, monkeypatch, name):
    kw = dict(MUTATIONS[name])
    if name.startswith("cfg"):
        monkeypatch.setattr(smp_mod.DiffusionSampler, "_eval", _cfg_swapped_eval)
    with pytest.raises(AssertionError, match="outside the bound"):
        _run(**kw)
    if name.startswith("v_u"):          # the same mutation is invisible on a VE schedule, where it does not apply
        assert _run("ddim", "karras_ve", "v", tr=_VSignFlippedOnVP()) <= 1.0
