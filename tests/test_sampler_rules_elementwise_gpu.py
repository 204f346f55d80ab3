"""Every sampler update rule and prediction transform, step by step and element by element against the float64
restatement of tests/sampler_ref.py, with the analytic Gaussian denoiser in place of the UNet.

At every step the restatement is fed the device's own state x_i (and, inside Heun and RK4, the device's own stages,
which are checked too), so errors do not compound and the bound stays at a few f32 roundings of each step.  Each
model input must be bf16(f32(x) f32(c_in)) bit for bit.  The stochastic rules draw from a `utils.ThreefryKey`; the
reference noise is the host restatement of jax.random.normal along the same split chain, never read back."""
import pytest
import torch

import sampler_ref as S
from flaxdiff_b200 import utils
from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.samplers import RK4Sampler
from test_sampler_rules_ref_cpu import CLASSES, SCHEDULES, TRANSFORMS, make

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
WORST = {}

VE = ("karras_ve", "edm")


def _allowed(rule, sched_name):
    if rule == "rk4":
        return sched_name in VE                       # GeneralizedNoiseScheduler only (rk4_sampler.py:10)
    if rule == "ddpm":
        return sched_name in ("linear", "cosine")      # posterior tables: discrete schedules only
    if rule == "ddim_eta":
        return sched_name not in VE                    # sqrt(1 - alpha^2) / ... is 0 / 0 at alpha = 1
    return True


MATRIX = [(r, s, k) for r in S.RULES for s in SCHEDULES for k in TRANSFORMS if _allowed(r, s)]


def _start_end(rule, sched_name, kind):
    """Start at the schedule's top; end at step 0 (into sigma(0), which is 0 for the continuous cosine schedule)
    except where the reference itself divides by sigma(0) = 0 there: Heun's dx_1 / next_sigma, and the Karras
    transform's c_out = 0."""
    if sched_name == "cosine_continuous":
        return 990, (1 if rule == "heun" or kind == "karras" else 0)
    return (999 if sched_name in ("linear", "cosine") else 1000), 0


def _setup(rule, sched_name, kind, g=0.0, B=2, H=8, spacing="linear", n=5, seed=0, cls=None, graph=False):
    smp, model, conds = make(rule, sched_name, kind, g, H, cls=cls, spacing=spacing, device=dev)
    smp.use_cuda_graph = graph
    mci = ()
    if g > 0:
        mci = (conds[0].encoder([f"prompt {i}" for i in range(B)]).to(dev),)
    start, end = _start_end(rule, sched_name, kind)
    steps = [smp.scale_steps(float(s)) for s in smp.get_steps(start, end if spacing != "karras" else max(end, 1), n)]
    a, s = smp.noise_schedule.get_rates(torch.tensor([steps[0]], device=dev), shape=(-1,))
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, H, H, 3, generator=gen) * float(torch.sqrt(a ** 2 + s ** 2))).to(dev)
    return smp, model, mci, steps, x


def _report(key, worst):
    WORST[key] = max(WORST.get(key, 0.0), worst)
    print(f"{key}: worst |err|/bound {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("rule,sched_name,kind", MATRIX, ids=["-".join(c) for c in MATRIX])
def test_rule_step_by_step(rule, sched_name, kind):
    i = MATRIX.index((rule, sched_name, kind))
    B, H = (1, 3, 2)[i % 3], (8, 16, 32)[i % 3]
    smp, model, mci, steps, x = _setup(rule, sched_name, kind, B=B, H=H, seed=i)
    _, chk = S.run_checked(smp, model, rule, steps, x, mci, utils.RandomMarkovState(utils.jax_key(i)))
    _report(f"{rule} / {sched_name} / {kind}", chk.worst)


# karras spacing reads the schedule's min_inv_rho / max_inv_rho: Karras-family schedules only
GUIDED = [(r, sp) for r in S.RULES for sp in ("linear", "quadratic", "karras", "exponential")
          if sp != "karras" or any(_allowed(r, s) for s in VE)]


@pytest.mark.parametrize("rule,spacing", GUIDED, ids=[f"{r}-{sp}-g3" for r, sp in GUIDED])
def test_rule_with_guidance_and_spacing(rule, spacing):
    """Guidance 3 with a text context (conditional and unconditional rows differ), every spacing; schedule and
    transform rotate over the ones the rule allows."""
    allowed = [(s, k) for (r, s, k) in MATRIX if r == rule and (spacing != "karras" or s in VE)]
    i = GUIDED.index((rule, spacing))
    sched_name, kind = allowed[(5 * i) % len(allowed)]
    smp, model, mci, steps, x = _setup(rule, sched_name, kind, g=3.0, B=2, H=8, spacing=spacing, n=6, seed=100 + i)
    assert len(set(steps)) == len(steps), steps
    _, chk = S.run_checked(smp, model, rule, steps, x, mci, utils.RandomMarkovState(utils.jax_key(i)))
    _report(f"{rule} / {sched_name} / {kind} / g=3 / {spacing}", chk.worst)


def test_large_image_every_rule():
    """One 256 x 256 x 3 batch per rule."""
    for rule in S.RULES:
        sched_name = "linear" if rule in ("ddpm", "ddim_eta") else "karras_ve"
        smp, model, mci, steps, x = _setup(rule, sched_name, "eps" if sched_name == "linear" else "karras", B=1,
                                           H=256, n=3)
        _, chk = S.run_checked(smp, model, rule, steps, x, mci, utils.RandomMarkovState(utils.jax_key(3)))
        _report(f"{rule} / {sched_name} / 256x256", chk.worst)


@pytest.mark.parametrize("sched_name", ["linear", "cosine", "cosine_continuous"])
def test_rk4_refuses_variance_preserving_schedules(sched_name):
    with pytest.raises(FdxError, match="GeneralizedNoiseScheduler"):
        RK4Sampler(None, SCHEDULES[sched_name](), TRANSFORMS["eps"](), DiffusionInputConfig("image", (8, 8, 3), []))


@pytest.mark.parametrize("spacing,n,end", [("linear", 3, 0), ("linear", 1000, 0), ("karras", 10, 1)])
def test_multistep_orders_and_near_equal_sigmas(spacing, n, end):
    """First-, second- and third-order steps.  At 1000 linear steps adjacent Karras sigmas differ by as little as
    0.55 %, so d0 and d1 are small against the sigmas they are differences of.  Karras spacing runs to step 1:
    from step 0 its sequence is all zeros, and beyond 10 steps it repeats steps, where d1 = 0 (both as in the
    reference)."""
    smp, model, mci, _, x = _setup("multistep_dpm", "karras_ve", "karras", B=2, H=8, spacing=spacing)
    steps = [smp.scale_steps(float(s)) for s in smp.get_steps(1000, end, n)]
    assert len(set(steps)) == len(steps)
    sig = smp.noise_schedule.get_sigmas(torch.tensor(steps)).double()
    d = (sig[:-1] - sig[1:]) / sig[:-1]
    print(f"{spacing} x {n}: smallest relative sigma difference {d.min().item():.2e}")
    _, chk = S.run_checked(smp, model, "multistep_dpm", steps, x, mci)
    assert len(chk.history) == len(steps) - 1
    _report(f"multistep_dpm / karras_ve / {spacing} x {n}", chk.worst)


def test_multistep_history_carries_over_to_a_second_generate_samples():
    """MultiStepDPM never resets `history` (the reference does not either): a second generate_samples on the same
    instance starts with a third-order step on the first run's eps.  Pinned: the first run equals a fresh
    sampler's, the second does not, and the second equals the checked loop started from the first run's
    history."""
    n, B, H = 4, 2, 8
    smp, model, mci, steps, x = _setup("multistep_dpm", "karras_ve", "karras", B=B, H=H, n=n)
    fresh, _, _, _, _ = _setup("multistep_dpm", "karras_ve", "karras", B=B, H=H, n=n)
    kw = dict(diffusion_steps=n, start_step=1000, priors=x, device=dev)
    first = smp.generate_samples(model.params, B, H, **kw)
    assert torch.equal(first, fresh.generate_samples(model.params, B, H, **kw))
    assert len(smp.history) == n - 1
    hist_after_first = list(smp.history)
    second = smp.generate_samples(model.params, B, H, **kw)
    assert len(smp.history) == 2 * (n - 1) and not torch.equal(first, second)
    # the same second run, checked step by step with the first run's history
    chk_smp, chk_model, _, _, _ = _setup("multistep_dpm", "karras_ve", "karras", B=B, H=H, n=n)
    chk = S.StepChecker(chk_smp, chk_model, "multistep_dpm")
    chk_smp.history = list(hist_after_first)
    for h in hist_after_first:
        chk.history.append({"eps": S.V(S.t64(h["eps"], tuple(h["eps"].shape))), "sigma": S.V(S.t64(h["sigma"]))})
    y = x
    for i in range(n - 1):
        y, _ = chk.step(y, steps[i], steps[i + 1])
    y = chk.final(y, steps[-1])
    assert torch.equal(y, second)
    _report("multistep_dpm / second generate_samples", chk.worst)


def test_initial_sample_and_img2img_priors():
    """x_T = sqrt(alpha^2 + sigma^2) * noise from the first subkey; and priors with a start_step below the maximum
    (img2img): generate_samples equals the checked per-step loop from the same prior, bit for bit."""
    B, H = 3, 16
    for sched_name in ("karras_ve", "linear", "cosine_continuous"):
        smp, model, _, _, _ = _setup("euler", sched_name, "eps", B=B, H=H)
        start = 1000 if sched_name == "karras_ve" else 990
        state, k0 = utils.RandomMarkovState(utils.jax_key(11)).get_random_key()
        xT = smp._get_initial_samples(H, B, k0, start, dev)
        a, s = smp.noise_schedule.get_rates(torch.tensor([smp.scale_steps(float(start))], device=dev), shape=(-1,))
        ref = S.initial_sample(S.noise_ref(k0, (B, H, H, 3)), S.V(S.t64(a)), S.V(S.t64(s)))
        S.assert_elementwise(xT.cpu(), ref.v, ref.bound(6), f"x_T / {sched_name}")
    for rule in ("euler", "ddpm", "heun"):
        sched_name = "linear" if rule == "ddpm" else "karras_ve"
        smp, model, mci, _, x = _setup(rule, sched_name, "x0", B=B, H=H)
        start = 600
        steps = [smp.scale_steps(float(s)) for s in smp.get_steps(start, 0, 4)]
        key = utils.jax_key(12)
        got = smp.generate_samples(model.params, B, H, diffusion_steps=4, start_step=start, priors=x, device=dev,
                                   rngstate=utils.RandomMarkovState(key))
        want, chk = S.run_checked(smp, model, rule, steps, x, (), utils.RandomMarkovState(key))
        assert torch.equal(got, want)
        _report(f"{rule} / {sched_name} / img2img from {start}", chk.worst)


def test_post_process_clips_bit_for_bit():
    smp, _, _, _, _ = _setup("euler", "karras_ve", "x0")
    x = torch.tensor([-3.0, -1.0000001, -1.0, -0.9999999, -0.25, 0.0, 0.5, 0.9999999, 1.0, 1.0000001, 7.0, 1e30],
                     device=dev).repeat(2, 4, 1).reshape(2, 4, 4, 3)
    assert torch.equal(smp.post_process(x).cpu().double(), S.clip(x.cpu()))


@pytest.mark.parametrize("rule", S.RULES)
def test_graphed_generate_samples_equals_the_checked_eager_loop(rule):
    """generate_samples with use_cuda_graph=True (whole-step graph; per-evaluation graph for the history and RK4
    rules) equals the eager, step-by-step checked loop bit for bit; so its output lies within the bound of the
    last step given the eager loop's second-to-last state."""
    sched_name = "linear" if rule in ("ddpm", "ddim_eta") else "karras_ve"
    kind = "eps" if sched_name == "linear" else "karras"
    n, B, H = 6, 2, 16
    key = utils.jax_key(21)
    smp, model, mci, steps, x = _setup(rule, sched_name, kind, B=B, H=H, n=n, graph=True)
    model.record = False
    start, _ = _start_end(rule, sched_name, kind)
    got = smp.generate_samples(model.params, B, H, diffusion_steps=n, start_step=start, device=dev,
                               rngstate=utils.RandomMarkovState(key))
    assert len(smp._graphs) >= 1
    esmp, emodel, _, _, _ = _setup(rule, sched_name, kind, B=B, H=H, n=n)
    state, k0 = utils.RandomMarkovState(key).get_random_key()
    xT = esmp._get_initial_samples(H, B, k0, start, dev)
    want, chk = S.run_checked(esmp, emodel, rule, steps, xT, mci, state)
    assert torch.equal(got, want), (got - want).abs().max().item()
    _report(f"{rule} / {sched_name} / graphed loop", chk.worst)


# -------------------------------------------------------------------------------- discrimination, on the device
def _unet_end_to_end_rel(cls_good, cls_bad):
    """The relative L2 between a correct and a mutated sampler in test_samplers_gpu.py's end-to-end setting: the
    random-weight bf16 UNet, Karras VE, 16 x 16, B = 2, 4 steps from step 1000."""
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.schedulers import KarrasVENoiseScheduler
    torch.manual_seed(0)
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16)
    fp = model.init(4, device=dev)
    prior = (torch.randn(2, 16, 16, 3) * 80.0).to(dev)
    outs = []
    for cls in (cls_good, cls_bad):
        sched = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev)
        smp = cls(model, sched, KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (16, 16, 3), []),
                  use_cuda_graph=False)
        outs.append(smp.generate_samples(fp, 2, 16, diffusion_steps=4, start_step=1000, priors=prior, device=dev))
    a, b = (o.double().cpu() for o in outs)
    return ((b - a).norm() / a.norm()).item()


@pytest.mark.parametrize("mutant,rule", [(S.HeunH1UsesCs, "heun"), (S.MultiStepSwappedCm, "multistep_dpm")],
                         ids=["heun_h1_uses_cs", "multistep_cm_d0_d1_swapped"])
def test_device_mutants_are_rejected(mutant, rule):
    smp, model, mci, steps, x = _setup(rule, "karras_ve", "karras", B=2, H=8, cls=mutant)
    with pytest.raises(AssertionError, match="outside the bound") as info:
        S.run_checked(smp, model, rule, steps, x, mci)
    good = {"heun": CLASSES["heun"], "multistep_dpm": CLASSES["multistep_dpm"]}[rule]
    rel = _unet_end_to_end_rel(good, mutant)
    print(f"{mutant.__name__}: rejected per step ({str(info.value).splitlines()[0][:160]}); end to end with the "
          f"UNet it moves the output by relative L2 {rel:.3e} (test_samplers_gpu.py accepts up to 6e-2)")


def test_zz_report_worst_ratios():
    for k in sorted(WORST):
        print(f"  {WORST[k]:.3f}  {k}")
    assert all(v <= 1.0 for v in WORST.values())
