"""The samplers that draw one noise tensor per step (EulerAncestral, DDPM, SimpleDDPM, DDIM eta > 0) and the trainer,
with a `utils.ThreefryKey`: the draws are jax.random's (the host restatements of utils.py along the host `split`
chain), the samplers take the whole-step CUDA graph, and a plain tuple key keeps the per-evaluation path.

Two runs of the real UNet are not promised to agree bit for bit (f32 atomics in some reductions), so bit-for-bit
equality of the graphed and the eager step is shown with a deterministic stand-in denoiser (everything but the
model is the product's code); with the real UNet the two agree to the tolerance the other sampler tests use and
match the oracle's step restatements fed the same noise."""
import numpy as np
import pytest
import torch

from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.predictors import EpsilonPredictionTransform, KarrasPredictionTransform
from flaxdiff_b200.samplers import (DDIMSampler, DDPMSampler, EulerAncestralSampler, EulerSampler,
                                    SimpleDDPMSampler)
from flaxdiff_b200.schedulers import KarrasVENoiseScheduler, LinearNoiseSchedule
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw, rank_key
from oracle import diffusion_ref as R
from oracle import train_ref, unet_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
B, RES = 2, 16


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


class _Params:
    """What the sampler asks of a parameter set: a bf16 shadow to refresh before a replay."""

    def shadow(self):
        return None


class _StandInDenoiser:
    """F = 0.3 x_in - 0.1 + (mean of the text context): deterministic torch arithmetic in place of the UNet."""

    def __init__(self):
        self.params = _Params()

    def _as_flat(self, params, device):
        return self.params

    def forward(self, fp, x, t, ctx=None, save=False):
        y = x.float() * 0.3 - 0.1 + t.float().view(-1, 1, 1, 1) * 1e-3
        if ctx is not None:
            y = y + ctx.float().mean(dim=(1, 2)).view(-1, 1, 1, 1)
        return y.contiguous(), None


def _karras():
    return KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev), KarrasPredictionTransform(0.5)


def _linear():
    return LinearNoiseSchedule(1000).to(dev), EpsilonPredictionTransform()


CASES = {
    "euler_a": (EulerAncestralSampler, _karras, {}, 1000),
    "euler_a_cfg": (EulerAncestralSampler, _karras, {"guidance_scale": 3.0}, 1000),
    "ddpm": (DDPMSampler, _linear, {}, 1000),
    "simple_ddpm": (SimpleDDPMSampler, _linear, {}, 700),
    "ddim_eta": (DDIMSampler, _linear, {"eta": 0.5}, 700),
}


def _sampler(case, model, graph):
    cls, sched_fn, kw, start = CASES[case]
    sched, tr = sched_fn()
    conds, mci = [], ()
    if "guidance_scale" in kw:
        enc = RandomEmbeddingEncoder(77, 768, device=dev)
        conds, mci = [ConditionalInputConfig(enc)], (enc(["a cat", "a dog"]).to(dev),)
    smp = cls(model, sched, tr, DiffusionInputConfig("image", (RES, RES, 3), conds), use_cuda_graph=graph, **kw)
    return smp, mci, start


def _subkeys(key, n):
    """x_T's key and the n per-step subkeys generate_samples splits off a RandomMarkovState(key)."""
    state, out = utils.RandomMarkovState(key), []
    for _ in range(n + 1):
        state, k = state.get_random_key()
        out.append(k)
    return out[0], out[1:]


@pytest.fixture
def replays(monkeypatch):
    count = [0]
    orig = torch.cuda.CUDAGraph.replay

    def counted(self):
        count[0] += 1
        return orig(self)
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", counted)
    return count


@pytest.mark.parametrize("case", list(CASES))
def test_graphed_step_equals_eager_step_bit_for_bit_and_draws_jax_noise(case, replays, monkeypatch):
    n = 10
    key = utils.jax_key(7)
    drawn = []
    real = utils.device_normal

    def recording(k, shape, device, dtype=torch.float32):
        z = real(k, shape, device, dtype)
        drawn.append((k, z))
        return z
    monkeypatch.setattr(utils, "device_normal", recording)
    model = _StandInDenoiser()
    eager, mci, start = _sampler(case, model, False)
    want = eager.generate_samples(model.params, B, RES, diffusion_steps=n, start_step=start, device=dev,
                                  rngstate=utils.RandomMarkovState(key), model_conditioning_inputs=mci)
    # the eager run drew x_T and one noise per step but the last, each from the host chain's subkey, and each is
    # the host restatement of jax.random.normal for that subkey
    k0, ks = _subkeys(key, n - 1)
    assert [k for k, _ in drawn] == [k0] + ks and all(type(k) is utils.ThreefryKey for k, _ in drawn)
    for k, z in drawn:
        host = utils.normal_f32(k, B * RES * RES * 3).reshape(B, RES, RES, 3)
        np.testing.assert_allclose(z.cpu().numpy(), host, rtol=2e-5, atol=0)
    assert torch.isfinite(want).all() and want.abs().max() > 0
    monkeypatch.setattr(utils, "device_normal", real)
    graphed, mci, start = _sampler(case, model, True)
    for i in range(3):                                  # the first call captures, the others re-use the graphs
        if i == 1:
            replays[0] = 0
        got = graphed.generate_samples(model.params, B, RES, diffusion_steps=n, start_step=start, device=dev,
                                       rngstate=utils.RandomMarkovState(key), model_conditioning_inputs=mci)
        assert torch.equal(got, want)
    # one replay per step: n - 1 whole steps and the last evaluation, in two graphs
    assert replays[0] == 2 * n and len(graphed._graphs) == 2
    assert sorted(k[0] == "step" for k in graphed._graphs) == [False, True]
    other = graphed.generate_samples(model.params, B, RES, diffusion_steps=n, start_step=start, device=dev,
                                     rngstate=utils.RandomMarkovState(utils.jax_key(8)), model_conditioning_inputs=mci)
    assert not torch.equal(other, want) and len(graphed._graphs) == 2       # a new key is 8 bytes, not a new graph


def test_tuple_key_keeps_the_per_evaluation_graph_and_cache_stays_bounded(replays):
    n = 6
    model = _StandInDenoiser()
    state = utils.RandomMarkovState(utils.PRNGKey(7))
    eager, _, _ = _sampler("euler_a", model, False)
    graphed, _, _ = _sampler("euler_a", model, True)
    want = eager.generate_samples(model.params, B, RES, diffusion_steps=n, start_step=1000, device=dev, rngstate=state)
    for i in range(2):                                   # the first call captures the evaluation graph
        replays[0] = 0
        got = graphed.generate_samples(model.params, B, RES, diffusion_steps=n, start_step=1000, device=dev,
                                       rngstate=state)
        assert torch.equal(got, want)
    assert replays[0] == n and [k[0] == "step" for k in graphed._graphs] == [False]
    for i in range(8):                                   # batch sizes and both key kinds: the LRU stays bounded
        key = utils.jax_key(i) if i % 2 else utils.PRNGKey(i)
        graphed.generate_samples(model.params, 1 + i % 5, RES, diffusion_steps=3, start_step=1000, device=dev,
                                 rngstate=utils.RandomMarkovState(key))
        assert len(graphed._graphs) <= graphed.MAX_GRAPHS
    det = EulerSampler(model, *_karras(), DiffusionInputConfig("image", (RES, RES, 3), []))
    det.generate_samples(model.params, B, RES, diffusion_steps=3, start_step=1000, device=dev,
                         rngstate=utils.RandomMarkovState(utils.jax_key(1)))
    assert sorted(k[0] == "step" for k in det._graphs) == [False, True]     # deterministic rules: as before


def _unet():
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16)
    fp = model.init(4, device=dev)
    return model, fp, {k: v.detach().cpu().clone() for k, v in fp.named.items()}


@pytest.mark.parametrize("case", ["euler_a", "ddpm", "simple_ddpm", "ddim_eta"])
def test_unet_sampling_with_jax_noise_vs_oracle(case):
    """Real UNet, whole-step graph, ThreefryKey: against the oracle's step restatements fed normal_f32 of the
    host chain's subkeys (tolerances of tests/test_samplers_gpu.py and tests/test_unet_gpu.py)."""
    torch.manual_seed(0)
    model, fp, P = _unet()
    n = 4
    key = utils.jax_key(7)
    smp, _, start = _sampler(case, model, True)
    sched = smp.noise_schedule
    out = smp.generate_samples(fp, B, RES, diffusion_steps=n, start_step=start, device=dev,
                               rngstate=utils.RandomMarkovState(key))
    eager, _, _ = _sampler(case, model, False)
    out_eager = eager.generate_samples(fp, B, RES, diffusion_steps=n, start_step=start, device=dev,
                                       rngstate=utils.RandomMarkovState(key))
    assert rel(out, out_eager) < 3e-2, rel(out, out_eager)
    k0, ks = _subkeys(key, n - 1)
    shape = (B, RES, RES, 3)
    noises = [torch.from_numpy(utils.normal_f32(k, B * RES * RES * 3).reshape(shape)) for k in ks]
    freqs = model._fourier_freqs(dev).cpu()
    steps = [float(s) for s in smp.get_steps(start, 0, n)]
    a0, s0 = (v.reshape(-1)[0].item() for v in sched.get_rates(torch.full((B,), smp.scale_steps(float(start)), device=dev)))
    x = torch.from_numpy(utils.normal_f32(k0, B * RES * RES * 3).reshape(shape)) * float(np.sqrt(a0 ** 2 + s0 ** 2))
    if case == "euler_a":
        for i in range(n):
            cur, nxt = steps[i] / 1000.0, (steps[i + 1] if i + 1 < n else 0) / 1000.0
            x0, _ = train_ref.karras_denoise_eval(P, x, torch.full((B,), cur), freqs)
            if i == n - 1:
                x = x0.clamp(-1, 1)
                break
            one = np.ones(B, np.float32)
            cs, ns = R.karras_sigma(np.full(B, cur, np.float32)), R.karras_sigma(np.full(B, nxt, np.float32))
            x = torch.from_numpy(R.euler_ancestral_step(x.numpy(), x0.numpy(), noises[i].numpy(), one, cs, one, ns))
        assert rel(out, x) < 6e-2, rel(out, x)
        return
    T = R.linear_tables(1000)
    for i, s in enumerate(steps):
        nxt = steps[i + 1] if i + 1 < n else 0.0
        a, sg = (v.cpu().numpy().reshape(-1) for v in sched.get_rates(torch.full((B,), s, device=dev)))
        na, ns = (v.cpu().numpy().reshape(-1) for v in sched.get_rates(torch.full((B,), nxt, device=dev)))
        with torch.no_grad():
            F = unet_ref.unet_forward(P, x, torch.full((B,), s), freqs)
        x0 = (x - F * torch.from_numpy(sg).view(-1, 1, 1, 1)) / torch.from_numpy(a).view(-1, 1, 1, 1)
        if i == n - 1:
            x = x0.clamp(-1, 1)
            break
        z = noises[i].numpy()
        if case == "simple_ddpm":
            x = R.simple_ddpm_step(x0.numpy(), F.numpy(), z, a, sg, na, ns)
        elif case == "ddpm":
            idx = int(R.discrete_index([s])[0])
            x = R.ddpm_step(x0.numpy(), x.numpy(), z, np.full(B, T["posterior_mean_coef1"][idx]),
                            np.full(B, T["posterior_mean_coef2"][idx]),
                            np.full(B, T["posterior_log_variance_clipped"][idx]))
        else:       # DDIM with eta: the deterministic rule plus eta * sigma_tilde * noise
            sig = 0.5 * ns * np.sqrt(1 - a ** 2 / na ** 2) / np.sqrt(1 - a ** 2)
            x = R.ddim_step(x0.numpy(), F.numpy(), na, ns) + z * sig.reshape(-1, 1, 1, 1)
        x = torch.from_numpy(np.asarray(x, dtype=np.float32))
    assert torch.isfinite(out).all() and rel(out, x) < 6e-2, rel(out, x)


def _trainer(graph, rngs):
    model = Unet(attention_configs=(None, None, None, {"heads": 8}), dtype=torch.bfloat16, context_dim=768)
    enc = RandomEmbeddingEncoder(77, 768, device=dev)
    cfg = DiffusionInputConfig("image", (RES, RES, 3), [ConditionalInputConfig(enc)])
    return GeneralDiffusionTrainer(model, adamw(1e-3), LinearNoiseSchedule(1000), cfg, rngs=rngs,
                                   unconditional_prob=0.5, model_output_transform=EpsilonPredictionTransform(),
                                   device=dev, use_cuda_graph=graph)


def _record(monkeypatch):
    log = {"uniform": [], "randint": [], "normal": []}
    for name in log:
        real = getattr(utils, "device_" + name)

        def rec(key, *a, _real=real, _name=name, **kw):
            out = _real(key, *a, **kw)
            log[_name].append((key, out.clone()))
            return out
        monkeypatch.setattr(utils, "device_" + name, rec)
    return log


def _two_steps(graph, log):
    """Two training steps with rngs=jax_key(4); checks every draw against the host chain, returns the losses."""
    torch.manual_seed(0)
    Bt = 4
    tr = _trainer(graph, utils.jax_key(4))
    assert type(tr.rngstate.rng) is utils.ThreefryKey
    step = tr._define_train_step(Bt)
    batch = {"image": torch.randint(0, 256, (Bt, RES, RES, 3), dtype=torch.uint8), "text": ["a", "b", "c", "d"]}
    state = utils.RandomMarkovState(utils.jax_key(4))
    losses = []
    for it in range(2):
        for v in log.values():
            v.clear()
        tr.state, loss, tr.rngstate = step(tr.state, tr.rngstate, dict(batch), 0)
        losses.append(loss.item())
        # the trainer's own chain: step key -> fold_in(rank) -> mask key, timestep key, noise key
        state, key_fold = state.get_random_key()
        local = utils.RandomMarkovState(rank_key(key_fold, 0))
        local, mask_key = local.get_random_key()
        local, t_key = local.get_random_key()
        local, noise_key = local.get_random_key()
        assert tr.rngstate.rng == state.rng and type(tr.rngstate.rng) is utils.ThreefryKey
        (k, uni), = log["uniform"]
        assert k == mask_key and np.array_equal(uni.cpu().numpy() < np.float32(0.5), utils.bernoulli(mask_key, 0.5, Bt))
        (k, t), = log["randint"]
        assert k == t_key and np.array_equal(t.cpu().numpy(), utils.randint(t_key, Bt, 0, 1000))
        (k, eps), = log["normal"]
        host = utils.normal_f32(noise_key, Bt * RES * RES * 3).reshape(Bt, RES, RES, 3)
        assert k == noise_key and eps.shape == (Bt, RES, RES, 3)
        np.testing.assert_allclose(eps.cpu().numpy(), host, rtol=2e-5, atol=0)
        # rank 1 folds another stream
        other = utils.RandomMarkovState(rank_key(key_fold, 1))
        for _ in range(3):
            other, k1 = other.get_random_key()
        assert not torch.equal(utils.device_normal(k1, (Bt, RES, RES, 3), dev), eps)
    assert all(np.isfinite(losses))
    return losses


def test_trainer_draws_mask_timesteps_and_noise_from_jax_streams(monkeypatch):
    log = _record(monkeypatch)
    eager, graphed = _two_steps(False, log), _two_steps(True, log)
    # eager step = CUDA-graphed step, to the UNet's run-to-run tolerance
    np.testing.assert_allclose(graphed, eager, rtol=2e-2)
