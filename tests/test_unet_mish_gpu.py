"""End to end with the mish activation (the reference's `--activation mish`): UNet forward + backward, a training
step (eager and CUDA graph), Euler / Euler-ancestral sampling and a checkpoint round trip, against the CPU oracle
with mish in place of swish (mish_ref.mish_oracle).  Tolerances as in test_unet_gpu.py: forward <= 3e-2 relative
L2, parameter gradients <= 6e-2 per tensor and <= 3e-2 globally, samplers <= 5e-2, loss <= 2e-2."""

import numpy as np
import pytest
import torch

from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import diffusion_ref as R
from mish_ref import mish_oracle
from oracle import train_ref, unet_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def cpu_params(fp, grad=False):
    return {k: v.detach().cpu().clone().requires_grad_(grad) for k, v in fp.named.items()}


def perturbed(model, seed=1):
    fp = model.init(4, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    for name, t in fp.named.items():           # non-trivial norm scales and biases
        leaf = name.rsplit("/", 1)[1]
        if leaf == "bias":
            t.copy_(0.1 * torch.randn(t.shape, generator=g, device=dev))
        elif leaf == "scale":
            t.copy_(1 + 0.1 * torch.randn(t.shape, generator=g, device=dev))
    fp.touch()
    return fp


@pytest.mark.parametrize("res,B,depths,levels", [
    (64, 2, (64, 128, 256, 512), (None,) * 4),
    (32, 2, (64, 128, 256, 512), (None, None, {"heads": 8}, {"heads": 8})),     # the 256^2 config's structure
    (32, 1, (128, 256, 512, 1024), (None, {"heads": 8}, {"heads": 8}, {"heads": 8}))],
    ids=["64px", "self_attention", "wide"])
def test_mish_unet_forward_backward_vs_oracle(res, B, depths, levels):
    torch.manual_seed(0)
    model = Unet(feature_depths=depths, attention_configs=levels, dtype=torch.bfloat16, activation="mish")
    fp = perturbed(model)
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    F, saved = model.forward(fp, x, t, None, save=True)
    P = cpu_params(fp, True)
    with mish_oracle():
        Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(),
                                   feature_depths=depths, attention_configs=levels)
    assert rel(F, Fr) < 3e-2, rel(F, Fr)
    # the swish oracle is far from the mish model: the activation really changed
    with torch.no_grad():
        Fs = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(),
                                   feature_depths=depths, attention_configs=levels)
    assert rel(Fs, Fr) > 6e-2
    dF = torch.randn(B, res, res, 3, device=dev) / (B * res * res * 3)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    (Fr * dF.cpu()).sum().backward()
    num = den = 0.0
    for k in P:
        g, gr = grads.named[k].cpu(), P[k].grad
        assert rel(g, gr) < 6e-2, (k, rel(g, gr))
        num += (g - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    assert (num / den) ** 0.5 < 3e-2


def _trainer(res, graph, **kw):
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16, activation="mish")
    return model, GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                          DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                          model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                          use_cuda_graph=graph, **kw)


@pytest.mark.parametrize("graph", [False, True])
def test_mish_train_step_vs_oracle(graph, monkeypatch):
    torch.manual_seed(0)
    res, B = 16, 4
    model, trainer = _trainer(res, graph)
    P = cpu_params(trainer.state.params, True)
    ema = {k: v.detach().clone() for k, v in P.items()}
    freqs = model._fourier_freqs(dev).cpu()
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8)
    step_fn = trainer._define_train_step(B)
    opt = {}
    for it in range(2):
        noise = torch.randn(B, res, res, 3)
        t = torch.randn(B)
        monkeypatch.setattr(utils, "device_normal",
                            lambda key, shape, device, dtype=torch.float32, _n=noise, _t=t:
                            (_t if len(shape) == 1 else _n).to(device))
        trainer.state, loss, trainer.rngstate = step_fn(trainer.state, trainer.rngstate, {"image": img.clone()}, 0)
        with mish_oracle():
            want = train_ref.edm_train_step(P, opt, img, noise, t, freqs, lr=1e-3, wd=1e-4, ema=ema, step=it + 1)
        assert abs(loss.item() - want.item()) / want.item() < 2e-2, (it, loss.item(), want.item())
    p0 = Unet(attention_configs=(None,) * 4).init(utils.split(utils.PRNGKey(4))[1], device=torch.device("cpu"))
    cos_n = cos_a = cos_b = 0.0
    for k, v in trainer.state.params.named.items():
        d_got = v.cpu() - p0.named[k]
        d_ref = P[k].detach() - p0.named[k]
        cos_n += (d_got * d_ref).sum().item()
        cos_a += d_got.pow(2).sum().item()
        cos_b += d_ref.pow(2).sum().item()
    assert cos_n / (cos_a * cos_b) ** 0.5 > 0.9
    assert torch.isfinite(trainer.state.params.flat).all()


@pytest.mark.parametrize("kind,cls", [("euler", EulerSampler), ("euler_a", EulerAncestralSampler)])
def test_mish_samplers_vs_oracle(kind, cls, monkeypatch):
    torch.manual_seed(0)
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16, activation="mish")
    fp = perturbed(model)
    B, res, n = 2, 16, 4
    sched = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev)
    smp = cls(model, sched, KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (res, res, 3), []))
    prior = torch.randn(B, res, res, 3) * 80.0
    noises = [torch.randn(B, res, res, 3) for _ in range(n)]
    it = iter(noises)
    monkeypatch.setattr(utils, "device_normal", lambda key, shape, device, dtype=torch.float32: next(it).to(device))
    out = smp.generate_samples(fp, B, res, diffusion_steps=n, start_step=1000, priors=prior, device=dev)
    steps = [float(s) for s in smp.get_steps(1000, 0, n)]
    P, freqs = cpu_params(fp), model._fourier_freqs(dev).cpu()
    x = prior.clone()
    for i in range(n):
        cur, nxt = steps[i] / 1000.0, (steps[i + 1] if i + 1 < n else 0) / 1000.0
        with mish_oracle():
            x0, _ = train_ref.karras_denoise_eval(P, x, torch.full((B,), cur), freqs)
        if i == n - 1:
            x = x0.clamp(-1, 1)
            break
        cs = R.karras_sigma(np.full(B, cur, np.float32))
        ns = R.karras_sigma(np.full(B, nxt, np.float32))
        one = np.ones(B, np.float32)
        if kind == "euler":
            x = torch.from_numpy(R.euler_step(x.numpy(), x0.numpy(), one, cs, one, ns))
        else:
            x = torch.from_numpy(R.euler_ancestral_step(x.numpy(), x0.numpy(), noises[i].numpy(), one, cs, one, ns))
    assert out.shape == (B, res, res, 3) and torch.isfinite(out).all()
    assert rel(out, x) < 5e-2


def test_mish_checkpoint_roundtrip(tmp_path):
    """save -> train further -> load restores the parameters of a mish model; the restored model computes the
    mish forward (checked against the oracle)."""
    torch.manual_seed(0)
    res, B = 16, 2
    model, tr = _trainer(res, True, checkpoint_base_path=str(tmp_path), name="mish ck")
    step = tr._define_train_step(B)
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8)
    tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, {"image": img}, 0)
    tr.save(epoch=1, step=1)
    saved = tr.state.params.flat.clone()
    for _ in range(2):
        tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, {"image": img}, 0)
    assert not torch.equal(tr.state.params.flat, saved)
    got_step, st, _, _ = tr.load()
    assert got_step == 1 and torch.equal(st.params.flat, saved)
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    F = model.apply(st.params, x, t, None)
    with mish_oracle():
        Fr = unet_ref.unet_forward(cpu_params(st.params), x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu())
    assert rel(F, Fr) < 3e-2
