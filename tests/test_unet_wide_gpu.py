"""The text-to-image UNet of the reference README's gallery, feature_depths=(128, 256, 512, 1024) with 8-head
attention at the last three levels: its 1024-channel attention blocks (middle_attention_0, up_0_attention_1) have
128-channel heads and run on the head-width-128 attention kernels.  Checked against the CPU oracle with the
tolerances of tests/test_unet_gpu.py: forward <= 3e-2, global gradient <= 3e-2, every parameter gradient <= 6e-2
(8e-2 with a text context); training loss <= 2e-2; sampler output <= 6e-2."""
import functools

import numpy as np
import pytest
import torch

from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import diffusion_ref as R
from oracle import train_ref, unet_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

DEPTHS = (128, 256, 512, 1024)
GALLERY = (None, {"heads": 8}, {"heads": 8}, {"heads": 8})
FULL = {"heads": 8, "only_pure_attention": False, "use_projection": True}


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def cpu_params(fp, grad=False):
    return {k: v.detach().cpu().clone().requires_grad_(grad) for k, v in fp.named.items()}


def perturbed(model, seed=2):
    fp = model.init(4, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    for name, t in fp.named.items():           # non-trivial norm scales and biases
        if name.endswith("scale"):
            t.copy_(1 + 0.1 * torch.randn(t.shape, generator=g, device=dev))
        elif name.endswith("bias"):
            t.copy_(0.05 * torch.randn(t.shape, generator=g, device=dev))
    fp.touch()
    return fp


@pytest.mark.parametrize("levels,ctxdim,tol", [(GALLERY, None, 6e-2), (GALLERY, 768, 8e-2),
                                               ((None, None, None, FULL), 768, 8e-2)],
                         ids=["self_attention", "text_context", "full_block"])
def test_wide_unet_forward_backward_vs_oracle(levels, ctxdim, tol):
    torch.manual_seed(0)
    model = Unet(feature_depths=DEPTHS, attention_configs=levels, dtype=torch.bfloat16, context_dim=ctxdim)
    fp = perturbed(model)
    B, res = 2, 64
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    ctx = torch.randn(B, 77, 768, device=dev).bfloat16() if ctxdim else None
    F, saved = model.forward(fp, x, t, ctx, save=True)
    P = cpu_params(fp, True)
    Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), feature_depths=DEPTHS,
                               attention_configs=levels, textcontext=None if ctx is None else ctx.float().cpu())
    assert rel(F, Fr) < 3e-2, rel(F, Fr)
    dF = torch.randn(B, res, res, 3, device=dev) / (B * res * res * 3)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    (Fr * dF.cpu()).sum().backward()
    num = den = 0.0
    for k in P:
        g, gr = grads.named[k].cpu(), P[k].grad
        assert rel(g, gr) < tol, (k, rel(g, gr))
        num += (g - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    assert (num / den) ** 0.5 < 3e-2


@pytest.mark.parametrize("graph", [False, True])
def test_wide_unet_train_step_vs_oracle(graph, monkeypatch):
    """Two EDM training steps of the gallery model (eager and CUDA-graphed) against oracle/train_ref.py."""
    torch.manual_seed(0)
    res, B = 32, 2
    model = Unet(feature_depths=DEPTHS, attention_configs=GALLERY, dtype=torch.bfloat16)
    trainer = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                      DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                      model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                      use_cuda_graph=graph)
    # the oracle training step builds the default-width UNet; give it the gallery widths
    monkeypatch.setattr(unet_ref, "unet_forward", functools.partial(unet_ref.unet_forward, feature_depths=DEPTHS))
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
        want = train_ref.edm_train_step(P, opt, img, noise, t, freqs, attention_configs=GALLERY, lr=1e-3, wd=1e-4,
                                        ema=ema, step=it + 1)
        assert abs(loss.item() - want.item()) / want.item() < 2e-2, (it, loss.item(), want.item())
    p0 = Unet(feature_depths=DEPTHS, attention_configs=GALLERY).init(utils.split(utils.PRNGKey(4))[1],
                                                                      device=torch.device("cpu"))
    cos_n = cos_a = cos_b = 0.0
    for k, v in trainer.state.params.named.items():
        d_got = v.cpu() - p0.named[k]
        d_ref = P[k].detach() - p0.named[k]
        cos_n += (d_got * d_ref).sum().item()
        cos_a += d_got.pow(2).sum().item()
        cos_b += d_ref.pow(2).sum().item()
    assert cos_n / (cos_a * cos_b) ** 0.5 > 0.9
    assert torch.isfinite(trainer.state.params.flat).all()


def test_wide_unet_cfg_euler_ancestral_sampling_vs_oracle(monkeypatch):
    """Three classifier-free-guided Euler-ancestral steps of the gallery model with a 77 x 768 text context."""
    from flaxdiff_b200.inputs import ConditionalInputConfig, RandomEmbeddingEncoder
    torch.manual_seed(0)
    model = Unet(feature_depths=DEPTHS, attention_configs=GALLERY, dtype=torch.bfloat16, context_dim=768)
    fp = model.init(4, device=dev)
    enc = RandomEmbeddingEncoder(77, 768, device=dev)
    cfg = DiffusionInputConfig("image", (32, 32, 3), [ConditionalInputConfig(enc)])
    sched = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev)
    g = 3.0
    smp = EulerAncestralSampler(model, sched, KarrasPredictionTransform(0.5), cfg, guidance_scale=g)
    B, res, n = 2, 32, 3
    prior = torch.randn(B, res, res, 3) * 80.0
    noises = [torch.randn(B, res, res, 3) for _ in range(n)]
    it = iter(noises)
    monkeypatch.setattr(utils, "device_normal", lambda key, shape, device, dtype=torch.float32: next(it).to(device))
    cond = enc(["a cat", "a dog"]).to(dev)
    out = smp.generate_samples(fp, B, res, diffusion_steps=n, start_step=1000, priors=prior, device=dev,
                               model_conditioning_inputs=(cond,))
    P, freqs = cpu_params(fp), model._fourier_freqs(dev).cpu()
    null = cfg.get_unconditionals()[0].cpu().expand(B, -1, -1)
    steps = [float(s) for s in smp.get_steps(1000, 0, n)]
    x = prior.clone()
    for i, s in enumerate(steps):
        cur, nxt = s / 1000.0, (steps[i + 1] if i + 1 < n else 0) / 1000.0
        sig = R.karras_sigma(np.full(B, cur, np.float32))
        c_in, c_out, c_skip = (torch.from_numpy(a).view(-1, 1, 1, 1) for a in R.karras_coeffs(sig))
        tm = torch.from_numpy(R.karras_model_time(sig))
        with torch.no_grad():
            Fc = unet_ref.unet_forward(P, x * c_in, tm, freqs, feature_depths=DEPTHS, attention_configs=GALLERY,
                                       textcontext=cond.float().cpu())
            Fu = unet_ref.unet_forward(P, x * c_in, tm, freqs, feature_depths=DEPTHS, attention_configs=GALLERY,
                                       textcontext=null.float())
        Fm = Fu + g * (Fc - Fu)
        x0 = c_out * Fm + c_skip * x
        if i == n - 1:
            x = x0.clamp(-1, 1)
            break
        ns = R.karras_sigma(np.full(B, nxt, np.float32))
        one = np.ones(B, np.float32)
        x = torch.from_numpy(R.euler_ancestral_step(x.numpy(), x0.numpy(), noises[i].numpy(), one, sig, one, ns))
    assert rel(out, x) < 6e-2
