"""UNets with 256-channel attention heads: the default feature_depths (64, 128, 256, 512) with 2 heads (the
reference's `--attention_heads 2`), whose 512-channel middle and up_0 attention blocks run on the head-width-256
attention kernels, and (128, 256, 512, 1024) with 4 heads.  Checked against the CPU oracle with the tolerances of
tests/test_unet_gpu.py: forward <= 3e-2, global gradient <= 3e-2, every parameter gradient <= 6e-2 (8e-2 with a
text context); training loss <= 2e-2; sampler output <= 6e-2."""
import numpy as np
import pytest
import torch

import test_attention_launches_gpu as launches
from flaxdiff_b200 import utils
from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import diffusion_ref as R
from oracle import train_ref, unet_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

TWO = (None, {"heads": 2}, {"heads": 2}, {"heads": 2})
FULL2 = {"heads": 2, "only_pure_attention": False, "use_projection": True}
WIDE = (128, 256, 512, 1024)
FOUR = (None, {"heads": 4}, {"heads": 4}, {"heads": 4})


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


@pytest.mark.parametrize("depths,levels,ctxdim,tol", [
    ((64, 128, 256, 512), TWO, None, 6e-2),
    ((64, 128, 256, 512), (None, None, FULL2, FULL2), None, 6e-2),
    (WIDE, FOUR, 768, 8e-2)],
    ids=["two_heads", "two_heads_full_block", "four_heads_text_context"])
def test_heads256_unet_forward_backward_vs_oracle(depths, levels, ctxdim, tol):
    torch.manual_seed(0)
    model = Unet(feature_depths=depths, attention_configs=levels, dtype=torch.bfloat16, context_dim=ctxdim)
    fp = perturbed(model)
    B, res = 2, 64
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    ctx = torch.randn(B, 77, 768, device=dev).bfloat16() if ctxdim else None
    F, saved = model.forward(fp, x, t, ctx, save=True)
    P = cpu_params(fp, True)
    Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), feature_depths=depths,
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


def test_head_width_512_is_refused_at_the_first_forward():
    model = Unet(attention_configs=(None, None, None, {"heads": 1}), dtype=torch.bfloat16)
    fp = model.init(4, device=dev)
    x = torch.randn(1, 16, 16, 3, device=dev).bfloat16()
    with pytest.raises(FdxError, match="head width 512 > 256 is not supported"):
        model.forward(fp, x, torch.randn(1, device=dev), None)


def _trainer(res, graph, **kw):
    model = Unet(attention_configs=TWO, dtype=torch.bfloat16)
    return model, GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                          DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                          model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                          use_cuda_graph=graph, **kw)


def test_heads256_train_step_eager_and_graph_vs_oracle(monkeypatch):
    """Two EDM training steps of the 2-head UNet, eager and CUDA-graphed from the same start, against
    oracle/train_ref.py and against each other."""
    torch.manual_seed(0)
    res, B = 32, 2
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8)
    draws = [(torch.randn(B, res, res, 3), torch.randn(B)) for _ in range(2)]
    losses, params = {}, {}
    for graph in (False, True):
        model, trainer = _trainer(res, graph)
        P = cpu_params(trainer.state.params, True)
        ema = {k: v.detach().clone() for k, v in P.items()}
        freqs = model._fourier_freqs(dev).cpu()
        step_fn = trainer._define_train_step(B)
        opt, losses[graph] = {}, []
        for it, (noise, t) in enumerate(draws):
            monkeypatch.setattr(utils, "device_normal",
                                lambda key, shape, device, dtype=torch.float32, _n=noise, _t=t:
                                (_t if len(shape) == 1 else _n).to(device))
            trainer.state, loss, trainer.rngstate = step_fn(trainer.state, trainer.rngstate, {"image": img.clone()}, 0)
            want = train_ref.edm_train_step(P, opt, img, noise, t, freqs, attention_configs=TWO, lr=1e-3, wd=1e-4,
                                            ema=ema, step=it + 1)
            assert abs(loss.item() - want.item()) / want.item() < 2e-2, (graph, it, loss.item(), want.item())
            losses[graph].append(loss.item())
        params[graph] = trainer.state.params.flat.clone()
        assert torch.isfinite(params[graph]).all()
    for a, b in zip(losses[False], losses[True]):
        assert abs(a - b) / abs(a) < 1e-2, (losses[False], losses[True])
    assert rel(params[True], params[False]) < 1e-2


@pytest.mark.parametrize("kind,cls", [("euler", EulerSampler), ("euler_a", EulerAncestralSampler)])
def test_heads256_samplers_vs_oracle(kind, cls, monkeypatch):
    torch.manual_seed(0)
    model = Unet(attention_configs=TWO, dtype=torch.bfloat16)
    fp = perturbed(model)
    B, res, n = 2, 32, 3
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
        x0, _ = train_ref.karras_denoise_eval(P, x, torch.full((B,), cur), freqs, attention_configs=TWO)
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
    assert rel(out, x) < 6e-2


def test_heads256_cfg_euler_ancestral_with_text_context_vs_oracle(monkeypatch):
    """Three classifier-free-guided Euler-ancestral steps of the 4-head (128 .. 1024) UNet, 77 x 768 context."""
    torch.manual_seed(0)
    model = Unet(feature_depths=WIDE, attention_configs=FOUR, dtype=torch.bfloat16, context_dim=768)
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
            Fc = unet_ref.unet_forward(P, x * c_in, tm, freqs, feature_depths=WIDE, attention_configs=FOUR,
                                       textcontext=cond.float().cpu())
            Fu = unet_ref.unet_forward(P, x * c_in, tm, freqs, feature_depths=WIDE, attention_configs=FOUR,
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


def test_heads256_checkpoint_roundtrip(tmp_path):
    """save -> train further -> load restores the 2-head model's parameters, and the restored model's forward
    matches the oracle."""
    torch.manual_seed(0)
    res, B = 16, 2
    model, tr = _trainer(res, True, checkpoint_base_path=str(tmp_path), name="heads256 ck")
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
    Fr = unet_ref.unet_forward(cpu_params(st.params), x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(),
                               attention_configs=TWO)
    assert rel(F, Fr) < 3e-2


@pytest.mark.parametrize("block", ["pure_self", "pure_text", "full_both_proj_self", "full_text"])
def test_width256_adds_no_launches(block, monkeypatch):
    """(C, heads) = (512, 2) issues as many kernels as the 64-wide heads of (512, 8): width adds no launches."""
    monkeypatch.setitem(launches.WIDTHS, 256, (512, 2))
    before = launches.launch_count()
    F, grads = launches.unet_fwd_bwd(block, 256, dev)
    torch.cuda.synchronize()
    assert launches.launch_count() - before == launches.LAUNCHES[block][64]
    assert torch.isfinite(F).all() and torch.isfinite(grads.flat).all()
