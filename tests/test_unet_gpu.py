"""End-to-end parity of the UNet hot path (forward, backward, sampling, one training step) on the GPU
against the CPU oracle with identical parameters and injected (x0, eps, t) tensors.

Stated tolerances (bf16 tensor-core path vs fp32 oracle; reference's own bf16 mode has the same budget):
  UNet forward   relative L2 error <= 3e-2         (measured ~9e-3)
  parameter grads every tensor <= 6e-2, global <= 3e-2   (measured ~1.3e-2)
  sampler output after N steps <= 5e-2; training loss <= 2e-2 relative."""
import numpy as np
import pytest
import torch

from flaxdiff_b200 import ops, utils
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.predictors import EpsilonPredictionTransform, KarrasPredictionTransform
from flaxdiff_b200.samplers import DDIMSampler, DDPMSampler, EulerAncestralSampler, EulerSampler, HeunSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler, LinearNoiseSchedule
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import diffusion_ref as R
from oracle import train_ref, unet_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def make_model(attn, seed=4, perturb=True):
    acfg = (None, None, None, {"heads": 8}) if attn else (None,) * 4
    model = Unet(attention_configs=acfg, dtype=torch.bfloat16)
    fp = model.init(seed, device=dev)
    if perturb:
        g = torch.Generator(device=dev)
        g.manual_seed(1)
        for name, t in fp.named.items():
            leaf = name.rsplit("/", 1)[1]
            if leaf == "bias":
                t.copy_(0.1 * torch.randn(t.shape, generator=g, device=dev))
            elif leaf == "scale":
                t.copy_(1 + 0.1 * torch.randn(t.shape, generator=g, device=dev))
    return model, fp, acfg


def cpu_params(fp, grad=False):
    return {k: v.detach().cpu().clone().requires_grad_(grad) for k, v in fp.named.items()}


@pytest.mark.parametrize("res,B,attn", [(32, 2, False), (64, 2, True), (16, 3, False), (64, 1, True),
                                        (48, 2, False)])
def test_unet_forward_backward_vs_oracle(res, B, attn):
    torch.manual_seed(0)
    model, fp, acfg = make_model(attn)
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    F, saved = model.forward(fp, x, t, None, save=True)
    P = cpu_params(fp, True)
    Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), attention_configs=acfg)
    assert rel(F, Fr) < 3e-2
    dF = torch.randn(B, res, res, 3, device=dev) / (B * res * res * 3)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    (Fr * dF.cpu()).sum().backward()
    num = den = 0.0
    for k in P:
        g, gr = grads.named[k].cpu(), P[k].grad
        assert rel(g, gr) < 6e-2, k
        num += (g - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    assert (num / den) ** 0.5 < 3e-2


def test_apply_accepts_plain_flax_tree_and_is_deterministic():
    model, fp, acfg = make_model(False)
    x = torch.randn(2, 16, 16, 3, device=dev)
    t = torch.tensor([0.3, -0.7], device=dev)
    tree = {"params": {k: v for k, v in fp["params"].items()}}
    y1 = model.apply(fp, x, t, None)
    y2 = model.apply(tree, x, t, None)
    # f32 atomics in the GroupNorm statistics make runs differ at the 1e-3 level after bf16 rounding
    assert y1.shape == (2, 16, 16, 3) and rel(y1, y2) < 1e-2


def _oracle_sample(kind, P, freqs, x, steps, acfg, noises):
    """Oracle sampling loop (samplers/common.py:382-395) with KarrasVE schedule + Karras transform."""
    x = x.clone()
    n = len(steps)
    for i in range(n):
        cur = steps[i] / 1000.0
        nxt = (steps[i + 1] if i + 1 < n else 0) / 1000.0
        B = x.shape[0]
        tcur = torch.full((B,), cur)
        x0, eps = train_ref.karras_denoise_eval(P, x, tcur, freqs, attention_configs=acfg)
        if i == n - 1:
            return x0.clamp(-1, 1)
        cs = R.karras_sigma(np.full(B, cur, np.float32))
        ns = R.karras_sigma(np.full(B, nxt, np.float32))
        one = np.ones(B, np.float32)
        if kind == "euler":
            x = torch.from_numpy(R.euler_step(x.numpy(), x0.numpy(), one, cs, one, ns))
        elif kind == "euler_a":
            x = torch.from_numpy(R.euler_ancestral_step(x.numpy(), x0.numpy(), noises[i].numpy(), one, cs, one, ns))
        elif kind == "heun":
            def second(xp):
                return train_ref.karras_denoise_eval(P, torch.from_numpy(xp), torch.full((B,), nxt), freqs,
                                                     attention_configs=acfg)[0].numpy()
            x = torch.from_numpy(R.heun_step(x.numpy(), x0.numpy(), second, one, cs, one, ns).astype(np.float32))
        elif kind == "ddim":
            x = torch.from_numpy(R.ddim_step(x0.numpy(), eps.numpy(), one, ns).astype(np.float32))
    return x


@pytest.mark.parametrize("kind,cls", [("euler", EulerSampler), ("heun", HeunSampler), ("ddim", DDIMSampler),
                                      ("euler_a", EulerAncestralSampler)])
@pytest.mark.parametrize("graph", [True, False])
def test_samplers_vs_oracle(kind, cls, graph, monkeypatch):
    if kind == "euler_a" and graph:
        pytest.skip("one configuration is enough for the ancestral sampler")
    torch.manual_seed(0)
    model, fp, acfg = make_model(False)
    B, res, n = 2, 16, 4
    sched = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev)
    smp = cls(model, sched, KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (res, res, 3), []),
              use_cuda_graph=graph)
    prior = torch.randn(B, res, res, 3) * 80.0
    noises = [torch.randn(B, res, res, 3) for _ in range(n)]
    it = iter(noises)
    monkeypatch.setattr(utils, "device_normal", lambda key, shape, device, dtype=torch.float32: next(it).to(device))
    out = smp.generate_samples(fp, B, res, diffusion_steps=n, start_step=1000, priors=prior, device=dev)
    steps = [float(s) for s in smp.get_steps(1000, 0, n)]
    want = _oracle_sample(kind, cpu_params(fp), model._fourier_freqs(dev).cpu(), prior, steps, acfg, noises)
    assert out.shape == (B, res, res, 3) and torch.isfinite(out).all()
    assert rel(out, want) < 5e-2


def test_ddpm_sampler_vs_oracle(monkeypatch):
    torch.manual_seed(0)
    model, fp, acfg = make_model(False)
    B, res, n = 2, 16, 3
    sched = LinearNoiseSchedule(1000).to(dev)
    smp = DDPMSampler(model, sched, EpsilonPredictionTransform(), DiffusionInputConfig("image", (res, res, 3), []))
    prior = torch.randn(B, res, res, 3)
    noises = [torch.randn(B, res, res, 3) for _ in range(n)]
    it = iter(noises)
    monkeypatch.setattr(utils, "device_normal", lambda key, shape, device, dtype=torch.float32: next(it).to(device))
    out = smp.generate_samples(fp, B, res, diffusion_steps=n, start_step=1000, priors=prior, device=dev)
    # oracle loop: discrete table gathers with JAX clamping (start index 1000 -> 999)
    P, freqs = cpu_params(fp), model._fourier_freqs(dev).cpu()
    T = R.linear_tables(1000)
    steps = [float(s) for s in smp.get_steps(1000, 0, n)]
    x = prior.clone()
    for i, s in enumerate(steps):
        idx = int(R.discrete_index([s])[0])
        a, sg = T["sqrt_alpha_cumprod"][idx], T["sqrt_one_minus_alpha_cumprod"][idx]
        with torch.no_grad():
            F = unet_ref.unet_forward(P, x, torch.full((B,), s), freqs, attention_configs=acfg)
        x0 = (x - F * float(sg)) / float(a)
        if i == n - 1:
            x = x0.clamp(-1, 1)
            break
        x = torch.from_numpy(R.ddpm_step(x0.numpy(), x.numpy(), noises[i].numpy(),
                                         np.full(B, T["posterior_mean_coef1"][idx]),
                                         np.full(B, T["posterior_mean_coef2"][idx]),
                                         np.full(B, T["posterior_log_variance_clipped"][idx])).astype(np.float32))
    assert rel(out, x) < 5e-2


@pytest.mark.parametrize("graph", [False, True])
def test_train_step_vs_oracle(graph, monkeypatch):
    torch.manual_seed(0)
    res, B = 16, 4
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16)
    trainer = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                      DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                      model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                      use_cuda_graph=graph)
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
        want = train_ref.edm_train_step(P, opt, img, noise, t, freqs, lr=1e-3, wd=1e-4, ema=ema, step=it + 1)
        assert abs(loss.item() - want.item()) / want.item() < 2e-2, (it, loss.item(), want.item())
    # after two AdamW steps parameters stay close (sign-like first update: compare the update direction)
    got = trainer.state.params.flat.cpu()
    p0 = Unet(attention_configs=(None,) * 4).init(utils.split(utils.PRNGKey(4))[1], device=torch.device("cpu"))
    num = den = 0.0
    cos_n = cos_a = cos_b = 0.0
    for k, v in trainer.state.params.named.items():
        d_got = v.cpu() - p0.named[k]
        d_ref = P[k].detach() - p0.named[k]
        cos_n += (d_got * d_ref).sum().item()
        cos_a += d_got.pow(2).sum().item()
        cos_b += d_ref.pow(2).sum().item()
    assert cos_n / (cos_a * cos_b) ** 0.5 > 0.9
    assert torch.isfinite(got).all()
    assert rel(trainer.state.params.shadow_flat_noupdate().float(), trainer.state.params.flat) < 4e-3


@pytest.mark.parametrize("graph", [False, True])
def test_ddpm_train_step_vs_oracle(graph, monkeypatch):
    """BASELINE configs[0] (the reference's own CPU-runnable case): unconditional DDPM UNet,
    LinearNoiseSchedule(1000), epsilon prediction - two training steps against the oracle."""
    torch.manual_seed(0)
    res, B = 16, 4
    model = Unet(attention_configs=(None,) * 4, dtype=torch.bfloat16)
    trainer = GeneralDiffusionTrainer(model, adamw(1e-3), LinearNoiseSchedule(1000),
                                      DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                      model_output_transform=EpsilonPredictionTransform(), device=dev,
                                      use_cuda_graph=graph)
    P = cpu_params(trainer.state.params, True)
    ema = {k: v.detach().clone() for k, v in P.items()}
    freqs = model._fourier_freqs(dev).cpu()
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8)
    step_fn = trainer._define_train_step(B)
    opt = {}
    for it, t in enumerate((torch.tensor([3, 250, 640, 999]), torch.tensor([0, 17, 500, 998]))):
        noise = torch.randn(B, res, res, 3)
        monkeypatch.setattr(utils, "device_normal",
                            lambda key, shape, device, dtype=torch.float32, _n=noise: _n.to(device))
        monkeypatch.setattr(utils, "device_randint",
                            lambda key, shape, lo, hi, device, _t=t: _t.to(device=device, dtype=torch.int32))
        trainer.state, loss, trainer.rngstate = step_fn(trainer.state, trainer.rngstate, {"image": img.clone()}, 0)
        want = train_ref.ddpm_train_step(P, opt, img, noise, t, freqs, lr=1e-3, wd=1e-4, ema=ema, step=it + 1)
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


@pytest.mark.parametrize("res,B,levels", [(32, 2, (None, {"heads": 8}, {"heads": 8}, {"heads": 8})),
                                          (64, 1, (None, None, {"heads": 8}, {"heads": 8}))])
def test_text_cross_attention_forward_backward_vs_oracle(res, B, levels):
    """BASELINE config 4 structure: cross-attention to a (B, 77, 768) text context at several levels
    (head widths 8..64, 77 keys padded to 96)."""
    torch.manual_seed(0)
    model = Unet(attention_configs=levels, dtype=torch.bfloat16, context_dim=768)
    fp = model.init(4, device=dev)
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    ctx = torch.randn(B, 77, 768, device=dev).bfloat16()
    F, saved = model.forward(fp, x, t, ctx, save=True)
    P = cpu_params(fp, True)
    Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), attention_configs=levels,
                               textcontext=ctx.float().cpu())
    assert rel(F, Fr) < 3e-2
    dF = torch.randn(B, res, res, 3, device=dev) / (B * res * res * 3)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    (Fr * dF.cpu()).sum().backward()
    num = den = 0.0
    for k in P:
        g, gr = grads.named[k].cpu(), P[k].grad
        assert rel(g, gr) < 8e-2, k
        num += (g - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    assert (num / den) ** 0.5 < 3e-2


def test_cfg_euler_ancestral_sampling_vs_oracle(monkeypatch):
    """Classifier-free guidance batching (samplers/common.py:70-96) with frozen random text embeddings."""
    from flaxdiff_b200.inputs import ConditionalInputConfig, RandomEmbeddingEncoder
    torch.manual_seed(0)
    levels = (None, None, {"heads": 8}, {"heads": 8})
    model = Unet(attention_configs=levels, dtype=torch.bfloat16, context_dim=768)
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
    # oracle: same loop with F = Fu + g (Fc - Fu)
    P, freqs = cpu_params(fp), model._fourier_freqs(dev).cpu()
    null = cfg.get_unconditionals()[0].cpu().expand(B, -1, -1)
    steps = [float(s) for s in smp.get_steps(1000, 0, n)]
    x = prior.clone()
    for i, s in enumerate(steps):
        cur, nxt = s / 1000.0, (steps[i + 1] if i + 1 < n else 0) / 1000.0
        sig = R.karras_sigma(np.full(B, cur, np.float32))
        s4 = torch.from_numpy(sig).view(-1, 1, 1, 1)
        c_in, c_out, c_skip = (torch.from_numpy(a).view(-1, 1, 1, 1) for a in R.karras_coeffs(sig))
        tm = torch.from_numpy(R.karras_model_time(sig))
        with torch.no_grad():
            Fc = unet_ref.unet_forward(P, x * c_in, tm, freqs, attention_configs=levels, textcontext=cond.float().cpu())
            Fu = unet_ref.unet_forward(P, x * c_in, tm, freqs, attention_configs=levels, textcontext=null.float())
        Fm = Fu + g * (Fc - Fu)
        x0 = c_out * Fm + c_skip * x
        if i == n - 1:
            x = x0.clamp(-1, 1)
            break
        ns = R.karras_sigma(np.full(B, nxt, np.float32))
        one = np.ones(B, np.float32)
        x = torch.from_numpy(R.euler_ancestral_step(x.numpy(), x0.numpy(), noises[i].numpy(), one, sig, one, ns))
    assert rel(out, x) < 6e-2


FULL_BLOCKS = [
    # (attention config, context_dim)
    ({"heads": 8, "only_pure_attention": False}, None),                                  # self + "cross to itself" + FF
    ({"heads": 8, "only_pure_attention": False, "use_projection": True}, 768),           # the full text block
    ({"heads": 8, "only_pure_attention": False, "use_self_and_cross": False}, 768),      # cross + FF only
    ({"heads": 8, "only_pure_attention": True, "use_projection": True}, None),           # projections around pure attention
]


@pytest.mark.parametrize("cfg,ctxdim", FULL_BLOCKS)
def test_full_transformer_block_forward_backward_vs_oracle(cfg, ctxdim):
    """SURVEY $8 f3: only_pure_attention=False (self-attention + cross-attention + GEGLU feed-forward) and
    use_projection=True (models/attention.py:179-303, 327-374) at the 8x8 (C=512, d=64) and 16x16 (C=256,
    d=32) levels of a 64x64 UNet, against the oracle restatement."""
    torch.manual_seed(0)
    levels = (None, None, cfg, cfg)
    model = Unet(attention_configs=levels, dtype=torch.bfloat16, context_dim=ctxdim)
    fp = model.init(4, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(2)
    for name, t in fp.named.items():           # non-trivial norm scales and feed-forward biases
        if name.endswith("scale"):
            t.copy_(1 + 0.1 * torch.randn(t.shape, generator=g, device=dev))
        elif name.endswith("bias"):
            t.copy_(0.05 * torch.randn(t.shape, generator=g, device=dev))
    fp.touch()
    B, res = 2, 64
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    ctx = torch.randn(B, 77, 768, device=dev).bfloat16() if ctxdim else None
    F, saved = model.forward(fp, x, t, ctx, save=True)
    P = cpu_params(fp, True)
    Fr = unet_ref.unet_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), attention_configs=levels,
                               textcontext=None if ctx is None else ctx.float().cpu())
    assert rel(F, Fr) < 3e-2, rel(F, Fr)
    dF = torch.randn(B, res, res, 3, device=dev) / (B * res * res * 3)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    (Fr * dF.cpu()).sum().backward()
    num = den = 0.0
    for k in P:
        gg, gr = grads.named[k].cpu(), P[k].grad
        assert rel(gg, gr) < 8e-2, (k, rel(gg, gr))
        num += (gg - gr).pow(2).sum().item()
        den += gr.pow(2).sum().item()
    assert (num / den) ** 0.5 < 3e-2
