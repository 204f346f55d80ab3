"""SimpleDiT on the GPU: forward and every parameter gradient against the fp32 oracle (oracle/dit_ref.py), the trainer's
eager and graphed steps, a short fit on a fixed batch, Euler / Euler-ancestral sampling and a checkpoint round trip.
Tolerances are the UNet's: forward <= 3e-2 relative L2, each gradient <= 6e-2."""
import numpy as np
import pytest
import torch

from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.simple_dit import SimpleDiT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import dit_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _live_params(model, seed, ctx=None):
    """init, then random ada_proj / final_proj kernels and biases so every gate and modulation is live."""
    fp = model.init(seed, textcontext=ctx, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, t in fp.named.items():
        if "ada_proj" in name or name.startswith("final_proj") or name.endswith("bias"):
            t.copy_(0.2 * torch.randn(t.shape, generator=g, device=dev))
    return fp


CONFIGS = {
    "f64_d32_p2": dict(kw=dict(patch_size=2, emb_features=64, num_layers=2, num_heads=2), res=(16, 16), text=None),
    "f192_d48_p4_sigma": dict(kw=dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4, learn_sigma=True),
                              res=(32, 16), text=None),
    "f128_d64_p2_text": dict(kw=dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2), res=(16, 16),
                             text=(7, 64)),
}


@pytest.mark.parametrize("case", sorted(CONFIGS))
def test_forward_and_gradients_match_oracle(case):
    cfg = CONFIGS[case]
    torch.manual_seed(0)
    B, (H, W) = 2, cfg["res"]
    ctx = torch.randn(B, *cfg["text"], device=dev) if cfg["text"] else None
    model = SimpleDiT(**cfg["kw"])
    fp = _live_params(model, 3, ctx)
    x = torch.randn(B, H, W, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    Fo, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(B, H, W, 3, device=dev)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    torch.cuda.synchronize()
    P = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fp.named.items()}
    kw = {k: v for k, v in cfg["kw"].items() if k in ("patch_size", "num_layers", "num_heads")}
    Fr = dit_ref.simple_dit_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(),
                                    textcontext=None if ctx is None else ctx.cpu(), **kw)
    (Fr * dF.cpu()).sum().backward()
    assert rel(Fo, Fr) < 3e-2, rel(Fo, Fr)
    bad = {}
    for k in P:
        ref = P[k].grad
        if ref.norm() == 0:                      # the unused learn_sigma half of final_proj
            assert grads.named[k].abs().max().item() == 0, k
            continue
        e = rel(grads.named[k], ref)
        if e >= 6e-2:
            bad[k] = e
    assert not bad, bad


def _trainer(graph, model=None, res=16):
    model = model or SimpleDiT(patch_size=2, emb_features=128, num_layers=2, num_heads=2)
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 use_cuda_graph=graph)
    return model, tr


def _batch(seed=0, B=4, res=16):
    rng = np.random.default_rng(seed)
    return {"image": torch.from_numpy(rng.integers(0, 256, (B, res, res, 3), dtype=np.uint8))}


def test_eager_and_graphed_trainer_steps_agree():
    _, eager = _trainer(False)
    _, graphed = _trainer(True)
    se, sg = eager._define_train_step(), graphed._define_train_step()
    stE, stG, rE, rG = eager.state, graphed.state, eager.rngstate, graphed.rngstate
    for i in range(3):
        b = _batch(i)
        stE, lE, rE = se(stE, rE, b)
        stG, lG, rG = sg(stG, rG, b)
        assert abs(lE.item() - lG.item()) <= 1e-3 * abs(lE.item()), (i, lE.item(), lG.item())
    assert rel(stG.params.flat, stE.params.flat) < 1e-3


def test_loss_decreases_on_a_fixed_batch():
    _, tr = _trainer(True)
    step = tr._define_train_step()
    st, r = tr.state, tr.rngstate
    b = _batch(7)
    losses = []
    for _ in range(30):
        st, loss, _ = step(st, r, b)            # same key every step: same noise and timesteps
        losses.append(loss.item())
    assert np.isfinite(losses).all() and np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses


@pytest.mark.parametrize("cls", [EulerSampler, EulerAncestralSampler])
def test_sampling_whole_step_graph_matches_eager(cls):
    model = SimpleDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2)
    fp = _live_params(model, 5)
    sched, tr = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev), KarrasPredictionTransform(0.5)
    cfg = DiffusionInputConfig("image", (16, 16, 3), [])
    key = utils.RandomMarkovState(utils.ThreefryKey(utils.PRNGKey(11)))
    outs = []
    for graph in (False, True):
        smp = cls(model, sched, tr, cfg, use_cuda_graph=graph)
        outs.append(smp.generate_samples(fp, 2, 16, diffusion_steps=6, start_step=1000, device=dev,
                                         rngstate=utils.RandomMarkovState(key.rng)))
    assert outs[0].shape == (2, 16, 16, 3) and torch.isfinite(outs[1]).all()
    assert rel(outs[1], outs[0]) < 1e-2


def test_checkpoint_round_trip(tmp_path):
    model, tr = _trainer(True)
    step = tr._define_train_step()
    tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, _batch(1))
    tr.save(0, 1, path=str(tmp_path))
    _, tr2 = _trainer(False, SimpleDiT(**model.config()))
    tr2.load(checkpoint_path=str(tmp_path))
    assert torch.equal(tr2.state.params.flat, tr.state.params.flat)
    assert torch.equal(tr2.state.opt_state["mu"], tr.state.opt_state["mu"])
    assert tr2.state.step == tr.state.step
