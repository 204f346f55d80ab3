"""SimpleUDiT on the GPU: forward and every parameter gradient against the CPU oracle (oracle/udit_ref.py) - 3-D text
with learn_sigma, 2-D text, no text, the Hilbert order on a 6 x 4 grid, num_layers 2 and 4 - then the trainer's eager
and graphed steps (with random text embeddings and with the in-graph fdx CLIP text tower), a short fit on a fixed
batch, Euler / Euler-ancestral sampling and a checkpoint round trip.  Tolerances are SimpleDiT's: forward <= 3e-2
relative L2, each gradient <= 6e-2.

The ada, up_dense, final_proj and bias values are random, so no gate, skip weight or output weight sits at its init."""
import numpy as np
import pytest
import torch

from clip_text_ref import Tok, clip_model, token_batch
from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.udit import SimpleUDiT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import udit_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _live_params(model, seed, ctx=None):
    """init, then random ada_proj / up_dense / final_proj kernels and every bias.  The ada kernels are scaled by
    0.5 / sqrt(F), as in test_mmdit_gpu.py, so that the modulations and gates stay O(1) at every width and with text
    added to the conditioning: larger ones amplify the bf16 rounding of the early layers' gradients through the U's
    two paths past the tolerance, whatever the program does."""
    fp = model.init(seed, textcontext=ctx, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    F = model.emb_features
    for name, t in fp.named.items():
        if "ada_proj" in name or name.startswith("final_proj") or name.endswith("bias"):
            std = 0.5 / F ** 0.5 if name.endswith("ada_proj/kernel") else 0.2
            t.copy_(std * torch.randn(t.shape, generator=g, device=dev))
        elif name.startswith("up_dense_"):
            t.copy_(torch.randn(t.shape, generator=g, device=dev) / (2 * F) ** 0.5)
    return fp


CONFIGS = {
    "text3d_sigma": dict(kw=dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2, learn_sigma=True),
                         res=(16, 16), text=(7, 64)),
    "text2d_d48": dict(kw=dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4), res=(32, 16),
                       text=(96,)),
    "notext_layers4": dict(kw=dict(patch_size=2, emb_features=128, num_layers=4, num_heads=2), res=(16, 16),
                           text=None),
    "hilbert_6x4": dict(kw=dict(patch_size=4, emb_features=64, num_layers=4, num_heads=2, use_hilbert=True),
                        res=(24, 16), text=(5, 64)),
}


@pytest.mark.parametrize("case", sorted(CONFIGS))
def test_forward_and_gradients_match_oracle(case):
    cfg = CONFIGS[case]
    torch.manual_seed(0)
    B, (H, W) = 2, cfg["res"]
    ctx = torch.randn(B, *cfg["text"], device=dev) if cfg["text"] else None
    model = SimpleUDiT(**cfg["kw"])
    fp = _live_params(model, 3, ctx)
    x = torch.randn(B, H, W, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    Fo, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(B, H, W, 3, device=dev)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    torch.cuda.synchronize()
    P = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fp.named.items()}
    p = model.patch_size
    Fr = udit_ref.simple_udit_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), patch_size=p,
                                      num_layers=model.num_layers, num_heads=model.num_heads,
                                      textcontext=None if ctx is None else ctx.cpu(),
                                      order=model._scan_indices(H // p, W // p))
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


def test_forward_is_deterministic_and_apply_matches():
    cfg = CONFIGS["text3d_sigma"]
    model = SimpleUDiT(**cfg["kw"])
    ctx = torch.randn(2, 7, 64, device=dev)
    fp = _live_params(model, 4, ctx)
    x = torch.randn(2, 16, 16, 3, device=dev)
    t = torch.rand(2, device=dev)
    a, _ = model.forward(fp, x, t, ctx, save=True)
    b = model.apply(fp, x, t, ctx)
    assert torch.equal(a, b)


def test_final_proj_is_float32():
    """The output projection carries the f32 kernel's bits below bf16: against the same program with the kernel
    rounded to bf16, the output moves by the rounding (with final_norm's output fixed, the rest of the model is
    unchanged)."""
    model = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2)
    fp = _live_params(model, 6)
    x = torch.randn(2, 16, 16, 3, device=dev)
    t = torch.rand(2, device=dev)
    a = model.apply(fp, x, t)
    k = fp.named["final_proj/kernel"]
    k.copy_(k.bfloat16().float())
    fp.touch()
    b = model.apply(fp, x, t)
    assert not torch.equal(a, b) and rel(a, b) < 1e-2


def _trainer(graph, model=None, res=16, encoder="random"):
    model = model or SimpleUDiT(patch_size=2, emb_features=128, num_layers=2, num_heads=2, use_hilbert=True)
    if encoder == "random":
        cond = ConditionalInputConfig(RandomEmbeddingEncoder(7, 64, device=dev))
    else:
        enc = CLIPTextEncoder(clip_model("tiny"), Tok(1000), modelname="tiny-random", backend="fdx")
        cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True,
                                      unconditional_input="")
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (res, res, 3), [cond]), rngs=4, unconditional_prob=0.25,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 use_cuda_graph=graph)
    return model, tr


def _batch(seed=0, B=4, res=16, tokens=False):
    rng = np.random.default_rng(seed)
    b = {"image": torch.from_numpy(rng.integers(0, 256, (B, res, res, 3), dtype=np.uint8))}
    if tokens:
        ids, mask = token_batch(1000, [3, 10, 0, 20][:B], seed=seed)
        b["text"] = {"input_ids": ids, "attention_mask": mask}
    else:
        b["text"] = [f"prompt {seed} {i}" for i in range(B)]
    return b


@pytest.mark.parametrize("encoder", ["random", "fdx_tower"])
def test_eager_and_graphed_trainer_steps_agree(encoder):
    _, eager = _trainer(False, encoder=encoder)
    _, graphed = _trainer(True, encoder=encoder)
    se, sg = eager._define_train_step(), graphed._define_train_step()
    stE, stG, rE, rG = eager.state, graphed.state, eager.rngstate, graphed.rngstate
    for i in range(3):
        b = _batch(i, tokens=encoder != "random")
        stE, lE, rE = se(stE, rE, b)
        stG, lG, rG = sg(stG, rG, b)
        assert abs(lE.item() - lG.item()) <= 1e-3 * abs(lE.item()), (i, lE.item(), lG.item())
    assert rel(stG.params.flat, stE.params.flat) < 1e-3


def test_loss_decreases_on_a_fixed_batch():
    _, tr = _trainer(True, model=SimpleUDiT(patch_size=2, emb_features=128, num_layers=4, num_heads=2))
    step = tr._define_train_step()
    st, r = tr.state, tr.rngstate
    b = _batch(7)
    losses = []
    for _ in range(30):
        st, loss, _ = step(st, r, b)            # same key every step: same noise, timesteps and null mask
        losses.append(loss.item())
    assert np.isfinite(losses).all() and np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses


@pytest.mark.parametrize("cls", [EulerSampler, EulerAncestralSampler])
@pytest.mark.parametrize("hilbert", [False, True])
def test_sampling_whole_step_graph_matches_eager(cls, hilbert):
    model = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, use_hilbert=hilbert)
    enc = RandomEmbeddingEncoder(7, 64, device=dev)
    ctx = enc(["a cat", "a dog"]).to(dev)
    fp = _live_params(model, 5, ctx)
    sched, tr = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev), KarrasPredictionTransform(0.5)
    cfg = DiffusionInputConfig("image", (16, 16, 3), [ConditionalInputConfig(enc)])
    key = utils.RandomMarkovState(utils.ThreefryKey(utils.PRNGKey(11)))
    outs = []
    for graph in (False, True):
        smp = cls(model, sched, tr, cfg, use_cuda_graph=graph)
        outs.append(smp.generate_samples(fp, 2, 16, diffusion_steps=6, start_step=1000, device=dev,
                                         rngstate=utils.RandomMarkovState(key.rng), model_conditioning_inputs=(ctx,)))
    assert outs[0].shape == (2, 16, 16, 3) and torch.isfinite(outs[1]).all()
    assert rel(outs[1], outs[0]) < 1e-2


def test_checkpoint_round_trip(tmp_path):
    model, tr = _trainer(True)
    step = tr._define_train_step()
    tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, _batch(1))
    tr.save(0, 1, path=str(tmp_path))
    _, tr2 = _trainer(False, SimpleUDiT(**model.config()))
    tr2.load(checkpoint_path=str(tmp_path))
    assert torch.equal(tr2.state.params.flat, tr.state.params.flat)
    assert torch.equal(tr2.state.opt_state["mu"], tr.state.opt_state["mu"])
    assert tr2.state.step == tr.state.step
