"""SimpleMMDiT on the GPU: forward and every parameter gradient against the CPU oracle (oracle/mmdit_ref.py) - 3-D text
with learn_sigma, 2-D text, the Hilbert order on a 6 x 4 grid - then the trainer's eager and graphed steps (with random
text embeddings and with the in-graph fdx CLIP text tower), a short fit on a fixed batch, Euler / Euler-ancestral
sampling and a checkpoint round trip.  Tolerances are SimpleDiT's: forward <= 3e-2 relative L2, each gradient <= 6e-2.

The ada, final_proj and bias values are random so every gate and modulation is live, and a few MLP scale / shift
biases sit at +-40, far past the clip, so that the clip's forward and its zero gradient are on the path."""
import numpy as np
import pytest
import torch

from clip_text_ref import Tok, clip_model, token_batch
from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.mmdit import HierarchicalMMDiT, SimpleMMDiT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import mmdit_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _live_params(model, seed, ctx):
    """init, then random ada / final_proj kernels and biases; a few scale_mlp / shift_mlp biases past the clip.  The
    ada kernels are scaled by 0.5 / sqrt(2F), so that the modulations stay O(1) at every width: larger ones make the
    attention so peaked that the bf16 rounding of its inputs, not the program, dominates the q / k gradients."""
    fp = model.init(seed, textcontext=ctx, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    F = model.emb_features
    for name, t in fp.named.items():
        if "/ada_ln_zero/" in name or name.startswith("final_proj") or name.endswith("bias"):
            std = 0.5 / (2 * F) ** 0.5 if name.endswith("ada_ln_zero/ada_t_proj/kernel") or \
                name.endswith("ada_ln_zero/ada_text_proj/kernel") else 0.2
            t.copy_(std * torch.randn(t.shape, generator=g, device=dev))
        if name.endswith("ada_ln_zero/ada_t_proj/bias"):
            t[0:F:7] = 40.0          # scale_mlp columns clipped to +10
            t[F + 3:2 * F:9] = -40.0  # shift_mlp columns clipped to -10
    return fp


CONFIGS = {
    "text3d_sigma": dict(kw=dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2, learn_sigma=True),
                         res=(16, 16), text=(7, 64)),
    "text2d_d48": dict(kw=dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4), res=(32, 16),
                       text=(96,)),
    "hilbert_6x4": dict(kw=dict(patch_size=4, emb_features=64, num_layers=2, num_heads=2, use_hilbert=True),
                        res=(24, 16), text=(5, 64)),
}


def _oracle_case(model, fp, x, t, ctx, H, W):
    P = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fp.named.items()}
    p = model.patch_size
    Fr = mmdit_ref.simple_mmdit_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), ctx.cpu(),
                                        patch_size=p, num_layers=model.num_layers, num_heads=model.num_heads,
                                        order=model._scan_indices(H // p, W // p))
    return P, Fr


@pytest.mark.parametrize("case", sorted(CONFIGS))
def test_forward_and_gradients_match_oracle(case):
    cfg = CONFIGS[case]
    torch.manual_seed(0)
    B, (H, W) = 2, cfg["res"]
    ctx = torch.randn(B, *cfg["text"], device=dev)
    model = SimpleMMDiT(**cfg["kw"])
    fp = _live_params(model, 3, ctx)
    x = torch.randn(B, H, W, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    Fo, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(B, H, W, 3, device=dev)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    torch.cuda.synchronize()
    P, Fr = _oracle_case(model, fp, x, t, ctx, H, W)
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
    # the clipped columns pass no gradient to their ada parameters
    F = model.emb_features
    for i in range(model.num_layers):
        gb = grads.named[f"mmdit_block_{i}/ada_ln_zero/ada_t_proj/bias"]
        assert gb[0:F:7].abs().max().item() == 0 and gb[F + 3:2 * F:9].abs().max().item() == 0


def test_forward_is_deterministic_and_apply_matches():
    cfg = CONFIGS["text3d_sigma"]
    model = SimpleMMDiT(**cfg["kw"])
    ctx = torch.randn(2, 7, 64, device=dev)
    fp = _live_params(model, 4, ctx)
    x = torch.randn(2, 16, 16, 3, device=dev)
    t = torch.rand(2, device=dev)
    a, _ = model.forward(fp, x, t, ctx, save=True)
    b = model.apply(fp, x, t, ctx)
    assert torch.equal(a, b)


def _trainer(graph, model=None, res=16, encoder="random"):
    model = model or SimpleMMDiT(patch_size=2, emb_features=128, num_layers=2, num_heads=2, use_hilbert=True)
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
    _, tr = _trainer(True, model=SimpleMMDiT(patch_size=2, emb_features=128, num_layers=2, num_heads=2))
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
    model = SimpleMMDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, use_hilbert=hilbert)
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
    _, tr2 = _trainer(False, SimpleMMDiT(**model.config()))
    tr2.load(checkpoint_path=str(tmp_path))
    assert torch.equal(tr2.state.params.flat, tr.state.params.flat)
    assert torch.equal(tr2.state.opt_state["mu"], tr.state.opt_state["mu"])
    assert tr2.state.step == tr.state.step


# ------------------------------------------------------------------------------------------ HierarchicalMMDiT
HCONFIGS = {
    "two_stages_text3d_sigma": dict(kw=dict(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 2),
                                            num_heads=(2, 2), learn_sigma=True), res=(16, 24), text=(7, 64)),
    "three_stages_text2d": dict(kw=dict(base_patch_size=2, emb_features=(64, 128, 192), num_layers=(1, 1, 2),
                                        num_heads=(2, 2, 3)), res=(16, 16), text=(96,)),
    "three_stages_hilbert_6x4": dict(kw=dict(base_patch_size=2, emb_features=(64, 128, 192), num_layers=(1, 1, 1),
                                             num_heads=(2, 2, 3), use_hilbert=True), res=(24, 16), text=(5, 64)),
}


def _hier_live_params(model, seed, ctx):
    """As _live_params at every stage; LayerNorm scales around one so the merge / expand / fusion norms are live."""
    fp = model.init(seed, textcontext=ctx, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, t in fp.named.items():
        if "/ada_ln_zero/" in name:
            F = model._widths(name.split("/")[0])[0]
            std = 0.2 if name.endswith("bias") else 0.5 / (2 * F) ** 0.5
            t.copy_(std * torch.randn(t.shape, generator=g, device=dev))
            if name.endswith("ada_t_proj/bias"):
                t[0:F:7] = 40.0
                t[F + 3:2 * F:9] = -40.0
        elif name.startswith("final_proj") or name.endswith("bias"):
            t.copy_(0.2 * torch.randn(t.shape, generator=g, device=dev))
        elif name.endswith("/scale"):
            t.copy_(1 + 0.2 * torch.randn(t.shape, generator=g, device=dev))
    return fp


@pytest.mark.parametrize("case", sorted(HCONFIGS))
def test_hierarchical_forward_and_gradients_match_oracle(case):
    cfg = HCONFIGS[case]
    torch.manual_seed(0)
    B, (H, W) = 2, cfg["res"]
    ctx = torch.randn(B, *cfg["text"], device=dev)
    model = HierarchicalMMDiT(**cfg["kw"])
    fp = _hier_live_params(model, 3, ctx)
    x = torch.randn(B, H, W, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    Fo, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(B, H, W, 3, device=dev)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    torch.cuda.synchronize()
    P = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fp.named.items()}
    p = model.base_patch_size
    Fr = mmdit_ref.hierarchical_mmdit_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), ctx.cpu(),
                                              base_patch_size=p, num_layers=model.num_layers,
                                              num_heads=model.num_heads, order=model._scan_indices(H // p, W // p))
    (Fr * dF.cpu()).sum().backward()
    assert rel(Fo, Fr) < 3e-2, rel(Fo, Fr)
    bad = {}
    for k in P:
        ref = P[k].grad
        if ref.norm() == 0:
            assert grads.named[k].abs().max().item() == 0, k
            continue
        e = rel(grads.named[k], ref)
        if e >= 6e-2:
            bad[k] = e
    assert not bad, bad


def _hier_trainer(graph, model=None):
    model = model or HierarchicalMMDiT(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 1), num_heads=(2, 2),
                                       use_hilbert=True)
    return _trainer(graph, model=model)


def test_hierarchical_eager_and_graphed_trainer_steps_agree():
    _, eager = _hier_trainer(False)
    _, graphed = _hier_trainer(True)
    se, sg = eager._define_train_step(), graphed._define_train_step()
    stE, stG, rE, rG = eager.state, graphed.state, eager.rngstate, graphed.rngstate
    for i in range(3):
        b = _batch(i)
        stE, lE, rE = se(stE, rE, b)
        stG, lG, rG = sg(stG, rG, b)
        assert abs(lE.item() - lG.item()) <= 1e-3 * abs(lE.item()), (i, lE.item(), lG.item())
    assert rel(stG.params.flat, stE.params.flat) < 1e-3


def test_hierarchical_loss_decreases_on_a_fixed_batch():
    _, tr = _hier_trainer(True, HierarchicalMMDiT(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 1),
                                                  num_heads=(2, 2)))
    step = tr._define_train_step()
    st, r = tr.state, tr.rngstate
    b = _batch(7)
    losses = []
    for _ in range(30):
        st, loss, _ = step(st, r, b)
        losses.append(loss.item())
    assert np.isfinite(losses).all() and np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses


@pytest.mark.parametrize("cls", [EulerSampler, EulerAncestralSampler])
@pytest.mark.parametrize("hilbert", [False, True])
def test_hierarchical_sampling_whole_step_graph_matches_eager(cls, hilbert):
    model = HierarchicalMMDiT(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 1), num_heads=(2, 2),
                              use_hilbert=hilbert)
    enc = RandomEmbeddingEncoder(7, 64, device=dev)
    ctx = enc(["a cat", "a dog"]).to(dev)
    fp = _hier_live_params(model, 5, ctx)
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


def test_hierarchical_checkpoint_round_trip(tmp_path):
    model, tr = _hier_trainer(True)
    step = tr._define_train_step()
    tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, _batch(1))
    tr.save(0, 1, path=str(tmp_path))
    _, tr2 = _hier_trainer(False, HierarchicalMMDiT(**model.config()))
    tr2.load(checkpoint_path=str(tmp_path))
    assert torch.equal(tr2.state.params.flat, tr.state.params.flat)
    assert torch.equal(tr2.state.opt_state["mu"], tr.state.opt_state["mu"])
