"""UViT on the GPU: forward and every parameter gradient against the CPU oracle (oracle/uvit_ref.py) - the default
block with and without 77 x 768 text, use_projection, use_self_and_cross, norm_inputs, Hilbert on 8 x 8 and 6 x 4, the
convolutional output head with swish and with mish, num_layers 2 and 12 at F = 64 (the bf16 stream at full depth) -
then the trainer's eager and graphed steps (random text embeddings and the in-graph fdx CLIP text tower), a short fit
on a fixed batch, Euler / Euler-ancestral sampling with CFG and a checkpoint round trip.  Tolerances are SimpleDiT's:
forward <= 3e-2 relative L2, each gradient <= 6e-2.

final_proj's kernel and every bias are random, so the output does not start at zero and no bias sits at its init."""
import numpy as np
import pytest
import torch

from clip_text_ref import Tok, clip_model, token_batch
from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.uvit import UViT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler, EulerSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from oracle import uvit_ref

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _live_params(model, seed, ctx=None, key_scale=1.0):
    """init, then a random final_proj kernel and random biases (0.2), so that no output or bias sits at its init.
    key_scale multiplies every to_k kernel (see CONFIGS["layers12_f64"])."""
    fp = model.init(seed, textcontext=ctx, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, t in fp.named.items():
        if name.startswith("final_proj") or name.endswith("bias"):
            t.copy_(0.2 * torch.randn(t.shape, generator=g, device=dev))
        elif name.endswith("to_k/kernel"):
            t.mul_(key_scale)
    fp.touch()
    return fp


def _small(**kw):
    base = dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2)
    base.update(kw)
    return base


CONFIGS = {
    "default": dict(kw=_small(), res=(16, 16), text=None),
    "default_text77": dict(kw=_small(), res=(16, 16), text=(77, 768)),
    "projection": dict(kw=_small(use_projection=True), res=(16, 16), text=(5, 64)),
    "self_and_cross": dict(kw=_small(use_self_and_cross=True), res=(16, 16), text=None),
    "norm_inputs": dict(kw=_small(norm_inputs=True), res=(16, 16), text=(5, 64)),
    "no_residual": dict(kw=_small(explicitly_add_residual=False, norm_inputs=True), res=(16, 16), text=None),
    "hilbert_8x8": dict(kw=_small(use_hilbert=True), res=(16, 16), text=(5, 64)),
    "hilbert_6x4": dict(kw=_small(patch_size=4, emb_features=64, use_hilbert=True), res=(24, 16), text=None),
    "head_swish": dict(kw=_small(add_residualblock_output=True), res=(16, 16), text=(5, 64)),
    "head_mish": dict(kw=_small(add_residualblock_output=True, activation="mish"), res=(16, 16), text=None),
    # Full depth.  The default block's output is x + (x + attention + feed-forward), so the stream doubles per block,
    # and its keys read that un-normed stream: at flax's init the logits saturate by mid-depth and the reference
    # itself maps a 1e-6 relative perturbation of each block's output to an O(1) change of the output, so no two
    # implementations can agree there.  With the key kernels scaled by 1e-3 the attention stays soft; the reference
    # then moves by about 1 % under that perturbation, and rounding the stream to bf16 moves it by as much.
    "layers12_f64": dict(kw=_small(emb_features=64, num_layers=12, num_heads=2), res=(16, 16), text=(5, 64),
                         key_scale=1e-3),
}


@pytest.mark.parametrize("case", sorted(CONFIGS))
def test_forward_and_gradients_match_oracle(case):
    cfg = CONFIGS[case]
    torch.manual_seed(0)
    B, (H, W) = 2, cfg["res"]
    ctx = torch.randn(B, *cfg["text"], device=dev) if cfg["text"] else None
    model = UViT(**cfg["kw"])
    fp = _live_params(model, 3, ctx, cfg.get("key_scale", 1.0))
    x = torch.randn(B, H, W, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    Fo, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(B, H, W, 3, device=dev)
    grads = fp.zeros_like()
    model.backward(fp, saved, dF, grads)
    torch.cuda.synchronize()
    P = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in fp.named.items()}
    p = model.patch_size
    kw = {k: getattr(model, k) for k in ("use_projection", "use_self_and_cross", "norm_inputs",
                                          "explicitly_add_residual", "add_residualblock_output", "activation")}
    Fr = uvit_ref.uvit_forward(P, x.float().cpu(), t.cpu(), model._fourier_freqs(dev).cpu(), patch_size=p,
                               num_layers=model.num_layers, num_heads=model.num_heads,
                               textcontext=None if ctx is None else ctx.cpu(),
                               order=model._scan_indices(H // p, W // p), **kw)
    (Fr * dF.cpu()).sum().backward()
    assert rel(Fo, Fr) < 3e-2, rel(Fo, Fr)
    bad = {}
    for k in P:
        ref = P[k].grad
        if k == "pos_encoding":                  # only the first N rows are read
            N = (H // p) * (W // p)
            assert grads.named[k][:, N:].abs().max().item() == 0
        e = rel(grads.named[k], ref)
        if e >= 6e-2:
            bad[k] = e
    assert not bad, bad


def test_forward_is_deterministic_and_apply_matches():
    model = UViT(**_small(add_residualblock_output=True))
    ctx = torch.randn(2, 7, 64, device=dev)
    fp = _live_params(model, 4, ctx)
    x = torch.randn(2, 16, 16, 3, device=dev)
    t = torch.rand(2, device=dev)
    a, _ = model.forward(fp, x, t, ctx, save=True)
    b = model.apply(fp, x, t, ctx)
    assert torch.equal(a, b)


def test_backward_is_bitwise_reproducible_for_the_position_table():
    model = UViT(**_small())
    fp = _live_params(model, 5)
    x = torch.randn(4, 16, 16, 3, device=dev)
    t = torch.rand(4, device=dev)
    dF = torch.randn(4, 16, 16, 3, device=dev)
    outs = []
    for _ in range(2):
        _, saved = model.forward(fp, x, t, None, save=True)
        g = fp.zeros_like()
        model.backward(fp, saved, dF, g)
        outs.append(g.named["pos_encoding"].clone())
    assert torch.equal(outs[0], outs[1])

def _trainer(graph, model=None, res=16, encoder="random"):
    model = model or UViT(patch_size=2, emb_features=128, num_layers=2, num_heads=2, use_hilbert=True,
                          add_residualblock_output=True)
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
    _, tr = _trainer(True, model=UViT(patch_size=2, emb_features=128, num_layers=4, num_heads=2))
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
    model = UViT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, use_hilbert=hilbert)
    enc = RandomEmbeddingEncoder(7, 64, device=dev)
    ctx = enc(["a cat", "a dog"]).to(dev)
    fp = _live_params(model, 5, ctx)
    sched, tr = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev), KarrasPredictionTransform(0.5)
    cfg = DiffusionInputConfig("image", (16, 16, 3), [ConditionalInputConfig(enc)])
    key = utils.RandomMarkovState(utils.ThreefryKey(utils.PRNGKey(11)))
    outs = []
    for graph in (False, True):
        smp = cls(model, sched, tr, cfg, use_cuda_graph=graph,
                  guidance_scale=2.0 if cls is EulerAncestralSampler else 0.0)     # CFG on the ancestral leg
        outs.append(smp.generate_samples(fp, 2, 16, diffusion_steps=6, start_step=1000, device=dev,
                                         rngstate=utils.RandomMarkovState(key.rng), model_conditioning_inputs=(ctx,)))
    assert outs[0].shape == (2, 16, 16, 3) and torch.isfinite(outs[1]).all()
    assert rel(outs[1], outs[0]) < 1e-2


def test_checkpoint_round_trip(tmp_path):
    model, tr = _trainer(True)
    step = tr._define_train_step()
    tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, _batch(1))
    tr.save(0, 1, path=str(tmp_path))
    _, tr2 = _trainer(False, UViT(**model.config()))
    tr2.load(checkpoint_path=str(tmp_path))
    assert torch.equal(tr2.state.params.flat, tr.state.params.flat)
    assert torch.equal(tr2.state.opt_state["mu"], tr.state.opt_state["mu"])
    assert tr2.state.step == tr.state.step
