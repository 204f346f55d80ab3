"""use_remat on the GPU: the training forward keeps only each trunk block's input, and the backward re-runs the block's
forward from it right before the block's backward.  The models and inputs are test_inference_forward_gpu.py's, every
parameter random.

  * With and without the flag: the forward output, every block record the backward reads (the recomputed one against
    the taped one, tensor by tensor), every block's input gradient and the sequence of on_ready offsets are equal bit
    for bit.  The use_remat=False run is first repeated and reproduces all of these bit for bit itself.
  * Parameter gradients are not bit-reproducible even without the flag: the weight gradients of fdx_gemm's split-K
    launches (red.global.add of f32 partials), the bias gradients of fdx_colsum (f32 atomics across blocks) and UViT's
    RMSNorm scale gradients (shared- and global-memory atomics) add their partial sums in arrival order, so two
    use_remat=False backwards differ in the last bits of those leaves.  The inputs of every one of those launches are
    the records and block input gradients checked above, so each gradient is held to the rounding bound that two
    use_remat=False runs meet (relative L2 <= 1e-5), the bound test_ssm_dit_gpu.py holds them to.
  * One eager and one CUDA-graphed GeneralDiffusionTrainer step (adamw, EMA): the same loss, parameters, Adam moments
    and EMA within that rounding bound (the loss, too, is a sum of f32 atomics: fdx_loss_fwd_bwd).
  * Peak memory of forward + backward at num_layers 2 and 8: with the flag it grows by at most one bf16 row of the
    block's own token rows and width per extra block (U models: plus, per extra up layer, the up_dense input the tape
    holds either way and the gradient row that waits for its skip's down block), plus one row of allocator slack;
    without it, by at least six block records.
"""
import numpy as np
import pytest
import torch

from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.simple_dit import SimpleDiT
from flaxdiff_b200.models.simple_unet import Node
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT
from flaxdiff_b200.models.udit import SimpleUDiT
from flaxdiff_b200.models.uvit import UViT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.schedulers import EDMNoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from test_inference_forward_gpu import DEPTH, DEPTH_B, DEPTH_F, DEPTH_RES, MODELS, _inputs, _random_params

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
BLOCK_FWD = ("_block_fwd", "_ssm_block_fwd", "_mm_block_fwd")
BLOCK_BWD = ("_block_bwd", "_ssm_block_bwd", "_mm_block_bwd")


def _tensors(obj, out):
    """Every tensor a block record holds, in a fixed order (copies: the backward may overwrite buffers in place)."""
    if isinstance(obj, torch.Tensor):
        out.append(obj.clone())
    elif isinstance(obj, Node):
        out.append(obj.t.clone())
    elif isinstance(obj, (tuple, list)):
        for o in obj:
            _tensors(o, out)
    elif isinstance(obj, dict):
        for k in sorted(obj):
            _tensors(obj[k], out)
    return out


def _spy(model, records, dxs):
    """Wraps the instance's block programs: records[name] gets each record a forward with save=True returns, dxs[name]
    each block backward's input gradient."""
    for attr in BLOCK_FWD:
        f = getattr(model, attr, None)
        if f is not None:
            def fwd(n, *a, _f=f, **k):
                out, rec = _f(n, *a, **k)
                if rec is not None:
                    records[n] = _tensors(rec, [])
                return out, rec
            setattr(model, attr, fwd)
    for attr in BLOCK_BWD:
        f = getattr(model, attr, None)
        if f is not None:
            def bwd(rec, *a, _f=f, **k):
                dx = _f(rec, *a, **k)
                dxs[len(dxs)] = dx.clone()
                return dx
            setattr(model, attr, bwd)


def _run(cls, kw, remat, x, t, ctx, seed):
    """forward(save=True) + backward of a random output gradient -> (output, gradients, records, block input
    gradients, on_ready offsets)."""
    model = cls(**kw, use_remat=remat)
    fp = _random_params(model, seed, ctx)
    records, dxs, offsets = {}, {}, []
    _spy(model, records, dxs)
    out, saved = model.forward(fp, x, t, ctx, save=True)
    dF = torch.randn(out.shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
    g = fp.zeros_like()
    model.backward(fp, saved, dF, g, on_ready=lambda lo, streams: offsets.append(lo))
    torch.cuda.synchronize()
    return out, g.named, records, dxs, offsets


def _equal(a, b):
    return a.shape == b.shape and torch.equal(a, b)


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


GRAD_REL = 1e-5             # two use_remat=False backwards agree to this (the split-K / column-sum atomics' order)


@pytest.mark.parametrize("case", sorted(MODELS))
def test_remat_backward_equals_taped_backward_bitwise(case):
    cls, kw, res, text = MODELS[case]
    x, t, ctx = _inputs(3, res, text, 1)
    base = _run(cls, kw, False, x, t, ctx, 2)
    again = _run(cls, kw, False, x, t, ctx, 2)
    remat = _run(cls, kw, True, x, t, ctx, 2)
    assert torch.isfinite(base[0]).all() and base[0].abs().max() > 0
    for run, what in ((again, "use_remat=False again"), (remat, "use_remat=True")):
        assert torch.equal(run[0], base[0]), what
        # the records the backward reads (under use_remat recomputed, in reverse block order), tensor by tensor
        assert sorted(run[2]) == sorted(base[2]) and len(base[2]) > 0, what
        for n in base[2]:
            assert len(run[2][n]) == len(base[2][n]), (what, n)
            for i, (a, b) in enumerate(zip(run[2][n], base[2][n])):
                assert _equal(a, b), (what, n, i)
        assert len(run[3]) == len(base[3]) and all(torch.equal(run[3][i], base[3][i]) for i in base[3]), what
        assert run[4] == base[4] and base[4][-1] == 0, what
        bad = {k: rel(run[1][k], base[1][k]) for k in base[1] if rel(run[1][k], base[1][k]) > GRAD_REL}
        assert not bad, (what, bad)
    exact = sum(torch.equal(remat[1][k], base[1][k]) for k in base[1])
    print(f"{case}: {exact} of {len(base[1])} gradient leaves bit for bit")


# ---------------------------------------------------------------------------------------------- the trainer
TRAINER = {
    "dit": (SimpleDiT, dict(patch_size=2, emb_features=128, num_layers=3, num_heads=2, learn_sigma=True)),
    "hybrid": (HybridSSMAttentionDiT, dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2,
                                           ssm_state_dim=16, ssm_attention_ratio="1:1")),
    "udit": (SimpleUDiT, dict(patch_size=2, emb_features=128, num_layers=4, num_heads=2)),
    "uvit_head": (UViT, dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2,
                             add_residualblock_output=True)),
}


def _step(cls, kw, remat, graph):
    model = cls(**kw, use_remat=remat)
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (16, 16, 3), []), rngs=4,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 use_cuda_graph=graph)
    step = tr._define_train_step()
    rng = np.random.default_rng(3)
    batch = {"image": torch.from_numpy(rng.integers(0, 256, (3, 16, 16, 3), dtype=np.uint8))}
    st, loss, _ = step(tr.state, tr.rngstate, batch)
    torch.cuda.synchronize()
    return loss.clone(), st.params.flat.clone(), st.ema_params.flat.clone(), st.opt_state["mu"].clone()


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("case", sorted(TRAINER))
def test_trainer_step_is_unchanged(case, graph):
    cls, kw = TRAINER[case]
    base = _step(cls, kw, False, graph)
    assert torch.isfinite(base[0]).all()
    for run, what in ((_step(cls, kw, False, graph), "use_remat=False again"), (_step(cls, kw, True, graph), "remat")):
        for name, a, b in zip(("loss", "params", "ema", "mu"), run, base):
            assert rel(a, b) <= GRAD_REL, (what, name, rel(a, b))


# ---------------------------------------------------------------------------------------------- memory vs depth
def _train_peak(model, fp, x, t, ctx):
    """Bytes allocated above the resident set (parameters, their bf16 shadow, the gradient buffer, cached tables) at
    the peak of forward(save=True) + backward."""
    g = fp.zeros_like()

    def once():
        out, saved = model.forward(fp, x, t, ctx, save=True)
        model.backward(fp, saved, torch.ones_like(out), g)
    once()                                                      # the shadow and the constant tables are made here
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    once()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("case", sorted(DEPTH))
def test_remat_peak_grows_by_one_row_per_block(case):
    cls, kw, text, u_shaped = DEPTH[case]
    x, t, ctx = _inputs(DEPTH_B, DEPTH_RES, text, 6)
    common = {} if cls.__name__ == "HierarchicalMMDiT" else dict(patch_size=2, emb_features=DEPTH_F, num_heads=4)
    M = DEPTH_B * (DEPTH_RES[0] // 2) * (DEPTH_RES[1] // 2)     # token rows at the finest level
    if cls is UViT:
        M += DEPTH_B                                            # the time token
    row = M * DEPTH_F * 2                                       # one bf16 [M, F] row matrix
    peaks = {}
    for n in (2, 8):
        for remat in (False, True):
            model = cls(**common, **kw(n), use_remat=remat)
            fp = _random_params(model, 7, ctx)
            peaks[n, remat] = _train_peak(model, fp, x, t, ctx)
            del model, fp
            torch.cuda.empty_cache()
    grow_remat = peaks[8, True] - peaks[2, True]
    grow_tape = peaks[8, False] - peaks[2, False]
    detail = f"{case}: use_remat {peaks[2, True]} -> {peaks[8, True]}, taped {peaks[2, False]} -> {peaks[8, False]} " \
             f"bytes, row {row}"
    print(detail)
    # six more blocks (U models: three more up layers, each adding its up_dense input and its skip's waiting gradient;
    # HierarchicalMMDiT: six more per stage loop, the second stage's rows a quarter of the finest level's)
    rows = 6 * 2 + 6 / 4 if cls.__name__ == "HierarchicalMMDiT" else 6 + (2 * 3 if u_shaped else 0)
    assert grow_remat <= rows * row + row, detail
    # every record keeps at least the block's input and its [M, 4F] MLP hidden rows
    assert grow_tape >= 6 * 5 * row, detail
    assert peaks[8, True] < peaks[8, False], detail
