"""The UNet's inference forward (Unet.forward(save=False), which apply() and the samplers run) on the GPU.

  * apply() equals forward(save=True)'s output bit for bit: the launches are the same, only the lifetimes differ.
    Every parameter is random first (biases start at zero, which would hide a wrong bias read).  The comparison runs
    at 8 x 8 images, where every level is below ops.COLSTATS_MIN_PIXELS: there the convolutions leave no fused column
    sums, whose f32 atomics make two runs of the same forward differ in the last bits, and the training forward is
    shown to reproduce itself bit for bit first.  At 32 x 32, where the fused sums run, apply() is compared to a
    relative L2 of 5e-3, a bound on that run-to-run noise.
  * The inference peak (max_memory_allocated above the resident parameters) stays within the concat buffers and
    the output plus the largest single block's working set, both computed from _plan() by _budget below; the
    training forward's peak is above 1.2 times that bound.  At num_res_blocks 1 and 3 the inference peak grows by no more
    than the extra concat buffers (and their timestep rows).
  * A classifier-free-guided Euler-ancestral whole-step graph with a threefry key gives its eager loop's samples
    bit for bit, with the timestep projections on the side stream (the default).
"""
import pytest
import torch

from flaxdiff_b200 import utils
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder
from flaxdiff_b200.models.simple_unet import Unet, _attn_width
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import EulerAncestralSampler
from flaxdiff_b200.schedulers import KarrasVENoiseScheduler

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

FULL = {"heads": 8, "only_pure_attention": False, "use_projection": True}
CROSS_ONLY = {"heads": 4, "only_pure_attention": False, "use_self_and_cross": False}
GALLERY = (None, {"heads": 8}, {"heads": 8}, {"heads": 8})          # 1024-channel levels: 128-wide heads
TWO = (None, {"heads": 2}, {"heads": 2}, {"heads": 2})              # 512-channel levels: 256-wide heads

# case -> (Unet keyword arguments, text context [77, 768]?)
CASES = {
    "no_attention": (dict(feature_depths=(64, 128, 256), attention_configs=(None, None, None)), False),
    "self_attention_two_levels": (dict(feature_depths=(64, 128, 256),
                                       attention_configs=(None, {"heads": 8}, {"heads": 8})), False),
    "full_block_projections_text": (dict(feature_depths=(64, 128, 256), attention_configs=(None, FULL, FULL)), True),
    "full_block_self": (dict(feature_depths=(64, 128, 256), attention_configs=(None, None, FULL)), False),
    "cross_only_text": (dict(feature_depths=(64, 128, 256), attention_configs=(None, CROSS_ONLY, CROSS_ONLY)), True),
    "mish": (dict(feature_depths=(64, 128, 256), attention_configs=(None, None, {"heads": 4}), activation="mish"),
             False),
    "gallery_heads128_text": (dict(feature_depths=(128, 256, 512, 1024), attention_configs=GALLERY), True),
    "heads256": (dict(attention_configs=TWO), False),
    "res_blocks_1": (dict(feature_depths=(64, 128, 256), attention_configs=(None, None, {"heads": 4}),
                          num_res_blocks=1), False),
    "res_blocks_3_middle_2": (dict(feature_depths=(64, 128, 256), attention_configs=(None, {"heads": 4}, None),
                                   num_res_blocks=3, num_middle_res_blocks=2), False),
}


def _model(kw, text):
    return Unet(dtype=torch.bfloat16, context_dim=768 if text else None, **kw)


def _random_params(model, seed):
    """init, then every kernel, bias and scale random, at magnitudes that keep the activations O(1)."""
    fp = model.init(seed, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, t in fp.named.items():
        leaf = name.rsplit("/", 1)[-1]
        r = torch.randn(t.shape, generator=g, device=dev)
        if leaf == "scale":
            t.copy_(1.0 + 0.1 * r)
        elif leaf == "kernel":
            t.copy_(r * 0.5 / (t.numel() // t.shape[-1]) ** 0.5)
        else:
            t.copy_(0.1 * r)
    fp.touch()
    return fp


def _inputs(B, res, text, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((B, res, res, 3), generator=g, device=dev)
    t = torch.rand(B, generator=g, device=dev)
    ctx = torch.randn((B, 77, 768), generator=g, device=dev) if text else None
    return x, t, ctx


@pytest.mark.parametrize("case", list(CASES))
def test_apply_equals_training_forward_bitwise(case):
    kw, text = CASES[case]
    model = _model(kw, text)
    fp = _random_params(model, 2)
    x, t, ctx = _inputs(3, 8, text, 1)
    xb = x.bfloat16()
    ref, tape = model.forward(fp, xb, t, ctx, save=True)
    again, _ = model.forward(fp, xb, t, ctx, save=True)
    assert tape is not None and torch.isfinite(ref).all() and ref.abs().max() > 0
    assert torch.equal(again, ref)                      # no f32 atomics in the forward at this size
    assert torch.equal(model.apply(fp, xb, t, ctx), ref)
    out, none = model.forward(fp, xb, t, ctx, save=False)
    assert none is None and torch.equal(out, ref)


@pytest.mark.parametrize("case", ["self_attention_two_levels", "full_block_projections_text"])
def test_apply_matches_training_forward_with_fused_column_sums(case):
    kw, text = CASES[case]
    model = _model(kw, text)
    fp = _random_params(model, 3)
    x, t, ctx = _inputs(2, 32, text, 4)
    ref, _ = model.forward(fp, x.bfloat16(), t, ctx, save=True)
    y = model.apply(fp, x.bfloat16(), t, ctx)
    err = ((y - ref).double().norm() / ref.double().norm()).item()
    assert torch.isfinite(y).all() and err < 5e-3, err


# ---------------------------------------------------------------------------------------------- peak memory
# a cached block handed to a smaller request is split only when more than 1 MiB would remain, so a live tensor may
# hold up to 1 MiB more than it asked for: room for eight such tensors
SLACK = 8 << 20


def _budget(model, B, H, W, ctx_len=77):
    """(concat buffers + output + resident-for-the-forward bytes, {block: working-set bytes}) of one inference
    forward, from _plan().  Per block, u = 2 B h w is the bytes of one bf16 channel at the block's level and
    cs = 32 B the bytes per channel of a buffer's column-sum workspace (4 slots x (sum, sum of squares) f32).
    Inputs and outputs are counted in every working set even when they are concat slots (an upper bound).
      res  cin -> cout : input + output, then the larger of a1 + h (conv1), h + a2 (norm2), a2 + the 1x1
                         residual (conv2), and the column sums of h and the output
      attn C           : input, output, RMSNorm_0 and project_in rows (4 C), then the larger of one attention
                         (normed input, residual in, output: 3 C; q and o over L tokens, k and v over the context;
                         the log-sum-exp; the head-padded weights) and the feed-forward (h2, the 8 C GEGLU input and
                         its 4 C output: 13 C)
      down / conv / up : input + output (+ the packed 16 cin cout upsample weights)
      out              : input, the normalised input, the f32 32-column im2col product, the f32 output
    The rest of the forward's memory: the output, the text context in bf16, every res block's f32 timestep row
    (all issued up front on the side stream) and the timestep embedding, plus SLACK for the caching allocator's
    rounding."""
    plan = model._plan()
    E = model.emb_features
    h, w = H, W
    cat, ws = 0, {}
    rest = B * H * W * 3 * 4 + 3 * B * E * 4 + SLACK
    if model.context_dim:
        rest += 2 * B * ctx_len * model.context_dim
    for kind, name, cin, cout in plan:
        u, cs = 2 * B * h * w, 32 * B
        if kind == "cat":
            cat += (u + cs) * (cin + cout)
        elif kind == "res":
            rest += 4 * B * cout
            ws[name] = (u + cs) * (cin + cout) + u * max(cin + cout, 2 * cout) + cs * cout
        elif kind == "attn":
            acfg, C = cout, cin
            heads = acfg["heads"]
            HD = heads * _attn_width(C // heads)
            Lk, Cc = (ctx_len, model.context_dim) if model.context_dim else (h * w, C)
            proj = acfg.get("use_projection", False)
            attn = 3 * u * C + 2 * B * (2 * h * w + 2 * Lk) * HD + 4 * B * heads * h * w + 2 * HD * (2 * C + 2 * Cc)
            ff = 0 if acfg.get("only_pure_attention", True) else 13 * u * C
            ws[name] = (u + cs) * 2 * C + u * C * (1 + proj) + max(attn, ff)
        elif kind == "down":
            h, w = h // 2, w // 2
            ws[name] = u * cin + (2 * B * h * w + cs) * cout
        elif kind == "up":
            h, w = h * 2, w * 2
            ws[name] = u * cin + (2 * B * h * w + cs) * cout + 32 * cin * cout
        elif kind == "conv":
            ws[name] = (u + cs) * (cin + cout)
        elif kind == "out":
            ws[name] = 2 * u * cin + cs * cin + B * h * w * 32 * 4 + cin * 32 * 4
    return cat + rest, ws


def _peak(model, fp, x, t, ctx, save):
    """Bytes allocated above the resident set (parameters, their bf16 shadow, cached tables) at the forward's peak."""
    model.forward(fp, x, t, ctx, save=save)                     # the shadow and the constant tables are made here
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out, tape = model.forward(fp, x, t, ctx, save=save)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out, tape
    torch.cuda.empty_cache()
    return peak


PEAK_B, PEAK_RES = 8, 64
PEAK_CASES = {
    "self_attention": (dict(attention_configs=(None, None, {"heads": 8}, {"heads": 8})), False),
    "full_block_text": (dict(attention_configs=(None, FULL, FULL, FULL)), True),
}


@pytest.mark.parametrize("case", list(PEAK_CASES))
def test_inference_peak_is_concat_buffers_plus_one_block(case):
    kw, text = PEAK_CASES[case]
    model = _model(kw, text)
    fp = _random_params(model, 5)
    x, t, ctx = _inputs(PEAK_B, PEAK_RES, text, 6)
    xb = x.bfloat16()
    floor, ws = _budget(model, PEAK_B, PEAK_RES, PEAK_RES)
    block = max(ws, key=ws.get)
    bound = floor + ws[block]
    inf, train = _peak(model, fp, xb, t, ctx, False), _peak(model, fp, xb, t, ctx, True)
    detail = f"{case}: inference {inf}, training {train}, bound {bound} ({floor} + {block} {ws[block]})"
    print(detail)
    assert inf <= bound, detail
    assert train > 1.2 * bound, detail


def test_inference_peak_grows_only_by_the_extra_skips():
    acfg = (None, None, {"heads": 8}, {"heads": 8})
    x, t, _ = _inputs(PEAK_B, PEAK_RES, False, 7)
    xb = x.bfloat16()
    peaks, floors = {}, {}
    for n in (1, 3):
        model = Unet(attention_configs=acfg, num_res_blocks=n, dtype=torch.bfloat16)
        fp = _random_params(model, 8)
        floors[n] = _budget(model, PEAK_B, PEAK_RES, PEAK_RES)[0]
        peaks[n] = (_peak(model, fp, xb, t, None, False), _peak(model, fp, xb, t, None, True))
        del model, fp
        torch.cuda.empty_cache()
    (inf1, train1), (inf3, train3) = peaks[1], peaks[3]
    extra = floors[3] - floors[1]                 # the extra concat buffers and timestep rows
    detail = f"inference {inf1} -> {inf3}, training {train1} -> {train3}, extra skips {extra}"
    print(detail)
    assert inf3 - inf1 <= extra + SLACK, detail
    assert train3 - train1 > extra, detail


# ---------------------------------------------------------------------------------------------- CFG sampling graph
def test_cfg_euler_ancestral_whole_step_graph_matches_eager_bitwise():
    model = _model(dict(feature_depths=(64, 128, 256), attention_configs=(None, FULL, {"heads": 8})), True)
    fp = _random_params(model, 9)
    enc = RandomEmbeddingEncoder(77, 768, device=dev)
    ctx = enc(["a cat", "a dog"]).to(dev)
    sched, tr = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev), KarrasPredictionTransform(0.5)
    cfg = DiffusionInputConfig("image", (8, 8, 3), [ConditionalInputConfig(enc)])
    key = utils.jax_key(12)
    outs, smps = [], []
    for graph in (False, True):
        smp = EulerAncestralSampler(model, sched, tr, cfg, guidance_scale=3.0, use_cuda_graph=graph)
        outs.append(smp.generate_samples(fp, 2, 8, diffusion_steps=6, start_step=1000, device=dev,
                                         rngstate=utils.RandomMarkovState(key), model_conditioning_inputs=(ctx,)))
        smps.append(smp)
    assert any(k[0] == "step" for k in smps[1]._graphs)          # the whole-step graph ran
    assert outs[0].shape == (2, 8, 8, 3) and torch.isfinite(outs[0]).all() and outs[0].abs().max() > 0
    assert torch.equal(outs[1], outs[0])
