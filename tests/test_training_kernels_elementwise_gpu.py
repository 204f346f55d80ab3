"""The kernels that run once per training step over every parameter or sample, compared element by element with
the float64 references of tests/elementwise_ref.py: the optimiser (adam / adamw / LAMB, clip_by_global_norm,
DynamicScale), fdx_grad_stats, fdx_ema_update, fdx_dynscale_update (csrc/fdx_optim.cu), the time embedding
(csrc/fdx_misc.cu) and the diffusion / loss / sampler streams (csrc/fdx_stream.cu).

The optimiser runs over the flat buffer of the UNet the tests train (234 tensors, 32,040,768 elements, the
smallest 3), so every thread's grid-stride loop runs about 30 times and LAMB's per-tensor sums meet the real
segment layout.  Outputs are compared against per-element bounds derived in elementwise_ref (never tuned to a
run); copies and casts that must be exact are compared bit for bit.  Each check prints `WORST <name> <x>`, the
largest |err| / bound it saw."""
import ctypes
import math

import numpy as np
import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops, utils
from flaxdiff_b200._lib import OPT_ADAM, OPT_LAMB, check, load, ptr, stream_ptr
from flaxdiff_b200.models.params import FlatParams
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.trainer import DynamicScale, TrainState, adamw, chain, clip_by_global_norm

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
B1, B2, EPS, LR, WD = 0.9, 0.999, 1e-8, 2.7e-4, 1e-4


def sms() -> int:
    return torch.cuda.get_device_properties(dev).multi_processor_count


def chk(name, got, val, delta, bound=None):
    b = R.f32_bound(val, delta) if bound is None else bound
    print(f"WORST {name} {R.assert_elementwise(got, val, b, name):.3f}")


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32),
                       b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32))


_powf = ctypes.CDLL("libm.so.6").powf
_powf.restype, _powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]


def bc(b: float, step: int) -> float:
    """1.f - powf(b, step), as fdx_optimizer_step computes it on the host (the same libm powf)."""
    return float(np.float32(1.0) - np.float32(_powf(b, float(step))))


_LAYOUT = None


def layout():
    """(ParamLayout, slot offsets, tensor sizes, slot lengths, mask of parameter elements) of the UNet."""
    global _LAYOUT
    if _LAYOUT is None:
        lay = Unet(attention_configs=(None,) * 4).layout()
        offs = [o for o, _ in lay.table.values()]
        lens = [math.prod(s) for _, s in lay.table.values()]
        slots = [b - a for a, b in zip(offs, offs[1:] + [lay.total])]
        mask = torch.zeros(lay.total, dtype=torch.bool, device=dev)
        for o, n in zip(offs, lens):
            mask[o:o + n] = True
        _LAYOUT = (lay, offs, lens, slots, mask)
    return _LAYOUT


def test_layout_is_the_full_unet():
    lay, offs, lens, slots, _ = layout()
    assert (len(lens), lay.total, min(lens)) == (234, 32040768, 3)
    # adjacent 64-element tensors: the warps of lamb_pass1_kernel that straddle two segments
    assert any(a == b == 64 for a, b in zip(slots, slots[1:]))


def opt_buffers(seed, n=None, specials=True):
    """p, g, m, v (f32, zero in the gaps between tensors) over the UNet layout, with unused parameters
    (g = m = v = 0), subnormal and large gradients in the first tensors' range."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    _, _, _, _, mask = layout()
    n = mask.numel() if n is None else n
    r = lambda s=1.0: torch.randn(n, generator=gen, device=dev) * s  # noqa: E731
    p, g = r(0.05), r()
    m = r(0.1 / 8)
    v = (r(1 / 8) ** 2) * r().abs()
    if specials:
        g[1000:5096] = 0
        m[1000:5096] = 0
        v[1000:5096] = 0
        g[8192:12288] = r()[8192:12288] * 1e-40             # subnormal f32
        g[16384:20480] = r()[16384:20480] * 1e15            # large: (g/8)^2 still a normal f32
    mk = mask[:n].float()
    return [(t * mk).contiguous() for t in (p, g, m, v)]


# ----------------------------------------------------------------------------------------------- grad stats
def _sumsq_case(n, seed=0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    g = torch.randn(n, generator=gen, device=dev) * torch.exp(torch.randn(n, generator=gen, device=dev) * 2)
    return g


@pytest.mark.parametrize("which", ["4", "260", "sweep+4", "unet"])
def test_grad_stats_sum_of_squares(which):
    n = {"4": 4, "260": 260, "sweep+4": 4 * 8 * sms() * 256 + 4, "unet": layout()[0].total}[which]
    g = _sumsq_case(n)
    g64 = g.to(F64)
    D = R.grad_stats_depth(n, sms())
    out = ops.grad_stats(g)
    val, delta = R.sumsq_ref(g64, 1.0, D)
    chk(f"grad_stats_sumsq_{which}", out[:1], val.reshape(1), delta.reshape(1))
    assert out[1].item() == 0
    # with a DynamicScale state: the squares of g / scale
    st = torch.tensor([2.0 ** 20, 0.0, 1.0], device=dev)
    out = ops.grad_stats(g, st)
    val, delta = R.sumsq_ref(g64, 2.0 ** -20, D)
    chk(f"grad_stats_sumsq_scaled_{which}", out[:1], val.reshape(1), delta.reshape(1))
    assert out[1].item() == 0


NONFINITE = {
    "nan": ({777: math.nan}, 1),
    "inf_first": ({0: math.inf}, 1),
    "minus_inf_last": ({-1: -math.inf}, 1),
    "inf_minus_inf_one_float4": ({4100: math.inf, 4101: -math.inf}, 2),
    "finite_overflow_one_float4": ({4100: 3e38, 4101: 3e38}, 0),
}


@pytest.mark.parametrize("case", list(NONFINITE))
def test_grad_stats_counts_non_finite_elements(case):
    """out[1] counts non-finite ELEMENTS, each tested on its own: finite values whose sum overflows are
    finite (flax's DynamicScale tests isfinite per element and takes that step)."""
    n = 4 * 8 * sms() * 256 + 4
    g = _sumsq_case(n, 1)
    put, count = NONFINITE[case]
    for i, x in put.items():
        g[i] = x
    out = ops.grad_stats(g)
    assert out[1].item() == count, (case, out.tolist())
    if count == 0:
        assert out[0].item() == math.inf           # (3e38)^2 overflows the sum of squares, correctly
    else:
        assert not math.isfinite(out[0].item())


# ----------------------------------------------------------------------------------------------- adam / adamw
def _check_adam(tag, p, g, m, v, got_p, got_m, got_v, *, lr, bc1, bc2, wd, mul, rho_mul=0.0):
    r = R.adam_ref(p, g, m, v, lr=R.f32(lr), b1=R.f32(B1), b2=R.f32(B2), eps=R.f32(EPS), wd=R.f32(wd),
                   bc1=bc1, bc2=bc2, mul=mul, rho_mul=rho_mul)
    chk(f"{tag}_p", got_p, *r["p"])
    chk(f"{tag}_m", got_m, *r["m"])
    chk(f"{tag}_v", got_v, *r["v"])
    return r


@pytest.mark.parametrize("step", [1, 2, 1000, 10 ** 6])
@pytest.mark.parametrize("ema_shadow", [True, False])
def test_adam_unet_layout(step, ema_shadow):
    """fdx_optimizer_step (adamw with EMA and the bf16 shadow; adam alone) over the whole UNet buffer,
    grad_scale = 1/8."""
    p, g, m, v = opt_buffers(step)
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    wd = WD if ema_shadow else 0.0
    ema = (p + 0.01 * torch.randn_like(p)) if ema_shadow else None
    ema64 = ema.to(F64) if ema_shadow else None
    sh = torch.full(p.shape, math.nan, dtype=torch.bfloat16, device=dev) if ema_shadow else None
    tp, tm, tv = p.clone(), m.clone(), v.clone()
    ops.optimizer_step(OPT_ADAM, tp, g, tm, tv, ema, sh, LR, B1, B2, EPS, wd, step, 0.999, grad_scale=0.125)
    r = _check_adam(f"adam_step{step}", p64, g64, m64, v64, tp, tm, tv, lr=LR, bc1=bc(B1, step), bc2=bc(B2, step),
                    wd=wd, mul=0.125)
    if ema_shadow:
        pv, pd = r["p"]
        chk(f"adam_step{step}_ema", ema, *R.ema_ref(ema64, pv, R.f32(0.999), pd))
        assert bits_equal(sh, tp.bfloat16()), "the bf16 shadow is not bf16(p)"
    # unused parameters stay exactly where weight decay puts them
    assert torch.all(tm[1000:5096] == 0) and torch.all(tv[1000:5096] == 0)


def test_adamw_ema_step_device_hyperparameters():
    """fdx_adamw_ema_step with {lr, 1 - b1^t, 1 - b2^t} on the device (the CUDA-graph path): computed in float64
    on the host and rounded, so the reference uses those f32 values, not the host powf."""
    step = 1000
    p, g, m, v = opt_buffers(11)
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    ema = p.clone()
    sh = torch.full(p.shape, math.nan, dtype=torch.bfloat16, device=dev)
    dyn = torch.tensor([LR, 1 - B1 ** step, 1 - B2 ** step], dtype=torch.float32, device=dev)
    lr32, b1c, b2c = (float(x) for x in dyn.cpu())
    tp, tm, tv = p.clone(), m.clone(), v.clone()
    ops.adamw_ema_step(tp, g, tm, tv, ema, sh, 1.0, B1, B2, EPS, WD, 1, 0.999, grad_scale=0.125, dyn=dyn)
    r = _check_adam("adamw_dyn", p64, g64, m64, v64, tp, tm, tv, lr=lr32, bc1=b1c, bc2=b2c, wd=WD, mul=0.125)
    chk("adamw_dyn_ema", ema, *R.ema_ref(p64, r["p"][0], R.f32(0.999), r["p"][1]))
    assert bits_equal(sh, tp.bfloat16())


# ----------------------------------------------------------------------------------------------- clipping
def _rho_clip(n):
    """Relative error of the kernel's clipped multiplier: sqrtf of the grad-stats sum (half its gamma, plus
    one rounding), the product by grad_scale, clip / nrm and the product into the multiplier."""
    return R.gamma(R.grad_stats_depth(n, sms()) + 4) / 2 + 4 * R.U32


@pytest.mark.parametrize("clip", [1e9, 30.0])
def test_clip_by_global_norm_with_grad_scale(clip):
    """optax.chain(clip_by_global_norm, adamw) with grad_scale = 1/8: below and above the clip."""
    step = 7
    p, g, m, v = opt_buffers(21, specials=False)
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    nrm = 0.125 * g64.norm().item()
    clipped = nrm > clip
    assert clipped == (clip == 30.0) and abs(nrm / clip - 1) > 0.01
    gs = ops.grad_stats(g)
    tp, tm, tv = p.clone(), m.clone(), v.clone()
    ops.optimizer_step(OPT_ADAM, tp, g, tm, tv, None, None, LR, B1, B2, EPS, WD, step, grad_scale=0.125,
                       gstats=gs, clip_norm=clip)
    mul = 0.125 * (clip / nrm if clipped else 1.0)
    _check_adam(f"clip_{'above' if clipped else 'below'}", p64, g64, m64, v64, tp, tm, tv, lr=LR, bc1=bc(B1, step),
                bc2=bc(B2, step), wd=WD, mul=mul, rho_mul=_rho_clip(p.numel()) if clipped else 0.0)


@pytest.mark.parametrize("log2_scale", [15, 40, 70])
def test_clip_under_dynamic_scale_equals_unscaled_step(log2_scale):
    """use_dynamic_scale=True with clip_by_global_norm (training.py:604-608): gradients arrive multiplied by the
    loss scale; the clipped step must be the one of the unscaled gradients at every scale.  ||g|| ~ 5.7e3, so at
    2^70 scale ||g|| passes sqrt(FLT_MAX): the norm must be taken of the unscaled gradient."""
    lay, _, _, _, _ = layout()
    p, g, m, v = opt_buffers(31, specials=False)
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    scale = 2.0 ** log2_scale
    ds = DynamicScale(scale=scale)
    st = TrainState.create(None, FlatParams(lay, p.clone()), FlatParams(lay, p.clone()),
                           chain(clip_by_global_norm(1.0), adamw(LR)), dynamic_scale=ds)
    st.opt_state["mu"].copy_(m)
    st.opt_state["nu"].copy_(v)
    st.opt_state["count"] = 9
    st.apply_gradients(grads=FlatParams(lay, g * scale))
    nrm = g64.norm().item()
    assert nrm > 1e3
    _check_adam(f"dynscale_clip_2^{log2_scale}", p64, g64, m64, v64, st.params.flat, st.opt_state["mu"],
                st.opt_state["nu"], lr=LR, bc1=bc(B1, 10), bc2=bc(B2, 10), wd=WD, mul=1.0 / nrm,
                rho_mul=_rho_clip(p.numel()))
    assert ds.scale == scale and ds.fin_steps == 1


# ----------------------------------------------------------------------------------------------- DynamicScale skip
def _lamb_ws(n):
    _, offs, _, _, _ = layout()
    seg = torch.tensor(offs, dtype=torch.int64, device=dev)
    return seg, torch.full((2 * len(offs),), math.nan, device=dev), torch.full((n,), math.nan, device=dev)


@pytest.mark.parametrize("kind", [OPT_ADAM, OPT_LAMB])
def test_dynamic_scale_skip_leaves_state_bit_identical(kind):
    """A NaN in the buffer's last element: p, m, v and the bf16 shadow are untouched, the EMA still runs."""
    p, g, m, v = opt_buffers(41, specials=False)
    g = g * 2.0 ** 16
    g[-1] = math.nan
    st = torch.tensor([2.0 ** 16, 5.0, 1.0], device=dev)
    gs = ops.grad_stats(g, st)
    assert gs[1].item() == 1
    ema = p + 0.01 * torch.randn_like(p)
    ema64 = ema.to(F64)
    sh = p.bfloat16()
    tp, tm, tv, tsh = p.clone(), m.clone(), v.clone(), sh.clone()
    seg = _lamb_ws(p.numel()) if kind == OPT_LAMB else (None, None, None)
    ops.optimizer_step(kind, tp, g, tm, tv, ema, tsh, LR, B1, B2, EPS, WD, 3, 0.999, gstats=gs, clip_norm=1.0,
                       dynscale=st, seg_offsets=seg[0], seg_norms=seg[1], u_ws=seg[2])
    assert bits_equal(tp, p) and bits_equal(tm, m) and bits_equal(tv, v) and bits_equal(tsh, sh)
    chk(f"skip_{kind}_ema", ema, *R.ema_ref(ema64, p.to(F64), R.f32(0.999)))


# ----------------------------------------------------------------------------------------------- LAMB
@pytest.mark.parametrize("mode", ["plain", "clip_dynscale"])
def test_lamb_unet_layout(mode):
    """optax.lamb over the 234 tensors: every element of p, m, v, the update u, and each tensor's ||p||^2 and
    ||u||^2 (the trust ratio's inputs).  Tensor 5 has ||p|| = 0; tensor 9 has g = m = 0, so with weight decay 0
    its ||u|| = 0 (ratio 1 in both cases)."""
    _, offs, lens, slots, _ = layout()
    step = 5
    p, g, m, v = opt_buffers(51, specials=False)
    p[offs[5]:offs[5] + lens[5]] = 0
    g[offs[9]:offs[9] + lens[9]] = 0
    m[offs[9]:offs[9] + lens[9]] = 0
    p64, g64, m64, v64 = (t.to(F64) for t in (p, g, m, v))
    ema = p.clone()
    sh = torch.full(p.shape, math.nan, dtype=torch.bfloat16, device=dev)
    seg, norms, u_ws = _lamb_ws(p.numel())
    tp, tm, tv = p.clone(), m.clone(), v.clone()
    kw = {}
    wd, mul, rho = 0.01, 1.0, 0.0
    if mode == "clip_dynscale":
        scale = 2.0 ** 20
        st = torch.tensor([scale, 0.0, 1.0], device=dev)
        nrm = g64.norm().item()
        gin = g * scale
        kw = dict(gstats=ops.grad_stats(gin, st), clip_norm=1.0, dynscale=st)
        wd, mul, rho = 0.0, 1.0 / nrm, _rho_clip(p.numel())
        assert nrm > 10
    else:
        gin = g
    ops.optimizer_step(OPT_LAMB, tp, gin, tm, tv, ema, sh, 2e-3, B1, B2, 1e-6, wd, step, 0.99, seg_offsets=seg,
                       seg_norms=norms, u_ws=u_ws, **kw)
    r = R.lamb_ref(p64, g64, m64, v64, seg, torch.tensor(slots, device=dev), lr=R.f32(2e-3), b1=R.f32(B1),
                   b2=R.f32(B2), eps=R.f32(1e-6), wd=R.f32(wd), bc1=bc(B1, step), bc2=bc(B2, step), mul=mul,
                   rho_mul=rho)
    for name, got in (("p", tp), ("m", tm), ("v", tv), ("u", u_ws)):
        chk(f"lamb_{mode}_{name}", got, *r[name])
    chk(f"lamb_{mode}_sum_p2", norms[0::2], *r["np2"])
    chk(f"lamb_{mode}_sum_u2", norms[1::2], *r["nu2"])
    assert r["np2"][0][5].item() == 0 and norms[10].item() == 0
    if mode == "clip_dynscale":
        assert r["nu2"][0][9].item() == 0 and norms[19].item() == 0
    pv, pd = r["p"]
    chk(f"lamb_{mode}_ema", ema, *R.ema_ref(p64, pv, R.f32(0.99), pd))
    assert bits_equal(sh, tp.bfloat16())


# ----------------------------------------------------------------------------------------------- EMA
@pytest.mark.parametrize("decay", [0.0, 0.999, 1.0])
def test_ema_update_unet_layout(decay):
    p, _, m, _ = opt_buffers(61, specials=False)
    ema = p + m
    e0 = ema.clone()
    ops.ema_update(ema, p, decay)
    chk(f"ema_update_{decay}", ema, *R.ema_ref(e0.to(F64), p.to(F64), R.f32(decay)))
    if decay == 0.0:                   # exact (as values: 0 ema + p turns a -0 of p into +0)
        assert torch.equal(ema, p)
    elif decay == 1.0:
        assert torch.equal(ema, e0)


# ----------------------------------------------------------------------------------------------- dynscale update
FLT_MAX = float(np.finfo(np.float32).max)
TINY32 = float(np.finfo(np.float32).tiny)


def flax_dynscale_rule(scale, steps, finite, growth=2.0, backoff=0.5, interval=2000, min_scale=TINY32):
    """flax.training.dynamic_scale.DynamicScale.value_and_grad's update, in f32 as jnp evaluates it."""
    f = np.float32
    scale, growth, backoff = f(scale), f(growth), f(backoff)
    grow = steps == interval
    with np.errstate(over="ignore"):
        fin_scale = np.minimum(scale * growth, f(FLT_MAX)) if (grow and finite) else scale
    inf_scale = np.maximum(scale * backoff, f(min_scale))
    new_scale = fin_scale if finite else inf_scale
    new_steps = 0 if (grow or not finite) else steps + 1
    return float(new_scale), float(new_steps), 1.0 if finite else 0.0


DYNSCALE_CASES = [
    # (scale, fin_steps, finite, growth_interval, minimum_scale)
    (65536.0, 0, True, 2000, TINY32),
    (65536.0, 1999, True, 2000, TINY32),          # one short of the interval: no growth, counter 2000
    (65536.0, 2000, True, 2000, TINY32),          # exactly at the interval: doubled, counter reset
    (65536.0, 1234, False, 2000, TINY32),         # non-finite: halved, counter reset
    (65536.0, 2000, False, 2000, TINY32),         # non-finite at the interval: halved, not grown
    (2.0 ** 127, 2, True, 2, TINY32),             # growth past FLT_MAX: capped at FLT_MAX
    (FLT_MAX, 2, True, 2, TINY32),
    (TINY32, 7, False, 2000, TINY32),             # halving below minimum_scale: floored
    (3.0, 7, False, 2000, 2.0),                   # a user-set minimum_scale
    (1.0, 0, True, 1, TINY32),
]


@pytest.mark.parametrize("case", range(len(DYNSCALE_CASES)))
def test_dynscale_update_transition_table(case):
    scale, steps, finite, interval, mn = DYNSCALE_CASES[case]
    st = torch.tensor([scale, float(steps), 0.0 if finite else 1.0], dtype=torch.float32, device=dev)
    gs = torch.tensor([1.0, 0.0 if finite else 3.0], device=dev)
    ops.dynscale_update(st, gs, 2.0, 0.5, interval, mn)
    want = torch.tensor(flax_dynscale_rule(scale, steps, finite, interval=interval, min_scale=mn),
                        dtype=torch.float32, device=dev)
    assert bits_equal(st, want), (DYNSCALE_CASES[case], st.tolist(), want.tolist())


# ----------------------------------------------------------------------------------------------- time embedding
def _time_embed_bwd_ws(demb, saved, W2, dW1, db1, dW2, db2):
    four, h1, h2 = saved
    B, D = demb.shape
    ws1 = torch.full_like(demb, math.nan)
    ws2 = torch.full_like(demb, math.nan)
    check(load().fdx_time_embed_bwd(ptr(demb), ptr(four), ptr(h1), ptr(h2), ptr(W2), ctypes.c_int(B),
                                    ctypes.c_int(D), ptr(ws1), ptr(ws2), ptr(dW1), ptr(db1), ptr(dW2), ptr(db2),
                                    stream_ptr()), "time_embed_bwd")
    return ws1, ws2


@pytest.mark.parametrize("B", [1, 7, 8, 63, 64, 65, 256])
@pytest.mark.parametrize("D", [32, 64, 256, 512, 1024])
def test_time_embedding_elementwise(D, B):
    """FourierEmbedding + TimeProjection forward and backward: `four` within 2 ulp of the float64 sine / cosine
    of the kernel's f32 phase, t in the EDM model-time range and at DDPM integer steps 0 ... 999; the
    batch slices of dense_wgrad_small (1 / 4 / 16, ragged last slice) onto a zero and a non-zero prior."""
    gen = torch.Generator(device=dev).manual_seed(D * 1000 + B)
    freqs = torch.from_numpy(utils.normal(utils.PRNGKey(42), D // 2) * 16.0).float().to(dev)
    W1 = torch.randn(D, D, generator=gen, device=dev) / math.sqrt(D)
    W2 = torch.randn(D, D, generator=gen, device=dev) / math.sqrt(D)
    b1 = torch.randn(D, generator=gen, device=dev) * 0.1
    b2 = torch.randn(D, generator=gen, device=dev) * 0.1
    f64 = lambda t: t.to(F64)  # noqa: E731
    for regime in ("edm", "ddpm"):
        if regime == "edm":
            t = torch.rand(B, generator=gen, device=dev) * 2.65 - 1.55
        else:
            t = torch.randint(0, 1000, (B,), generator=gen, device=dev).float()
            t[0] = 999.0
            if B > 1:
                t[1] = 0.0
        emb, emb16, saved = ops.time_embed_fwd(t, freqs, W1, b1, W2, b2)
        four, h1, h2 = saved
        ref = R.time_embed_fwd_ref(R.time_phase_f32(t, freqs), f64(four), f64(h1), f64(h2), f64(W1), f64(b1),
                                   f64(W2), f64(b2))
        tag = f"temb_D{D}_B{B}_{regime}"
        fv, fb = ref["four"]
        chk(f"{tag}_four", four, fv, None, bound=fb)
        for name, got in (("h1", h1), ("h2", h2), ("emb", emb)):
            chk(f"{tag}_{name}", got, *ref[name])
        assert bits_equal(emb16, emb.bfloat16())
        demb = torch.randn(B, D, generator=gen, device=dev)
        for prior in ("zero", "prior"):
            s = 0.0 if prior == "zero" else 0.3
            dW1, dW2 = (torch.randn(D, D, generator=gen, device=dev) * s for _ in range(2))
            db1, db2 = (torch.randn(D, generator=gen, device=dev) * s for _ in range(2))
            p0 = [f64(x) for x in (dW1, db1, dW2, db2)]
            ws1, ws2 = _time_embed_bwd_ws(demb, saved, W2, dW1, db1, dW2, db2)
            rb = R.time_embed_bwd_ref(f64(demb), f64(four), f64(h1), f64(h2), f64(ws1), f64(ws2), f64(W2), *p0)
            for name, got in (("dh2", ws2), ("dh1", ws1), ("dW1", dW1), ("db1", db1), ("dW2", dW2), ("db2", db2)):
                chk(f"{tag}_{prior}_{name}", got, *rb[name])


# ----------------------------------------------------------------------------------------------- streams
def _loss_depth(n_total):
    """loss_kernel: per thread one term per grid-stride iteration, warp and block trees, one atomic per block."""
    n4 = n_total // 4
    blocks = max(1, min(math.ceil(n4 / 256), 8 * sms()))
    return math.ceil(n4 / (blocks * 256)) + 10 + blocks


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("src", ["u8", "f32"])
@pytest.mark.parametrize("B", [1, 5, 256])
def test_diffuse_forward_and_loss_elementwise(B, src, kind):
    """fdx_diffuse_forward (normalise, noise, c_in, x0 / eps / v target) at 64x64x3 with u8 pixels 0 and 255
    (exactly -1 and +1), then fdx_loss_fwd_bwd on the kernel's own x_t and target."""
    gen = torch.Generator(device=dev).manual_seed(B * 10 + kind)
    E = 64 * 64 * 3
    if src == "u8":
        x0 = torch.randint(0, 256, (B, 64, 64, 3), generator=gen, device=dev, dtype=torch.uint8)
        x0[:, 0, :2] = 0
        x0[:, 1, :2] = 255
    else:
        x0 = torch.randn(B, 64, 64, 3, generator=gen, device=dev)
    eps = torch.randn(B, 64, 64, 3, generator=gen, device=dev)
    sigma = torch.exp(torch.randn(B, generator=gen, device=dev) * 1.2 - 1.2)
    alpha = 1 / torch.sqrt(1 + sigma * sigma)
    c_in = 1 / torch.sqrt(alpha * alpha + sigma * sigma)
    x_t, target, model_in = ops.diffuse_forward(x0, eps, alpha, sigma, c_in, src == "u8", kind)
    ref = R.diffuse_ref(x0.reshape(B, E).to(F64), eps.reshape(B, E).to(F64), alpha.to(F64), sigma.to(F64),
                        src == "u8", kind)
    tag = f"diffuse_B{B}_{src}_k{kind}"
    chk(f"{tag}_x_t", x_t.reshape(B, E), *ref["x_t"])
    chk(f"{tag}_target", target.reshape(B, E), *ref["target"])
    assert bits_equal(model_in, (x_t * c_in[:, None, None, None]).bfloat16())
    if src == "u8" and kind == 0:
        assert torch.all(target[:, 0, :2] == -1.0) and torch.all(target[:, 1, :2] == 1.0)
    if kind == 1:
        assert bits_equal(target, eps)
    F = torch.randn(B, 64, 64, 3, generator=gen, device=dev)
    c_out = torch.rand(B, generator=gen, device=dev) + 0.2
    c_skip = torch.rand(B, generator=gen, device=dev)
    weight = torch.exp(torch.randn(B, generator=gen, device=dev))
    loss, dF = ops.loss_fwd_bwd(F, x_t, target, c_out, c_skip, weight)
    rl = R.loss_ref(F.reshape(B, E).to(F64), x_t.reshape(B, E).to(F64), target.reshape(B, E).to(F64),
                    c_out.to(F64), c_skip.to(F64), weight.to(F64), _loss_depth(B * E))
    lv, ld = rl["loss"]
    chk(f"loss_B{B}_{src}_k{kind}", loss, lv.reshape(1), ld.reshape(1))
    chk(f"loss_dF_B{B}_{src}_k{kind}", dF.reshape(B, E), *rl["dF"])


@pytest.mark.parametrize("n_in", [1, 2, 3, 4, 5, 6])
def test_affine_combine_elementwise(n_in):
    """out1 / out2 of up to six inputs with per-sample coefficients, the bf16 output with bf16_scale, and the
    clip with values exactly on its bounds."""
    gen = torch.Generator(device=dev).manual_seed(n_in)
    B, E = 5, 64 * 64 * 3
    ins = [torch.randn(B, E, generator=gen, device=dev) for _ in range(n_in)]
    c1 = torch.randn(n_in, B, generator=gen, device=dev)
    c2 = torch.randn(n_in, B, generator=gen, device=dev)
    s = torch.rand(B, generator=gen, device=dev) + 0.5
    o1, o2, ob = ops.affine_combine(ins, c1, c2, bf16_scale=s, want_bf16=True)
    for name, got, c in (("out1", o1, c1), ("out2", o2, c2)):
        chk(f"affine_n{n_in}_{name}", got, *R.affine_ref([x.to(F64) for x in ins], c.to(F64)))
    assert bits_equal(ob, (o1 * s[:, None]).bfloat16())
    # clip: a single input with coefficient 1 is exact, so values on the bounds stay on them
    x = ins[0].clone()
    x[:, :4] = torch.tensor([-1.0, 1.0, -1.0000001, 1.0000001], device=dev)
    lo, hi = -1.0, 1.0
    c, _, cb = ops.affine_combine([x], torch.ones(1, B, device=dev), want_bf16=True, clip=(lo, hi))
    assert bits_equal(c, x.clamp(lo, hi))
    assert bits_equal(cb, c.bfloat16())
    assert torch.all(c[:, :4] == torch.tensor([-1.0, 1.0, -1.0, 1.0], device=dev))
    if n_in > 1:
        c, _, _ = ops.affine_combine(ins, c1, clip=(lo, hi))
        v, d = R.affine_ref([t.to(F64) for t in ins], c1.to(F64))
        chk(f"affine_n{n_in}_clip", c, v.clamp(lo, hi), d)


def test_affine_clip_propagates_nan():
    """jnp.clip keeps a NaN (the sampler's final clip_images must not turn a diverged sample into -1)."""
    x = torch.randn(2, 64, device=dev)
    x[0, 5] = math.nan
    x[1, 7] = math.inf
    c, _, _ = ops.affine_combine([x], torch.ones(1, 2, device=dev), clip=(-1.0, 1.0))
    assert math.isnan(c[0, 5].item()) and c[1, 7].item() == 1.0
    ok = torch.ones_like(x, dtype=torch.bool)
    ok[0, 5] = False
    assert bits_equal(c[ok], x.clamp(-1.0, 1.0)[ok])
