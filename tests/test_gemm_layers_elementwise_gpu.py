"""The dense GEMM engine (fdx_gemm in modes KK, KMN and MNMN, and fdx_gemm_cat) compared element by element with
float64 at every call the models make.

A recorder wraps ops.gemm and ops.gemm_cat (linear_fwd, linear_cat_fwd, _dense_wgrad and _dense_dgrad reach them
through those module attributes) and runs each model once forward with its tape, once backward and once through the
inference forward: the transformer denoisers at the reference's widths (F = 768, 12 heads, MLP ratio 4, patch 2 at
64 x 64, B = 16, a 77 x 768 text context) and at their test suites' small widths (F = 64, 128, 192), the UNet of
the text-conditioned sampling workload (sampled at its model batch of 64, trained at B = 2), and the CLIP text and
vision towers.  Every call becomes a descriptor: mode,
M, N, K, K0, batch, every leading dimension and batch stride, alpha, bias, residual (and whether it is the output
itself), output type, atomic and batch reduction, and each operand's address modulo 128.

Each distinct descriptor of a family is replayed in the two kinds of test_conv_elementwise_gpu.py:
  * dense: random bf16 operands, each output within the per-element bound of elementwise_ref.gemm_ref (the worst
    |err| / bound is printed as `WORST <case> <ratio>`);
  * exact: integer operands in {-2, ..., 2} (B scaled by a power of two), integer bias, residual and prior; every
    output's sum of |terms| is below 2^24, so f32 outputs equal the float64 result and bf16 outputs its bf16
    rounding, bit for bit.  This is what sees a dropped k-chunk, split or column tile.
Outputs live in buffers with the recorded leading dimensions and batch strides, guard bands on both sides and gaps
that hold a sentinel, which must come back bit-identical.  Outputs that are not accumulated start as NaN, atomic
ones from a random prior, and a residual that is the output is replayed as the output.  Every gemm_cat output is
also bit for bit gemm's on the materialised concatenation.  A few fixed descriptors add what no model issues:
alpha != 1, and a bias on a split-K weight-gradient reduction.  A last test asserts that the recorded descriptors
still contain every class of launch the models are known to issue."""
import ctypes
import dataclasses
import functools
import inspect
import math
import os
import sys
import time

import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import _lib, ops
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
SENTINEL = -1234.0                                   # exactly representable in bf16
GUARD = 256                                          # bytes of sentinel before and after every output
KINDS = ("dense", "exact")
MODE = {GEMM_KK: "KK", GEMM_KMN: "KMN", GEMM_MNMN: "MNMN"}


def sms() -> int:
    return _lib.load().fdx_device_sm_count()


# ----------------------------------------------------------------------------------------------- the recorder
@dataclasses.dataclass(frozen=True)
class Desc:
    cat: bool
    mode: int
    M: int
    N: int
    K: int
    K0: int                                          # gemm_cat: the k where A switches from A0 to A1; else 0
    b1: int
    b2: int
    a_ld: int
    a_s: tuple
    a1_ld: int
    b_ld: int
    b_s: tuple
    d_ld: int
    d_s: tuple
    alpha: float                                     # as the f32 the descriptor carries
    bias: bool
    res: bool
    r_ld: int
    r_s: tuple
    d_f32: bool
    atomic: bool
    reduce_batch: bool
    alias: bool                                      # res is D
    off: tuple                                       # data_ptr() % 128 of A, A1, B, D, bias, res (-1: absent)


_GEMM, _CAT = ops.gemm, ops.gemm_cat
_HELPERS = ("_dense_wgrad", "_dense_dgrad")


def _site() -> str:
    """The model code that issued the call: the first frame under models/ outside the dense-layer helpers."""
    f = sys._getframe(2)
    while f is not None:
        fn = f.f_code.co_filename
        if os.sep + "models" + os.sep in fn and f.f_code.co_name not in _HELPERS:
            return f"{os.path.basename(fn)}:{f.f_lineno} {f.f_code.co_name}"
        f = f.f_back
    return "?"


def _off(t):
    return -1 if t is None else t.data_ptr() % 128


def _describe(cat: bool, a) -> Desc:
    D, res = a["D"], a["res"]
    A = a["A0"] if cat else a["A"]
    return Desc(cat=cat, mode=a["mode"], M=a["M"], N=a["N"], K=a["K"], K0=a["K0"] if cat else 0,
                b1=max(1, a.get("batch1", 1)), b2=max(1, a.get("batch2", 1)), a_ld=a["a_ld"],
                a_s=tuple(a.get("a_s", (0, 0))), a1_ld=a["a1_ld"] if cat else 0, b_ld=a["b_ld"],
                b_s=tuple(a.get("b_s", (0, 0))), d_ld=a["d_ld"], d_s=tuple(a.get("d_s", (0, 0))),
                alpha=ctypes.c_float(a.get("alpha", 1.0)).value, bias=a["bias"] is not None,
                res=res is not None, r_ld=a["r_ld"] if res is not None else 0,
                r_s=tuple(a.get("r_s", (0, 0))) if res is not None else (0, 0), d_f32=D.dtype == torch.float32,
                atomic=bool(a.get("atomic", False)), reduce_batch=bool(a.get("reduce_batch", False)),
                alias=res is not None and res.data_ptr() == D.data_ptr(),
                off=(_off(A), _off(a["A1"]) if cat else -1, _off(a["B"]), _off(D), _off(a["bias"]), _off(res)))


class Recorder:
    """While active, every ops.gemm / ops.gemm_cat call is run and its descriptor kept with its first call site."""

    def __init__(self):
        self.seen = {}
        self.label = ""

    def _wrap(self, fn, cat):
        sig = inspect.signature(fn)

        @functools.wraps(fn)
        def call(*args, **kwargs):
            b = sig.bind(*args, **kwargs)
            b.apply_defaults()
            d = _describe(cat, b.arguments)
            self.seen.setdefault(d, f"{self.label} {_site()}")
            return fn(*args, **kwargs)
        return call

    def __enter__(self):
        ops.gemm, ops.gemm_cat = self._wrap(_GEMM, False), self._wrap(_CAT, True)
        return self

    def __exit__(self, *exc):
        ops.gemm, ops.gemm_cat = _GEMM, _CAT


# ----------------------------------------------------------------------------------------------- the workloads
def _denoiser(cls, kw, res, B, text):
    """One forward with its tape, one backward and one inference forward of a transformer denoiser."""
    torch.manual_seed(0)
    model = cls(**kw)
    ctx = torch.randn(B, *text, device=dev) if text else None
    fp = model.init(3, textcontext=ctx, device=dev)
    x = torch.randn(B, *res, 3, device=dev).bfloat16()
    t = torch.rand(B, device=dev) * 2 - 1
    _, saved = model.forward(fp, x, t, ctx, save=True)
    grads = fp.zeros_like()
    model.backward(fp, saved, torch.randn(B, *res, 3, device=dev), grads)
    del saved, grads
    model.forward(fp, x, t, ctx, save=False)


def _unet(acfg, res, B, context_dim, train=True):
    """train: one forward with its tape and one backward, then the inference forward; else the inference forward."""
    from flaxdiff_b200.models.simple_unet import Unet
    torch.manual_seed(0)
    model = Unet(attention_configs=acfg, dtype=torch.bfloat16, context_dim=context_dim)
    fp = model.init(4, device=dev)
    x = torch.randn(B, res, res, 3, device=dev).bfloat16()
    t = torch.randn(B, device=dev)
    ctx = torch.randn(B, 77, context_dim, device=dev).bfloat16() if context_dim else None
    if train:
        _, saved = model.forward(fp, x, t, ctx, save=True)
        grads = fp.zeros_like()
        model.backward(fp, saved, torch.randn(B, res, res, 3, device=dev), grads)
        del saved, grads
    model.forward(fp, x, t, ctx, save=False)


def _clip_text(kind, B):
    from clip_text_ref import clip_model, token_batch
    from flaxdiff_b200.models.clip_text import CLIPTextTower
    model = clip_model(kind)
    tower = CLIPTextTower.from_transformers(model, dev)
    ids, mask = token_batch(model.config.vocab_size, [int(n) for n in torch.arange(B) * 7 % 76], seed=1)
    tower.encode(ids.to(dev), mask.to(dev))


def _clip_vision(kind, B):
    from transformers.models.clip import CLIPImageProcessorPil

    from clip_metric_ref import clip_pair_model
    from clip_text_ref import token_batch
    from flaxdiff_b200.models.clip_vision import CLIPPair
    model = clip_pair_model(kind)
    pair = CLIPPair.from_transformers(model, CLIPImageProcessorPil(), dev)
    x = torch.rand(B, 224, 224, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1
    pair.image_embeds(x.to(dev))
    ids, mask = token_batch(model.config.text_config.vocab_size, [int(n) for n in torch.arange(B) * 5 % 76], seed=2)
    pair.text_embeds(ids.to(dev), mask.to(dev))


def _families():
    from flaxdiff_b200.models.mmdit import HierarchicalMMDiT, SimpleMMDiT
    from flaxdiff_b200.models.simple_dit import SimpleDiT
    from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT
    from flaxdiff_b200.models.udit import SimpleUDiT
    from flaxdiff_b200.models.uvit import UViT
    # the reference's default widths; depth only as far as it takes to reach every kind of layer
    ref = dict(patch_size=2, emb_features=768, num_heads=12, mlp_ratio=4)
    big = dict(res=(64, 64), B=16)
    t77 = (77, 768)

    def small(kw, res, text=None):                   # the families' own test configurations, at B = 2
        return dict(kw=kw, res=res, B=2, text=text)

    uv = dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2)
    den = {
        "simple_dit": (SimpleDiT, {
            "ref": dict(kw=dict(ref, num_layers=2), text=None, **big),
            "ref_sigma": dict(kw=dict(ref, num_layers=2, learn_sigma=True), text=None, **big),
            "ref_text77": dict(kw=dict(ref, num_layers=2), text=t77, **big),
            "f64_p2": small(dict(patch_size=2, emb_features=64, num_layers=2, num_heads=2), (16, 16)),
            "f192_p4_sigma": small(dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4, learn_sigma=True),
                                   (32, 16)),
            "f128_p2_text": small(dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2), (16, 16), (7, 64)),
        }),
        "ssm_dit": (HybridSSMAttentionDiT, {
            "ref_3to1_text77": dict(kw=dict(ref, num_layers=4), text=t77, **big),
            "ref_all_ssm": dict(kw=dict(ref, num_layers=1, ssm_attention_ratio="all-ssm", learn_sigma=True),
                                text=None, **big),
            "f64_all_ssm": small(dict(patch_size=2, emb_features=64, num_heads=2, ssm_state_dim=16, num_layers=2,
                                      ssm_attention_ratio="all-ssm"), (16, 16)),
            "f128_3to1_text_sigma": small(dict(patch_size=2, emb_features=128, num_heads=2, ssm_state_dim=32,
                                               num_layers=4, learn_sigma=True), (16, 16), (7, 64)),
            "f64_hilbert_6x4": small(dict(patch_size=4, emb_features=64, num_heads=2, ssm_state_dim=16, num_layers=2,
                                          ssm_attention_ratio="1:1", use_hilbert=True), (24, 16)),
            "f64_unidirectional": small(dict(patch_size=2, emb_features=64, num_heads=2, ssm_state_dim=16,
                                             num_layers=2, ssm_attention_ratio="all-ssm", bidirectional_ssm=False),
                                        (16, 16)),
        }),
        "mmdit": (SimpleMMDiT, {
            "ref_text77": dict(kw=dict(ref, num_layers=2), text=t77, **big),
            "ref_text2d_sigma": dict(kw=dict(ref, num_layers=1, learn_sigma=True), text=(768,), **big),
            "f128_text3d_sigma": small(dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2,
                                            learn_sigma=True), (16, 16), (7, 64)),
            "f192_text2d": small(dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4), (32, 16), (96,)),
            "f64_hilbert_6x4": small(dict(patch_size=4, emb_features=64, num_layers=2, num_heads=2,
                                          use_hilbert=True), (24, 16), (5, 64)),
        }),
        "hierarchical_mmdit": (HierarchicalMMDiT, {
            "ref_text77": dict(kw=dict(base_patch_size=2, emb_features=(512, 768, 1024), num_layers=(1, 1, 1),
                                       num_heads=(8, 12, 16)), text=t77, **big),
            "two_stages_text3d_sigma": small(dict(base_patch_size=2, emb_features=(64, 128), num_layers=(1, 2),
                                                  num_heads=(2, 2), learn_sigma=True), (16, 24), (7, 64)),
            "three_stages_text2d": small(dict(base_patch_size=2, emb_features=(64, 128, 192), num_layers=(1, 1, 2),
                                              num_heads=(2, 2, 3)), (16, 16), (96,)),
        }),
        "udit": (SimpleUDiT, {
            "ref_text77": dict(kw=dict(ref, num_layers=2), text=t77, **big),
            "ref_sigma": dict(kw=dict(ref, num_layers=2, learn_sigma=True), text=None, **big),
            "f128_text3d_sigma": small(dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2,
                                            learn_sigma=True), (16, 16), (7, 64)),
            "f192_text2d": small(dict(patch_size=4, emb_features=192, num_layers=2, num_heads=4), (32, 16), (96,)),
            "f64_hilbert_6x4": small(dict(patch_size=4, emb_features=64, num_layers=4, num_heads=2,
                                          use_hilbert=True), (24, 16), (5, 64)),
        }),
        "uvit": (UViT, {
            "ref_head_text77": dict(kw=dict(patch_size=2, emb_features=768, num_heads=12, num_layers=2,
                                            add_residualblock_output=True), text=t77, **big),
            "ref_projection": dict(kw=dict(patch_size=2, emb_features=768, num_heads=12, num_layers=2,
                                           use_projection=True, use_self_and_cross=True), text=t77, **big),
            "f128_default": small(uv, (16, 16)),
            "f128_projection": small(dict(uv, use_projection=True), (16, 16), (5, 64)),
            "f128_self_and_cross": small(dict(uv, use_self_and_cross=True), (16, 16)),
            "f128_norm_inputs": small(dict(uv, norm_inputs=True), (16, 16), (5, 64)),
            "f64_hilbert_6x4": small(dict(uv, patch_size=4, emb_features=64, use_hilbert=True), (24, 16)),
            "f128_head_swish": small(dict(uv, add_residualblock_output=True), (16, 16), (5, 64)),
        }),
    }
    fams = {name: {label: functools.partial(_denoiser, cls, c["kw"], c["res"], c["B"], c["text"])
                   for label, c in cfgs.items()} for name, (cls, cfgs) in den.items()}
    # the text-conditioned sampling workload's UNet (bench.py c4): attention at three levels with a 77 x 768 text
    # context at 256 x 256, sampled at its model batch of 64 (B = 32 images, doubled by classifier-free guidance),
    # and trained at B = 2 for the backward's GEMMs
    c4 = (None, {"heads": 8}, {"heads": 8}, {"heads": 8})
    fams["unet"] = {"c4_256px_B64_sample": functools.partial(_unet, c4, 256, 64, 768, train=False),
                    "c4_256px_B2_train": functools.partial(_unet, c4, 256, 2, 768)}
    fams["clip_text"] = {"clip-l_B64": functools.partial(_clip_text, "clip-l", 64),
                         "openclip_B64": functools.partial(_clip_text, "openclip", 64)}
    fams["clip_vision"] = {"vit-l_B16": functools.partial(_clip_vision, "vit-l", 16)}
    return fams


FAMILIES = ("simple_dit", "ssm_dit", "mmdit", "hierarchical_mmdit", "udit", "uvit", "unet", "clip_text",
            "clip_vision")
_RECORDED = {}


def recorded(family: str) -> dict:
    """{Desc: first call site} of every GEMM a family's configurations issue (recorded once per session)."""
    if family not in _RECORDED:
        rec = Recorder()
        with rec:
            for label, run in _families()[family].items():
                rec.label = f"{family}/{label}"
                run()
                torch.cuda.synchronize()
        torch.cuda.empty_cache()
        _RECORDED[family] = rec.seen
    return _RECORDED[family]


# ----------------------------------------------------------------------------------------------- routes and classes
def splits(d: Desc) -> int:
    """fdx_tc_launch's split-K count of an MNMN descriptor: wave-aware for an atomic batch reduction, else 1."""
    sp, _ = R.mnmn_splits(d.K, d.b1, d.b2, d.M, d.N, 1, sms(), gemm=True, splits=0 if d.reduce_batch and d.atomic
                          else 1, mn_batched=not d.reduce_batch)
    return sp


def depth(d: Desc) -> int:
    if d.mode != GEMM_MNMN:
        return d.K + R.EPI
    return R.mnmn_depth(d.K, d.b1, d.b2, d.M, d.N, 1, sms(), gemm=True,
                        splits=0 if d.reduce_batch and d.atomic else 1, mn_batched=not d.reduce_batch)


def route(d: Desc) -> str:
    r = f"tc-bn{R.tc_bn(d.N)}"
    if d.mode == GEMM_MNMN:
        r += f"-split{splits(d)}"
    return r + ("-cat" if d.cat else "")


def case_name(d: Desc, site: str) -> str:
    epi = "+".join(n for n, on in (("bias", d.bias), ("res=D" if d.alias else "res", d.res),
                                    (f"alpha{d.alpha:g}", d.alpha != 1.0), ("atomic", d.atomic)) if on)
    batch = f" b{d.b2}x{d.b1}" + (" reduce" if d.reduce_batch else "") if d.b1 * d.b2 > 1 or d.reduce_batch else ""
    return (f"{MODE[d.mode]} {route(d)} M{d.M} N{d.N} K{d.K}" + (f" K0={d.K0}" if d.cat else "") + batch
            + (f" {epi}" if epi else "") + (" f32" if d.d_f32 else " bf16") + f" [{site}]")


def classes(d: Desc) -> set:
    bn = R.tc_bn(d.N)
    c = {f"mode {MODE[d.mode]}", f"BN {bn}", "out f32" if d.d_f32 else "out bf16"}
    for name, on in (("ragged last column tile", d.N % bn != 0), ("N % 64 = 32", d.N % 64 == 32),
                     ("M % 128 != 0", d.M % 128 != 0), ("bias", d.bias), ("residual", d.res),
                     ("residual aliases D", d.alias), ("alpha != 1", d.alpha != 1.0),
                     ("split count > 1", d.mode == GEMM_MNMN and splits(d) > 1),
                     ("gemm_cat bf16", d.cat and not d.d_f32), ("gemm_cat f32", d.cat and d.d_f32)):
        if on:
            c.add(name)
    return c


# Every class the models are known to issue.  No model call passes alpha != 1, so that class is covered by the
# fixed cases below instead.
MODEL_CLASSES = {"mode KK", "mode KMN", "mode MNMN", "BN 64", "BN 128", "BN 256", "out f32", "out bf16",
                 "ragged last column tile", "N % 64 = 32", "M % 128 != 0", "split count > 1", "bias", "residual",
                 "residual aliases D", "gemm_cat bf16", "gemm_cat f32"}


def _fixed(**kw):
    base = dict(cat=False, mode=GEMM_KMN, M=300, N=96, K=128, K0=0, b1=1, b2=1, a_ld=128, a_s=(0, 0), a1_ld=0,
                b_ld=96, b_s=(0, 0), d_ld=96, d_s=(0, 0), alpha=1.0, bias=False, res=False, r_ld=0, r_s=(0, 0),
                d_f32=False, atomic=False, reduce_batch=False, alias=False, off=(0, -1, 0, 0, -1, -1))
    base.update(kw)
    return Desc(**base)


# Launches no model issues: alpha != 1 in the bf16 epilogue with bias and residual and in the f32 one, and a bias on
# a split-K weight-gradient reduction (132 splits on 132 SMs), which every split used to add.
FIXED = {
    _fixed(mode=GEMM_KK, M=333, N=576, K=768, a_ld=768, b_ld=768, d_ld=640, alpha=0.125, bias=True, res=True,
           r_ld=584, off=(32, -1, 0, 64, 16, 96)): "fixed alpha KK",
    _fixed(mode=GEMM_KMN, M=4928, N=160, K=3072, a_ld=3072, b_ld=160, d_ld=160, alpha=0.25, bias=True,
           d_f32=True): "fixed alpha KMN f32",
    _fixed(mode=GEMM_MNMN, M=128, N=128, K=32768, a_ld=128, b_ld=128, d_ld=128, bias=True, d_f32=True, atomic=True,
           reduce_batch=True, off=(0, -1, 0, 0, 0, -1)): "fixed split-K bias MNMN",
    _fixed(mode=GEMM_MNMN, M=192, N=576, K=4096, b1=4, a_ld=192, b_ld=576, d_ld=584, bias=True, d_f32=True,
           atomic=True, reduce_batch=True, off=(0, -1, 0, 16, 32, -1)): "fixed split-K bias MNMN batch 4",
}


# ----------------------------------------------------------------------------------------------- replay
def draw(n, kind, g, scale=1.0, dtype=torch.bfloat16):
    """dense: N(0, scale^2); exact: integers in {-2..2} times the power of two nearest to scale."""
    if kind == "exact":
        t = torch.randint(-2, 3, (n,), generator=g, device=dev).float() * 2.0 ** round(math.log2(scale))
    else:
        t = torch.randn((n,), generator=g, device=dev) * scale
    return t.to(dtype)


def strided(shape, strides, off_bytes, dtype, fill):
    """A view of `shape` / `strides` (elements) at an address that is off_bytes mod 128, inside a flat buffer with
    GUARD bytes before and after; fill(n) makes the buffer's contents -> (buffer, view)."""
    el = torch.empty((), dtype=dtype).element_size()
    lead = (GUARD + max(off_bytes, 0)) // el
    span = 1 + sum((n - 1) * s for n, s in zip(shape, strides))
    buf = fill(lead + span + GUARD // el)
    assert buf.data_ptr() % 128 == 0
    view = buf.as_strided(shape, strides, lead)
    assert view.data_ptr() % 128 == max(off_bytes, 0), (view.data_ptr() % 128, off_bytes)
    return buf, view


def layouts(d: Desc):
    """(shape, strides) of the A (A0, A1), B, D and residual views the descriptor addresses, as fdx_gemm resolves its
    default batch strides (include/fdx.h, fdx_api_tc.cu gemm_launch_desc)."""
    b1, b2 = d.b1, d.b2
    batched = b1 * b2 > 1
    if d.mode == GEMM_MNMN:
        s1 = d.a_s[0] or d.a_ld * d.K
        A = ((b2, b1, d.K, d.M), (d.a_s[1] or s1 * b1, s1, d.a_ld, 1))
        s1 = d.b_s[0] or d.b_ld * d.K
        B = ((b2, b1, d.K, d.N), (d.b_s[1] or s1 * b1, s1, d.b_ld, 1))
        D = ((d.M, d.N), (d.d_ld, 1)) if d.reduce_batch else ((b2, b1, d.M, d.N), (d.d_s[1], d.d_s[0], d.d_ld, 1))
        return dict(A=A, B=B, D=D)
    s1 = d.a_s[0] or d.a_ld * d.M
    A = ((b2, b1, d.M, d.K0 or d.K), (d.a_s[1] or s1 * b1, s1, d.a_ld, 1))
    rows, cols = (d.N, d.K) if d.mode == GEMM_KK else (d.K, d.N)
    if (d.b_s[0] or d.b_s[1]) and batched:
        s1 = d.b_s[0] or d.b_ld * rows
        B = ((b2, b1, rows, cols), (d.b_s[1] or s1 * b1, s1, d.b_ld, 1))
    else:
        B = ((rows, cols), (d.b_ld, 1))
    out = dict(A=A, B=B, D=((b2, b1, d.M, d.N), (d.d_s[1], d.d_s[0], d.d_ld, 1)))
    if d.cat:
        out["A1"] = ((d.M, d.K - d.K0), (d.a1_ld, 1))
    if d.res:
        out["res"] = ((b2, b1, d.M, d.N), (d.r_s[1], d.r_s[0], d.r_ld, 1))
    return out


def assert_outside_intact(buf, view):
    """Every element of buf outside view still holds SENTINEL, bit for bit."""
    keep = torch.ones(buf.shape, dtype=torch.bool, device=dev)
    keep.as_strided(view.shape, view.stride(), view.storage_offset()).fill_(False)
    bits = torch.int16 if buf.element_size() == 2 else torch.int32
    want = torch.tensor(SENTINEL, dtype=buf.dtype).view(bits).item()
    side = buf.view(bits)[keep]
    assert bool((side == want).all()), f"{int((side != want).sum())} elements outside the output were written"


def check(kind, what, got, val, mag, dep, bf16_out, unit=1.0):
    """dense: |got - ref| within the bound of gemm_ref -> the worst |err| / bound; exact: bit for bit (bf16 outputs:
    the exact value rounded to bf16), given that every term is a multiple of `unit` and every output's sum of |terms|
    is below 2^24 units (then every partial sum is an integer number of units of at most 24 bits)."""
    if kind == "exact":
        assert R.exact_case_ok(mag / unit), f"{what}: the exact case's sums reach 2^24 units of {unit!r}"
        want = val.to(torch.bfloat16).to(F64) if bf16_out else val
        bad = ~(got.to(F64) == want)
        if bad.any():
            i = tuple(int(j) for j in torch.nonzero(bad)[0])
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from the exact "
                                 f"result; first at {i}: got {got[i].item()!r}, exact {val[i].item()!r}")
        return 0.0
    delta = dep * R.TC_ADD * mag
    bound = R.bf16_bound(val, delta) if bf16_out else R.f32_bound(val, delta)
    return R.assert_elementwise(got, val, bound, what)


def replay(d: Desc, kind: str, name: str, seed: int):
    g = torch.Generator(device=dev).manual_seed(seed)
    lay = layouts(d)
    oA, oA1, oB, oD, oBias, oRes = d.off
    bscale = 1 / math.sqrt(d.K)

    def operand(key, off, scale=1.0):
        shape, strides = lay[key]
        return strided(shape, strides, off, torch.bfloat16, lambda n: draw(n, kind, g, scale))[1]

    A = operand("A", oA)
    A1 = operand("A1", oA1) if d.cat else None
    B = operand("B", oB, bscale)
    bias = None
    if d.bias:
        bias = strided((d.N,), (1,), oBias, torch.float32, lambda n: draw(n, kind, g, dtype=torch.float32))[1]
    odt = torch.float32 if d.d_f32 else torch.bfloat16
    dshape, dstrides = lay["D"]
    assert all(s != 0 for n, s in zip(dshape, dstrides) if n > 1), f"{name}: outputs overlap"
    Dbuf, D = strided(dshape, dstrides, oD, odt, lambda n: torch.full((n,), SENTINEL, dtype=odt, device=dev))
    prior = None
    if d.atomic:
        prior = draw(D.numel(), kind, g, 16.0, torch.float32).view(D.shape)
        D.copy_(prior)
    else:
        D.fill_(math.nan)
    res = None
    if d.res:
        rshape, rstrides = lay["res"]
        if d.alias:
            res = Dbuf.as_strided(rshape, rstrides, D.storage_offset())
            res.copy_(draw(math.prod(rshape), kind, g).view(rshape))
        else:                                        # may be shared by the batch (stride 0), so filled as a buffer
            res = strided(rshape, rstrides, oRes, torch.bfloat16, lambda n: draw(n, kind, g))[1]
        res_before = res.clone()
    alpha = d.alpha
    if kind == "exact" and alpha != 1.0:
        alpha = math.copysign(2.0 ** round(math.log2(abs(alpha))), alpha)
    # exact: products are multiples of B's power of two, alpha scales them, bias, residual and prior are integers
    unit = 2.0 ** round(math.log2(bscale)) * min(1.0, abs(alpha))

    if d.cat:
        _CAT(d.mode, A, A1, B, D, d.M, d.N, d.K, d.K0, d.a_ld, d.a1_ld, d.b_ld, d.d_ld, bias=bias, res=res,
             r_ld=d.r_ld)
    else:
        _GEMM(d.mode, A, B, D, d.M, d.N, d.K, d.a_ld, d.b_ld, d.d_ld, d.b1, d.b2, a_s=d.a_s, b_s=d.b_s, d_s=d.d_s,
              alpha=alpha, bias=bias, res=res, r_ld=d.r_ld, r_s=d.r_s, atomic=d.atomic,
              reduce_batch=d.reduce_batch)
    lib = _lib.load()
    ran = lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()
    assert ran == "fdx_tc_kernel", f"{name}: ran {ran}"
    assert_outside_intact(Dbuf, D)
    if d.res and not d.alias:
        assert torch.equal(res, res_before), f"{name}: the residual was written"

    # float64 reference: a (..., M, K) @ b (..., K, N), over row chunks of at most 2^25 outputs for KK / KMN
    extra = [None if t is None else t.to(F64) for t in (bias, res_before if d.res else None, prior)]
    if d.mode == GEMM_MNMN:
        a, b = A.to(F64).transpose(-1, -2), B.to(F64)
        if d.reduce_batch:
            a, b = a.permute(2, 0, 1, 3).reshape(d.M, -1), b.reshape(-1, d.N)
        chunks = [(slice(None), a, extra)]
    else:
        b = B.to(F64).transpose(-1, -2) if d.mode == GEMM_KK else B.to(F64)
        step = max(1, 2 ** 25 // (d.b1 * d.b2 * d.N))
        chunks = []
        for m0 in range(0, d.M, step):
            rows = slice(m0, m0 + step)
            chunks.append((rows, A[..., rows, :], [t if t is None or t.dim() == 1 else t[..., rows, :]
                                                   for t in extra]))
    worst = 0.0
    for rows, a, ex in chunks:
        if d.mode != GEMM_MNMN:
            a = a.to(F64)
            if d.cat:
                a = torch.cat([a, A1[rows].to(F64).expand(d.b2, d.b1, -1, -1)], -1)
        val, mag = R._plus(alpha * (a @ b), abs(alpha) * (a.abs() @ b.abs()), *ex)
        del a
        worst = max(worst, check(kind, f"{kind} {name} rows {rows.start or 0}..", D[..., rows, :], val, mag,
                                 depth(d), not d.d_f32, unit))
        del val, mag
    if kind == "dense":
        print(f"WORST {kind} {name} {worst:.3f}")

    if d.cat:
        # bit for bit gemm on the materialised concatenation
        want = torch.empty((d.M, d.N), dtype=odt, device=dev)
        _GEMM(d.mode, torch.cat([A[0, 0], A1], 1), B, want, d.M, d.N, d.K, d.K, d.b_ld, d.N, bias=bias,
              res=res_before[0, 0].contiguous() if d.res else None, r_ld=d.N if d.res else 0)
        assert torch.equal(D[0, 0].view(torch.int16 if odt == torch.bfloat16 else torch.int32),
                           want.view(torch.int16 if odt == torch.bfloat16 else torch.int32)), \
            f"{name}: gemm_cat differs from gemm on the concatenation"


def replay_all(cases: dict, label: str):
    """Replay {Desc: site} in both kinds; every failure is collected and reported together."""
    t0 = time.perf_counter()
    bad = []
    for i, (d, site) in enumerate(sorted(cases.items(), key=lambda kv: kv[1])):
        name = case_name(d, site)
        for kind in KINDS:
            try:
                replay(d, kind, name, seed=1000 + i)
            except AssertionError as e:
                bad.append(str(e).splitlines()[0])
        torch.cuda.empty_cache()
    print(f"REPLAYED {label}: {len(cases)} distinct descriptors x {len(KINDS)} kinds in "
          f"{time.perf_counter() - t0:.1f} s")
    assert not bad, f"{len(bad)} failing replays:\n" + "\n".join(bad[:20])


# ----------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("family", FAMILIES)
def test_replay_family(family):
    t0 = time.perf_counter()
    cases = recorded(family)
    print(f"RECORDED {family}: {len(cases)} distinct descriptors in {time.perf_counter() - t0:.1f} s")
    replay_all(cases, family)


def test_replay_fixed():
    replay_all(FIXED, "fixed")


def test_recorded_classes_cover_the_models():
    """The recorded descriptors (all families) contain every class of GEMM launch the models are known to issue, so
    that a refactor which silently stops exercising one fails here instead of shrinking the replays."""
    t0 = time.perf_counter()
    table = {}
    for fam in FAMILIES:
        for d in recorded(fam):
            for c in classes(d):
                table.setdefault(c, {}).setdefault(fam, 0)
                table[c][fam] += 1
    fixed = set().union(*(classes(d) for d in FIXED))
    print(f"\n{'class':<26}" + "".join(f"{f[:12]:>13}" for f in FAMILIES))
    for c in sorted(table.keys() | fixed):
        print(f"{c:<26}" + "".join(f"{table.get(c, {}).get(f, 0):>13}" for f in FAMILIES)
              + ("   (+ fixed)" if c in fixed else ""))
    print(f"total distinct descriptors: {sum(len(recorded(f)) for f in FAMILIES)} "
          f"({time.perf_counter() - t0:.1f} s)")
    missing = MODEL_CLASSES - table.keys()
    assert not missing, f"the models no longer issue: {sorted(missing)}"
    assert "alpha != 1" in fixed
