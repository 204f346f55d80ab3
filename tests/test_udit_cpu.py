"""SimpleUDiT host logic (no GPU): parameter names and shapes, the constructor's refusals, fdx_gemm_cat's refusals
through the C ABI, the oracle against a closed form and gradcheck, and a ptxas guard for the two-source GEMM kernels.

Parameter names: SimpleUDiT.setup (simple_vit.py:274-374) names patch_embed, hilbert_projection (only under
use_hilbert), time_embed, text_proj, down_block_{i}, mid_block, up_dense_{i}, up_block_{i}, final_norm and final_proj.
Modules built in setup() get parameters only when called: patch_embed has none under use_hilbert, text_proj none
without a text context.  No SimpleUDiT checkpoint exists in the reference tree, so the names are derived from flax's
naming rules, not pinned against a file flax wrote."""
import json
import os
import subprocess
import sys

import pytest
import torch

from flaxdiff_b200._lib import FdxError
from flaxdiff_b200.models.ssm_dit import hilbert_indices
from flaxdiff_b200.models.udit import SimpleUDiT
from oracle import udit_ref
from oracle.dit_ref import layernorm
from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _names(F, h, p, E, layers, ctx, out=3, sigma=False, hilbert=False):
    d = F // h
    n = p * p * out * (2 if sigma else 1)
    want = {"time_embed/layers_1/DenseGeneral_0/kernel": (F, E), "time_embed/layers_1/DenseGeneral_0/bias": (E,),
            "time_embed/layers_1/DenseGeneral_1/kernel": (E, E), "time_embed/layers_1/DenseGeneral_1/bias": (E,),
            "time_embed/layers_2/kernel": (E, F), "time_embed/layers_2/bias": (F,),
            "final_norm/scale": (F,), "final_norm/bias": (F,), "final_proj/kernel": (F, n), "final_proj/bias": (n,)}
    if ctx:
        want.update({"text_proj/kernel": (ctx, F), "text_proj/bias": (F,)})
    if hilbert:
        want.update({"hilbert_projection/kernel": (p * p * 3, F), "hilbert_projection/bias": (F,)})
    else:
        want.update({"patch_embed/Conv_0/kernel": (p, p, 3, F), "patch_embed/Conv_0/bias": (F,)})
    half = layers // 2
    blocks = [f"down_block_{i}" for i in range(half)] + ["mid_block"] + [f"up_block_{i}" for i in range(half)]
    for b in blocks:
        want[f"{b}/ada_params_module/ada_proj/kernel"] = (F, 6 * F)
        want[f"{b}/ada_params_module/ada_proj/bias"] = (6 * F,)
        for m in ("to_q", "to_k", "to_v"):
            want[f"{b}/attention/{m}/kernel"] = (F, h, d)
            want[f"{b}/attention/{m}/bias"] = (h, d)
        want[f"{b}/attention/to_out_0/kernel"] = (h, d, F)
        want[f"{b}/attention/to_out_0/bias"] = (F,)
        want[f"{b}/mlp/layers_0/kernel"] = (F, E)
        want[f"{b}/mlp/layers_0/bias"] = (E,)
        want[f"{b}/mlp/layers_2/kernel"] = (E, F)
        want[f"{b}/mlp/layers_2/bias"] = (F,)
    for i in range(half):
        want[f"up_dense_{i}/kernel"] = (2 * F, F)
        want[f"up_dense_{i}/bias"] = (F,)
    return want


@pytest.mark.parametrize("kw,F,h,p,E,layers,ctx,sigma,hilbert", [
    (dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12, context_dim=768), 768, 12, 2, 3072, 12, 768,
     False, False),                                                   # the reference's simple_udit config, 3-D text
    (dict(patch_size=4, emb_features=64, num_layers=2, num_heads=2), 64, 2, 4, 256, 2, None, False, False),
    (dict(patch_size=2, emb_features=128, num_layers=4, num_heads=4, context_dim=32, use_hilbert=True), 128, 4, 2,
     512, 4, 32, False, True),
    (dict(patch_size=2, emb_features=128, num_layers=2, num_heads=4, learn_sigma=True), 128, 4, 2, 512, 2, None,
     True, False),
])
def test_parameter_names_and_shapes(kw, F, h, p, E, layers, ctx, sigma, hilbert):
    m = SimpleUDiT(**kw)
    got = {k: s for k, (_, s) in m.layout().table.items()}
    assert got == _names(F, h, p, E, layers, ctx, sigma=sigma, hilbert=hilbert)
    # the layout follows the forward order: up_dense_{i} sits between up_block_{i-1} and up_block_{i}
    order = list(m.layout().table)
    for i in range(layers // 2):
        assert order.index(f"up_dense_{i}/bias") + 1 == order.index(f"up_block_{i}/ada_params_module/ada_proj/kernel")


def test_init_and_config_round_trip():
    m = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=16)
    fp = m.init(0, device="cpu")
    assert fp.named["up_dense_0/kernel"].std().item() == pytest.approx((1 / 128) ** 0.5, rel=0.2)   # lecun, fan-in 2F
    assert fp.named["up_dense_0/bias"].abs().max().item() == 0
    assert fp.named["final_proj/kernel"].abs().max().item() == 0
    assert fp.named["mid_block/ada_params_module/ada_proj/kernel"].abs().max().item() == 0
    m2 = SimpleUDiT(**m.config())
    assert m2.layout().table == m.layout().table


@pytest.mark.parametrize("kw,msg", [
    (dict(num_layers=3), "num_layers=3 must be even"),
    (dict(use_flash_attention=True), "use_flash_attention"),
    (dict(dtype=torch.float32), "dtype"),
    (dict(emb_features=768, num_heads=7), "not a multiple of num_heads"),
    (dict(emb_features=192, num_heads=64), "head width 3 is odd"),
    (dict(emb_features=1024, num_heads=2), "head width 512 > 256"),
    (dict(emb_features=96, num_heads=2), "multiple of 64, at most 1536"),
    (dict(emb_features=1600, num_heads=25), "multiple of 64, at most 1536"),
])
def test_refusals_name_the_class(kw, msg):
    args = dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12)
    args.update(kw)
    with pytest.raises(FdxError, match="SimpleUDiT") as e:
        SimpleUDiT(**args)
    assert msg in str(e.value)


def test_ignored_arguments_are_accepted():
    SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, dropout_rate=0.1, norm_groups=8,
               activation=torch.nn.functional.silu, force_fp32_for_softmax=False)


_CAT_CHILD = r"""
import ctypes, json, sys
from flaxdiff_b200 import _lib
lib = _lib.load()
base = 1 << 40                                   # fake, 16-byte aligned addresses: nothing is ever dereferenced
M, N, K, K0 = 1024, 768, 1536, 768


def desc():
    g = _lib.fdx_gemm_desc()
    g.mode, g.M, g.N, g.K = _lib.GEMM_KMN, M, N, K
    g.A, g.a_ld, g.B, g.b_ld, g.D, g.d_ld = base, K0, base + (1 << 30), N, base + (2 << 30), N
    g.alpha = 1.0
    return g


out = []
for field, value, a1, a1_ld, k0 in json.loads(sys.argv[1]):
    g = desc()
    if field:
        setattr(g, field, (base + value) if field == "A" else value)
    a1 = None if a1 is None else base + (3 << 30) + a1
    st = lib.fdx_gemm_cat(ctypes.byref(g), a1, a1_ld, k0, None)
    out.append([st, lib.fdx_last_error().decode()])
print(json.dumps(out))
"""


def test_gemm_cat_refusals_through_the_c_abi():
    """fdx_gemm_cat refuses, with a message naming the entry point, every launch it does not serve: batch > 1, the
    weight-gradient mode, K0 off the 64-wide k block or outside (0, K), null or misaligned A0 / A1 and row strides off
    16 bytes.  The calls run in a child process that sees no GPU, on fake addresses: a check that let one through
    could launch nothing."""
    cases = [
        ("batch1", 2, 0, 768, 768, "gemm_cat: batch 2 x 0"),
        ("batch2", 4, 0, 768, 768, "gemm_cat: batch 0 x 4"),
        ("mode", 2, 0, 768, 768, "gemm_cat: mode 2"),
        (None, 0, 0, 768, 96, "gemm_cat: K0=96 must be a multiple of 64"),
        (None, 0, 0, 768, 0, "gemm_cat: K0=0 must be"),
        (None, 0, 0, 768, -64, "gemm_cat: K0=-64 must be"),
        (None, 0, 0, 768, 1536, "gemm_cat: K0=1536 must be"),
        (None, 0, 0, 768, 2048, "gemm_cat: K0=2048 must be"),
        (None, 0, None, 768, 768, "gemm_cat: null pointer"),
        (None, 0, 8, 768, 768, "gemm_cat: A0 and A1 must be 16-byte aligned"),
        ("A", 8, 0, 768, 768, "gemm_cat: A0 and A1 must be 16-byte aligned"),
        ("a_ld", 772, 0, 768, 768, "gemm_cat: a_ld=772 must be"),
        ("a_ld", 704, 0, 768, 768, "gemm_cat: a_ld=704 must be"),
        (None, 0, 0, 772, 768, "gemm_cat: a1_ld=772 must be"),
        (None, 0, 0, 640, 768, "gemm_cat: a1_ld=640 must be"),
    ]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _CAT_CHILD, json.dumps([c[:5] for c in cases])], capture_output=True,
                       text=True, env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for c, (status, msg) in zip(cases, res):
        assert status == -1 and msg.startswith(c[5]), (c, status, msg)


# ------------------------------------------------------------------------------------------------------ oracle
def _params(m, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    fp = m.init(seed, device="cpu")
    return {k: (v.to(dtype) + 0.2 * torch.randn(v.shape, generator=g, dtype=dtype)) for k, v in fp.named.items()}


def test_oracle_closed_form_checks_the_skip_pairing():
    """With the attention gate zero, the MLP gate one and the MLP's first layer zero, every DiT block adds its MLP's
    output bias: block_n(x) = x + c_n.  The skips are then distinct, and the output is a hand-computable chain of
    up_dense layers over the embedded tokens: up layer i reads [x, skip of down_block_{half-1-i}]."""
    m = SimpleUDiT(patch_size=2, emb_features=64, num_layers=6, num_heads=2)
    P = _params(m, 1)
    F, half = 64, 3
    blocks = [f"down_block_{i}" for i in range(half)] + ["mid_block"] + [f"up_block_{i}" for i in range(half)]
    c = {}
    for b in blocks:
        ada_b = torch.zeros(6 * F, dtype=torch.float64)
        ada_b[2 * F:3 * F] = 1.0                                  # gate_mlp
        P[f"{b}/ada_params_module/ada_proj/kernel"].zero_()
        P[f"{b}/ada_params_module/ada_proj/bias"].copy_(ada_b)
        P[f"{b}/mlp/layers_0/kernel"].zero_()
        P[f"{b}/mlp/layers_0/bias"].zero_()                       # gelu(0) = 0: the MLP outputs its layers_2 bias
        c[b] = P[f"{b}/mlp/layers_2/bias"]
    B, H, W, p = 2, 8, 8, 2
    x = torch.randn(B, H, W, 3, dtype=torch.float64)
    t = torch.rand(B, dtype=torch.float64)
    freqs = m._fourier_freqs("cpu").double()
    got = udit_ref.simple_udit_forward(P, x, t, freqs, patch_size=p, num_layers=6, num_heads=2)

    patches = x.reshape(B, H // p, p, W // p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(B, -1, p * p * 3)
    tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(-1, F) + P["patch_embed/Conv_0/bias"]
    skips = []
    for i in range(half):
        tok = tok + c[f"down_block_{i}"]
        skips.append(tok)
    tok = tok + c["mid_block"]
    for i in range(half):
        k = P[f"up_dense_{i}/kernel"]
        tok = tok @ k[:F] + skips[half - 1 - i] @ k[F:] + P[f"up_dense_{i}/bias"] + c[f"up_block_{i}"]
    y = layernorm(tok, 1e-5, P["final_norm/scale"], P["final_norm/bias"]) @ P["final_proj/kernel"] + \
        P["final_proj/bias"]
    want = y.reshape(B, H // p, W // p, p, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, 3)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # the pairing matters: reversing the skips changes the result
    assert not torch.allclose(skips[0] @ P["up_dense_0/kernel"][F:], skips[2] @ P["up_dense_0/kernel"][F:])


def test_oracle_text_pooling_and_hilbert_order():
    """2-D text enters unpooled, 3-D text as the token mean of text_proj; under Hilbert the output returns to raster
    order (a permutation-equivariant model with no position signal but RoPE would otherwise scramble it)."""
    m = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=8)
    P = _params(m, 2)
    x = torch.randn(1, 8, 8, 3, dtype=torch.float64)
    t = torch.rand(1, dtype=torch.float64)
    freqs = m._fourier_freqs("cpu").double()
    ctx = torch.randn(1, 5, 8, dtype=torch.float64)
    kw = dict(patch_size=2, num_layers=2, num_heads=2)
    a = udit_ref.simple_udit_forward(P, x, t, freqs, textcontext=ctx, **kw)
    b = udit_ref.simple_udit_forward(P, x, t, freqs, textcontext=ctx.mean(1), **kw)
    torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
    mh = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, use_hilbert=True)
    Ph = _params(mh, 3)
    order = hilbert_indices(4, 4)
    y = udit_ref.simple_udit_forward(Ph, x, t, freqs, order=order, **kw)
    assert y.shape == (1, 8, 8, 3) and torch.isfinite(y).all()


def test_oracle_gradcheck():
    m = SimpleUDiT(patch_size=2, emb_features=64, num_layers=2, num_heads=2, context_dim=4, learn_sigma=True)
    P = _params(m, 4)
    x = torch.randn(1, 4, 4, 3, dtype=torch.float64)
    t = torch.rand(1, dtype=torch.float64)
    ctx = torch.randn(1, 3, 4, dtype=torch.float64)
    freqs = m._fourier_freqs("cpu").double()
    names = ["up_dense_0/kernel", "down_block_0/ada_params_module/ada_proj/kernel", "final_proj/kernel",
             "text_proj/kernel", "mid_block/mlp/layers_0/bias"]
    leaves = [P[n][:4, :4].clone().requires_grad_(True) if P[n].dim() == 2 else P[n][:4].clone().requires_grad_(True)
              for n in names]

    def f(*vals):
        Q = dict(P)
        for n, v in zip(names, vals):
            w = P[n].clone()
            if w.dim() == 2:
                w[:4, :4] = v
            else:
                w[:4] = v
            Q[n] = w
        return udit_ref.simple_udit_forward(Q, x, t, freqs, patch_size=2, num_layers=2, num_heads=2,
                                            textcontext=ctx)
    assert torch.autograd.gradcheck(f, leaves, eps=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------------ ptxas
@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_two_source_gemm_kernels_have_no_spills_and_no_frames():
    """The six two-source instantiations (TC_KK / TC_KMN x three column tiles) keep their accumulators in registers
    and their wgmma unserialised, as fdx_tc.cu's are held to in test_ptxas_cpu.py."""
    frames, notes = _report("fdx_tc_cat.cu")
    cat = {k: v for k, v in frames.items() if "fdx_tc_kernel" in k and "CUtensorMap_stEE" in k}
    assert len(cat) == 6, sorted(frames)
    assert all(v == (0, 0, 0) for v in cat.values()), cat
    assert not any("fdx_tc_kernel" in k for k in notes), notes
