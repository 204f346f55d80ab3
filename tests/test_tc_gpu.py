"""Parity of the wgmma tap-GEMM engine through the C-ABI (fdx_conv3x3_{fwd,dgrad,wgrad}, fdx_gemm)
against fp32 references on the same bf16-rounded inputs.  Tolerance: relative L2 error <= 5e-3 for bf16
outputs (one bf16 rounding of an f32 accumulator: 2^-9 ~ 2e-3), <= 1e-4 for f32 outputs."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import gpu_probe_tc as T  # noqa: E402

pytestmark = pytest.mark.gpu

BF16_TOL, F32_TOL = 5e-3, 1e-4

CASES = [
    ("gemm_kk", lambda: T.t_gemm_kk(256, 128, 128), F32_TOL),
    ("gemm_kk_ragged", lambda: T.t_gemm_kk(1000, 256, 320), F32_TOL),
    ("gemm_kmn", lambda: T.t_gemm_kmn(512, 512, 256), BF16_TOL),
    ("gemm_kmn_small", lambda: T.t_gemm_kmn(37, 64, 64, False), BF16_TOL),
    ("gemm_mnmn_splitk", lambda: T.t_gemm_mnmn(256, 512, 4096), F32_TOL),
    ("conv_fwd_64", lambda: T.t_conv_fwd(2, 16, 16, 64, 64), BF16_TOL),
    ("conv_fwd_fused_epilogue", lambda: T.t_conv_fwd(2, 32, 32, 128, 256, extras=True), BF16_TOL),
    ("conv_fwd_multi_image_tile", lambda: T.t_conv_fwd(4, 8, 8, 256, 512), BF16_TOL),
    ("conv_fwd_tiny_2x2", lambda: T.t_conv_fwd(3, 2, 2, 256, 256), BF16_TOL),
    ("conv_fwd_concat_k", lambda: T.t_conv_fwd(1, 64, 64, 320, 64), BF16_TOL),
    ("conv_fwd_slots", lambda: T.t_conv_fwd_slot(2, 16, 16, 128, 64), BF16_TOL),
    ("conv_fwd_stride2", lambda: T.t_conv_fwd(2, 32, 32, 64, 128, stride=2), BF16_TOL),
    ("conv_dgrad", lambda: T.t_conv_dgrad(2, 16, 16, 64, 128), BF16_TOL),
    ("conv_dgrad_accumulate", lambda: T.t_conv_dgrad(2, 32, 32, 192, 64, accumulate=True), BF16_TOL),
    ("conv_dgrad_stride2", lambda: T.t_conv_dgrad(2, 32, 32, 64, 128, stride=2), BF16_TOL),
    ("conv_wgrad", lambda: T.t_conv_wgrad(2, 16, 16, 64, 64), F32_TOL),
    ("conv_wgrad_wide", lambda: T.t_conv_wgrad(4, 32, 32, 192, 128), F32_TOL),
    ("conv_wgrad_stride2", lambda: T.t_conv_wgrad(2, 32, 32, 64, 128, stride=2), F32_TOL),
    ("conv_wgrad_8x8_tile", lambda: T.t_conv_wgrad(6, 8, 8, 256, 128), F32_TOL),
    ("conv_wgrad_many_splits", lambda: T.t_conv_wgrad(16, 64, 64, 64, 64), F32_TOL),
    ("conv_wgrad_4x4_generic", lambda: T.t_conv_wgrad(8, 4, 4, 128, 64), F32_TOL),
    ("attn_qk_d64", lambda: T.t_attn_qk(2, 256, 8, 64), BF16_TOL),
    ("attn_qk_d32", lambda: T.t_attn_qk(2, 128, 8, 32), BF16_TOL),
    ("attn_pv_d64", lambda: T.t_attn_pv(2, 256, 8, 64), BF16_TOL),
    ("attn_pv_d32", lambda: T.t_attn_pv(2, 128, 8, 32), BF16_TOL),
    ("attn_dv_d64", lambda: T.t_attn_dv(2, 256, 8, 64), BF16_TOL),
    ("attn_dv_d32_L64", lambda: T.t_attn_dv(3, 64, 8, 32), BF16_TOL),
]


@pytest.mark.parametrize("name,make,tol", CASES, ids=[c[0] for c in CASES])
def test_tc_engine_parity(name, make, tol):
    torch.manual_seed(0)
    rel, _ = make()()
    torch.cuda.synchronize()
    assert rel < tol, f"{name}: rel err {rel}"


def test_conv_full_size_properties():
    """BASELINE-size checks (64x64, B=256, C=64) through size-independent properties:
    linearity of the forward conv and the adjoint identities <conv(x),dy> = <x,dgrad(dy)> = <w,wgrad(x,dy)>."""
    from flaxdiff_b200 import ops
    dev = torch.device("cuda")
    torch.manual_seed(1)
    B, H, C = 256, 64, 64
    x = torch.randn(B, H, H, C, device=dev).bfloat16()
    y = torch.randn(B, H, H, C, device=dev).bfloat16()
    w = (torch.randn(3, 3, C, C, device=dev) / 24).bfloat16()
    cx, cy = ops.conv3x3_fwd(x, w).float(), ops.conv3x3_fwd(y, w).float()
    z = (x.float() + y.float()).bfloat16()
    cz = ops.conv3x3_fwd(z, w).float()
    # x + y is re-rounded to bf16, so compare against conv of the rounded sum's parts only loosely
    assert ((cz - (cx + cy)).norm() / (cx + cy).norm()).item() < 1e-2
    dy = torch.randn(B, H, H, C, device=dev).bfloat16()
    dx = torch.empty_like(x)
    ops.conv3x3_dgrad(dy, w, dx)
    dw = torch.zeros(3, 3, C, C, device=dev)
    ops.conv3x3_wgrad(x, dy, dw)
    a = (cx.double() * dy.double()).sum().item()
    b = (x.double() * dx.double()).sum().item()
    c = (w.double() * dw.double()).sum().item()
    assert abs(a - b) / abs(a) < 5e-3 and abs(a - c) / abs(a) < 5e-3, (a, b, c)
