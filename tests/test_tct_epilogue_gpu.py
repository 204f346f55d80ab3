"""The transposed engine's epilogue (fdx_tct_kernel) at shapes the other GPU tests leave out: column sums into a
channel slot of a wider buffer, the fused GroupNorm backward at 320 and 192 columns, in-place accumulation where
the last tile has no second pixel half (H % 32 == 16 at 64 columns), and 1x1 convolutions through the engine.
Each launch is checked to have run fdx_tct_kernel, and its result against fp32 torch."""

import pytest
import torch
import torch.nn.functional as Fnn

from flaxdiff_b200 import _lib, ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def last_kernel():
    lib = _lib.load()
    return lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()


def conv_ref(x, w, b=None):
    return Fnn.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(3, 2, 0, 1), b,
                      padding=w.shape[0] // 2).permute(0, 2, 3, 1)


def dgrad_ref(dy, w):
    n, h, wd, _ = dy.shape
    x = torch.zeros(n, h, wd, w.shape[2], device=dev, requires_grad=True)
    conv_ref(x, w).backward(dy.float())
    return x.grad


def test_forward_residual_column_sums_into_channel_slot():
    torch.manual_seed(1)
    B, H, W, cin, cout, coff = 2, 64, 64, 320, 64, 64
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    res = torch.randn(B, H, W, cout, device=dev).bfloat16()
    buf = torch.zeros(B, H, W, 320, device=dev, dtype=torch.bfloat16)
    y = buf[..., coff:coff + cout]
    cs = ops.ColStats(B, 320, dev)
    ops.conv3x3_fwd(x, w, bias, res=res, out=y, colstats=(cs, coff))
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(y, conv_ref(x, w, bias) + res.float()) < 5e-3
    assert torch.count_nonzero(buf[..., :coff]) == 0 and torch.count_nonzero(buf[..., coff + cout:]) == 0
    assert rel(ops.groupnorm_stats_from_cols(cs, 8, coff, cout), ops.groupnorm_stats(y, 8)) < 1e-5


@pytest.mark.parametrize("H,cin,cout", [(64, 320, 64), (32, 192, 128)])
def test_dgrad_fused_groupnorm_backward(H, cin, cout):
    torch.manual_seed(2)
    B = 2
    dy = torch.randn(B, H, H, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    x = torch.randn(B, H, H, cin, device=dev).bfloat16()
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = torch.empty(B, H, H, cin, device=dev, dtype=torch.bfloat16)
    ws = ops.conv3x3_dgrad_gn(dy, w, dz, x, ab)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    z = x.float() * ab[:, 0].view(B, 1, 1, cin) + ab[:, 1].view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    assert rel(dz, dgrad_ref(dy, w) * s * (1 + z * (1 - s))) < 1e-2
    sums = ws.sum(0)                                   # [B][2][cin]: sum dz, sum dz * x per (image, channel)
    dzf = dz.float()
    assert rel(sums[:, 0], dzf.sum((1, 2))) < 1e-4
    assert rel(sums[:, 1], (dzf * x.float()).sum((1, 2))) < 1e-4


@pytest.mark.parametrize("H", [16, 48])
def test_dgrad_accumulate_in_place_without_second_half(H):
    torch.manual_seed(3)
    B, W, cin, cout = 2, 32, 64, 128
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv3x3_dgrad(dy, w, dx, accumulate=True)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(dx, prior + dgrad_ref(dy, w)) < 5e-3


def test_conv1x1_forward_and_dgrad_through_the_engine():
    torch.manual_seed(4)
    B, H, W, cin, cout = 2, 32, 32, 128, 64
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(cin, cout, device=dev) / cin ** 0.5).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    res = torch.randn(B, H, W, cout, device=dev).bfloat16()
    y = ops.conv1x1_fwd(x, w, bias, res=res)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    w4 = w.view(1, 1, cin, cout)
    assert rel(y, conv_ref(x, w4, bias) + res.float()) < 5e-3
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv1x1_dgrad(dy, w, dx, accumulate=True)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(dx, prior + dgrad_ref(dy, w4)) < 5e-3
