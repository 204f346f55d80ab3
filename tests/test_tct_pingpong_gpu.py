"""The transposed engine's tile schedule (fdx_tct_kernel): the two consumer warpgroups take alternate tiles of a
CTA's tile sequence, so the edge cases are one tile in all, an odd number of tiles per CTA, fewer tiles than SMs,
and layers of 128 or 384 columns that run as several 64-column blocks.  Each launch is checked to have run
fdx_tct_kernel, and its result against fp32 torch."""
import ctypes

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
    lib.fdx_kernel_kind_name.restype = ctypes.c_char_p
    return lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()


def conv_ref(x, w, b=None):
    return Fnn.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(3, 2, 0, 1), b,
                      padding=w.shape[0] // 2).permute(0, 2, 3, 1)


def dgrad_ref(dy, w):
    n, h, wd, _ = dy.shape
    x = torch.zeros(n, h, wd, w.shape[2], device=dev, requires_grad=True)
    conv_ref(x, w).backward(dy.float())
    return x.grad


def sms():
    return torch.cuda.get_device_properties(dev).multi_processor_count


# (B, H, W) by the number of 16 x 16 pixel tiles of a 64-column layer
GEOMETRY = {
    "one_tile": lambda: (1, 16, 16),
    "fewer_tiles_than_sms": lambda: (2, 32, 32),
    "three_tiles_per_cta": lambda: (1, 16, 16 * 3 * sms()),
    "one_cta_with_an_odd_count": lambda: (1, 16, 16 * (2 * sms() + 1)),
}


@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_forward_residual_column_sums(geom):
    torch.manual_seed(5)
    B, H, W = GEOMETRY[geom]()
    cin, cout = 128, 64
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    res = torch.randn(B, H, W, cout, device=dev).bfloat16()
    cs = ops.ColStats(B, cout, dev)
    y = ops.conv3x3_fwd(x, w, bias, res=res, colstats=(cs, 0))
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(y, conv_ref(x, w, bias) + res.float()) < 5e-3
    assert rel(ops.groupnorm_stats_from_cols(cs, 8, 0, cout), ops.groupnorm_stats(y, 8)) < 1e-5


@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_dgrad_accumulate_and_fused_groupnorm_backward(geom):
    torch.manual_seed(6)
    B, H, W = GEOMETRY[geom]()
    cin, cout = 64, 64
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv3x3_dgrad(dy, w, dx, accumulate=True)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    want = dgrad_ref(dy, w)
    assert rel(dx, prior + want) < 5e-3
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = torch.empty(B, H, W, cin, device=dev, dtype=torch.bfloat16)
    ws = ops.conv3x3_dgrad_gn(dy, w, dz, x, ab)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    z = x.float() * ab[:, 0].view(B, 1, 1, cin) + ab[:, 1].view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    assert rel(dz, want * s * (1 + z * (1 - s))) < 1e-2
    sums = ws.sum(0)
    assert rel(sums[:, 0], dz.float().sum((1, 2))) < 1e-4
    assert rel(sums[:, 1], (dz.float() * x.float()).sum((1, 2))) < 1e-4


@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 128)])
def test_forward_128_columns_as_two_blocks(cin, cout):
    torch.manual_seed(7)
    B, H, W = 2, 32, 48
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    rowvec = torch.randn(B, cout, device=dev) * 0.3
    res = torch.randn(B, H, W, cout, device=dev).bfloat16()
    cs = ops.ColStats(B, cout, dev)
    y = ops.conv3x3_fwd(x, w, bias, rowvec=rowvec, res=res, colstats=(cs, 0))
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(y, conv_ref(x, w, bias) + rowvec.view(B, 1, 1, cout) + res.float()) < 5e-3
    assert rel(ops.groupnorm_stats_from_cols(cs, 8, 0, cout), ops.groupnorm_stats(y, 8)) < 1e-5


@pytest.mark.parametrize("cin,cout", [(128, 128), (384, 64)])
def test_dgrad_several_column_blocks(cin, cout):
    torch.manual_seed(8)
    B, H, W = 2, 32, 32
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv3x3_dgrad(dy, w, dx, accumulate=True)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(dx, prior + dgrad_ref(dy, w)) < 5e-3


def test_conv1x1_dgrad_320_columns():
    torch.manual_seed(9)
    B, H, W, cin, cout = 2, 32, 32, 320, 64
    w = (torch.randn(cin, cout, device=dev) / cin ** 0.5).bfloat16()
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv1x1_dgrad(dy, w, dx, accumulate=True)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert rel(dx, prior + dgrad_ref(dy, w.view(1, 1, cin, cout))) < 5e-3
