"""The transposed engine's halo launches at K = 64 (fdx_tct_kernel with resident weights): each CTA loads the nine
weight tiles of its 64-column block once and keeps that column block for all its tiles, so the grid is a whole
number of column-block groups (where that would idle SMs, the launch stays on the plain halo path).  The edge
cases are one tile, fewer tiles than SMs, an odd tile count on one CTA, a pixel-block count that leaves the
last group short, and column-block counts that do not divide the SM count (320 and 448 columns on a 132-SM
part).  Outputs start as NaN, so a tile that is never written fails; every
launch is checked to have run fdx_tct_kernel, and its result against fp32 torch."""

import pytest
import torch
import torch.nn.functional as Fnn

from flaxdiff_b200 import _lib, ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


def rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def last_kernel():
    lib = _lib.load()
    return lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()


def conv_ref(x, w, b=None):
    return Fnn.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(3, 2, 0, 1), b,
                      padding=1).permute(0, 2, 3, 1)


def dgrad_ref(dy, w):
    n, h, wd, _ = dy.shape
    x = torch.zeros(n, h, wd, w.shape[2], device=dev, requires_grad=True)
    conv_ref(x, w).backward(dy.float())
    return x.grad


def nan_like(shape):
    return torch.full(shape, float("nan"), device=dev, dtype=torch.bfloat16)


def sms():
    return torch.cuda.get_device_properties(dev).multi_processor_count


def groups(cblks):
    """CTA groups of the launch: each group of cblks CTAs walks the same pixel blocks."""
    return max(sms() // cblks, 1)


# (B, H, W) by the number of 16 x 16 pixel blocks, for a layer of cblks 64-column blocks
GEOMETRY = {
    "one_tile": lambda c: (1, 16, 16),
    "fewer_tiles_than_sms": lambda c: (2, 32, 32),
    "odd_count_on_one_cta": lambda c: (1, 16, 16 * (2 * groups(c) + 1)),
    "last_group_short": lambda c: (1, 16, 16 * (2 * groups(c) + max(groups(c) // 2, 1))),
    "several_images": lambda c: (3, 48, 80),
}
C2_SHAPES = {"64x64": (256, 64, 64), "32x32": (256, 32, 32)}


def run_forward(B, H, W, cout):
    cin = 64
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    rowvec = torch.randn(B, cout, device=dev) * 0.3
    res = torch.randn(B, H, W, cout, device=dev).bfloat16()
    cs = ops.ColStats(B, cout, dev)
    y = ops.conv3x3_fwd(x, w, bias, rowvec=rowvec, res=res, out=nan_like((B, H, W, cout)), colstats=(cs, 0))
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert torch.isfinite(y.float()).all()
    assert rel(y, conv_ref(x, w, bias) + rowvec.view(B, 1, 1, cout) + res.float()) < 5e-3
    assert rel(ops.groupnorm_stats_from_cols(cs, 8, 0, cout), ops.groupnorm_stats(y, 8)) < 1e-5


def run_dgrad(B, H, W, cin, accumulate):
    cout = 64
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cout ** 0.5)).bfloat16()
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16() if accumulate else nan_like((B, H, W, cin))
    prior = dx.float().clone() if accumulate else 0.0
    ops.conv3x3_dgrad(dy, w, dx, accumulate=accumulate)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert torch.isfinite(dx.float()).all()
    assert rel(dx, prior + dgrad_ref(dy, w)) < 5e-3


def run_dgrad_gn(B, H, W, cin):
    cout = 64
    dy = torch.randn(B, H, W, cout, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cout ** 0.5)).bfloat16()
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = nan_like((B, H, W, cin))
    ws = ops.conv3x3_dgrad_gn(dy, w, dz, x, ab)
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert torch.isfinite(dz.float()).all()
    z = x.float() * ab[:, 0].view(B, 1, 1, cin) + ab[:, 1].view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    assert rel(dz, dgrad_ref(dy, w) * s * (1 + z * (1 - s))) < 1e-2
    sums = ws.sum(0)
    assert rel(sums[:, 0], dz.float().sum((1, 2))) < 1e-4
    assert rel(sums[:, 1], (dz.float() * x.float()).sum((1, 2))) < 1e-4


@pytest.mark.parametrize("cout", [64, 128])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_forward_bias_row_residual_column_sums(geom, cout):
    torch.manual_seed(11)
    run_forward(*GEOMETRY[geom](cout // 64), cout)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("cin", [64, 128, 192, 320, 384, 448])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_dgrad(geom, cin, accumulate):
    torch.manual_seed(12)
    run_dgrad(*GEOMETRY[geom](cin // 64), cin, accumulate)


@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_dgrad_fused_groupnorm_backward_320_columns(geom):
    torch.manual_seed(13)
    run_dgrad_gn(*GEOMETRY[geom](5), 320)


@pytest.mark.parametrize("shape", sorted(C2_SHAPES))
def test_c2_forward(shape):
    torch.manual_seed(14)
    B, H, W = C2_SHAPES[shape]
    run_forward(B, H, W, 64 if H == 64 else 128)


@pytest.mark.parametrize("cin", [64, 128])
@pytest.mark.parametrize("shape", sorted(C2_SHAPES))
def test_c2_dgrad(shape, cin):
    torch.manual_seed(15)
    run_dgrad(*C2_SHAPES[shape], cin, accumulate=True)


def test_c2_dgrad_fused_groupnorm_backward_320_columns():
    torch.manual_seed(16)
    run_dgrad_gn(*C2_SHAPES["64x64"], 320)
