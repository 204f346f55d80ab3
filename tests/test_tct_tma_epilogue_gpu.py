"""The transposed engine's epilogue moves its side input and output by TMA: one {64 channels, 16 px, 2 rows, 1
image} box per 32-pixel chunk, through a ring of 128-byte-swizzled shared-memory buffers per consumer warpgroup.
The output and the side input are channel slots of wider buffers here (pixel stride above the channel count, a
non-zero channel offset), so the tensor maps must clip each box to the slot: the channels beside it are random
sentinels that must come back bit-identical.  Cases: the resident-weight halo launch (K = 64), the plain halo launch
(K = 128), the per-tap 1x1 launches, the fused GroupNorm backward, an in-place accumulate (side input and output
the same view), 64 to 448 columns, and tile counts
from one tile to several per CTA, so that each warpgroup's buffer ring wraps across tiles.  Outputs inside the slot
start as NaN (except where they are the accumulate source), every launch must have run fdx_tct_kernel, and
results are checked against fp32 torch at the tolerances of test_tct_resident_gpu.py."""

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
    k = w.shape[0]
    return Fnn.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(3, 2, 0, 1), b,
                      padding=k // 2).permute(0, 2, 3, 1)


def dgrad_ref(dy, w):
    n, h, wd, _ = dy.shape
    x = torch.zeros(n, h, wd, w.shape[2], device=dev, requires_grad=True)
    conv_ref(x, w).backward(dy.float())
    return x.grad


def sms():
    return torch.cuda.get_device_properties(dev).multi_processor_count


# (B, H, W) by the number of 16 x 16 pixel blocks, for a layer of cblks 64-column blocks
GEOMETRY = {
    "one_tile": lambda c: (1, 16, 16),
    "fewer_tiles_than_sms": lambda c: (2, 32, 32),
    "three_tiles_per_cta": lambda c: (1, 16, 16 * 3 * max(sms() // c, 1)),
    "many_tiles_per_cta": lambda c: (40, 64, 64),
}


class Slot:
    """A channel slot [off, off + c) of a wider NHWC buffer whose other channels are random sentinels."""

    def __init__(self, B, H, W, c, off, extra, fill=None):
        self.buf = torch.randn(B, H, W, off + c + extra, device=dev).bfloat16()
        self.off, self.c = off, c
        self.view = self.buf[..., off:off + c]
        if fill is not None:
            self.view.fill_(fill)
        self.saved = self.buf.clone()

    def sentinels_intact(self):
        bits = self.buf.view(torch.int16)
        old = self.saved.view(torch.int16)
        lo, hi = self.off, self.off + self.c
        return torch.equal(bits[..., :lo], old[..., :lo]) and torch.equal(bits[..., hi:], old[..., hi:])


def check(y, ref, tol, slot):
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    assert torch.isfinite(y.float()).all()
    assert rel(y, ref) < tol
    assert slot.sentinels_intact()


@pytest.mark.parametrize("cin", [64, 128])              # K = 64: resident weights; K = 128: plain halo
@pytest.mark.parametrize("cout", [64, 128])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_forward_residual_slot(geom, cout, cin):
    torch.manual_seed(21)
    B, H, W = GEOMETRY[geom](cout // 64)
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    rowvec = torch.randn(B, cout, device=dev) * 0.3
    res = Slot(B, H, W, cout, 64, 64)
    out = Slot(B, H, W, cout, 64, 128, fill=float("nan"))
    cs = ops.ColStats(B, cout + 192, dev)
    ops.conv3x3_fwd(x, w, bias, rowvec=rowvec, res=res.view, out=out.view, colstats=(cs, 64))
    check(out.view, conv_ref(x, w, bias) + rowvec.view(B, 1, 1, cout) + res.view.float(), 5e-3, out)
    assert rel(ops.groupnorm_stats_from_cols(cs, 8, 64, cout), ops.groupnorm_stats(out.view.contiguous(), 8)) < 1e-5


@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_1x1_forward_channel_offset_8(geom):
    """per-tap stages; the slots start 16 bytes into the pixel, off the 128-byte line the swizzle works in"""
    torch.manual_seed(22)
    B, H, W = GEOMETRY[geom](1)
    x = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(64, 64, device=dev) / 8).bfloat16()
    bias = torch.randn(64, device=dev) * 0.3
    res = Slot(B, H, W, 64, 8, 56)
    out = Slot(B, H, W, 64, 8, 8, fill=float("nan"))
    ops.conv1x1_fwd(x, w, bias, res=res.view, out=out.view)
    check(out.view, conv_ref(x, w.view(1, 1, 64, 64), bias) + res.view.float(), 5e-3, out)


@pytest.mark.parametrize("cin", [64, 192, 320, 448])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_dgrad_accumulate_in_place_slot(geom, cin):
    torch.manual_seed(23)
    B, H, W = GEOMETRY[geom](cin // 64)
    dy = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, 64, device=dev) / 24).bfloat16()
    dx = Slot(B, H, W, cin, 64, 64)
    prior = dx.view.float().clone()
    ops.conv3x3_dgrad(dy, w, dx.view, accumulate=True)
    check(dx.view, prior + dgrad_ref(dy, w), 5e-3, dx)


@pytest.mark.parametrize("cin", [64, 320])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_dgrad_fused_groupnorm_backward_slots(geom, cin):
    torch.manual_seed(24)
    B, H, W = GEOMETRY[geom](cin // 64)
    dy = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, 64, device=dev) / 24).bfloat16()
    x = Slot(B, H, W, cin, 128, 64)
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = Slot(B, H, W, cin, 64, 192, fill=float("nan"))
    ws = ops.conv3x3_dgrad_gn(dy, w, dz.view, x.view, ab)
    xf = x.view.float()
    z = xf * ab[:, 0].view(B, 1, 1, cin) + ab[:, 1].view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    check(dz.view, dgrad_ref(dy, w) * s * (1 + z * (1 - s)), 1e-2, dz)
    assert torch.equal(x.buf.view(torch.int16), x.saved.view(torch.int16))   # the side input is only read
    sums = ws.sum(0)
    assert rel(sums[:, 0], dz.view.float().sum((1, 2))) < 1e-4
    assert rel(sums[:, 1], (dz.view.float() * xf).sum((1, 2))) < 1e-4


@pytest.mark.parametrize("cin,cout", [(64, 64), (192, 128), (576, 128)])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_1x1_forward_residual_slot(geom, cin, cout):
    torch.manual_seed(25)
    B, H, W = GEOMETRY[geom](cout // 64)
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(cin, cout, device=dev) / cin ** 0.5).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    res = Slot(B, H, W, cout, 64, 0)
    out = Slot(B, H, W, cout, 128, 64, fill=float("nan"))
    ops.conv1x1_fwd(x, w, bias, res=res.view, out=out.view)
    check(out.view, conv_ref(x, w.view(1, 1, cin, cout), bias) + res.view.float(), 5e-3, out)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("cin", [64, 128, 320, 448])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_1x1_dgrad_slot(geom, cin, accumulate):
    torch.manual_seed(26)
    B, H, W = GEOMETRY[geom](cin // 64)
    dy = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(cin, 64, device=dev) / 8).bfloat16()
    dx = Slot(B, H, W, cin, 64, 64, fill=None if accumulate else float("nan"))
    prior = dx.view.float().clone() if accumulate else 0.0
    ops.conv1x1_dgrad(dy, w, dx.view, accumulate=accumulate)
    check(dx.view, prior + dgrad_ref(dy, w.view(1, 1, cin, 64)), 5e-3, dx)
