"""The transposed convolution engine's tile pipeline: the epilogue that moves each 32-pixel chunk between
accumulator fragments and its 128-byte-swizzled TMA buffer with ldmatrix / stmatrix (one named barrier per chunk),
and the five-stage per-tap ring.  Geometries: fewer tiles than SMs, and CTAs with an odd number of tiles (so the
last tile falls to either consumer warpgroup and the chunk-buffer ring wraps across tiles).

Every output element is checked against float64.  Outputs inside their channel slot start as NaN (except an
accumulate source), the channels beside the slot are random sentinels that must come back bit-identical, and each
launch must have run fdx_tct_kernel.  A bf16 output may differ from the float64 value by its rounding (2^-8
relative) plus the f32 accumulation error, bounded by 2^-12 of the same sum over absolute values; the fused
GroupNorm backward adds the error of its tanh.approx sigmoid."""

import pytest
import torch
import torch.nn.functional as Fnn

from flaxdiff_b200 import _lib, ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
f64 = torch.float64


def last_kernel():
    lib = _lib.load()
    return lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()


def sms():
    return torch.cuda.get_device_properties(dev).multi_processor_count


# (B, H, W): 16 x 16 images, one pixel block each
GEOMETRY = {
    "fewer_tiles_than_sms": lambda: (3, 16, 16),
    "odd_tiles_per_cta": lambda: (3 * sms() + 1, 16, 16),   # 1 or 2 column blocks: 3, 4, 6 or 7 tiles per CTA
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
        bits, old = self.buf.view(torch.int16), self.saved.view(torch.int16)
        lo, hi = self.off, self.off + self.c
        return torch.equal(bits[..., :lo], old[..., :lo]) and torch.equal(bits[..., hi:], old[..., hi:])


def conv64(x, w, stride=1):
    """flax SAME convolution in float64: x NHWC, w HWIO; stride 2 on even sizes pads (0, 1)"""
    xt, wt = x.to(f64).permute(0, 3, 1, 2), w.to(f64).permute(3, 2, 0, 1)
    if stride == 1:
        y = Fnn.conv2d(xt, wt, padding=w.shape[0] // 2)
    else:
        y = Fnn.conv2d(Fnn.pad(xt, (0, 1, 0, 1)), wt, stride=2)
    return y.permute(0, 2, 3, 1)


def dgrad64(dy, w, shape, stride=1):
    x = torch.zeros(shape, dtype=f64, device=dev, requires_grad=True)
    conv64(x, w, stride).backward(dy.to(f64))
    return x.grad


def check(y, ref, absref, slot, extra=0.0):
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tct_kernel"
    yf = y.to(f64)
    assert torch.isfinite(yf).all()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -12 * absref + extra
    over = (yf - ref).abs() > bound
    assert not over.any(), f"{int(over.sum())} of {over.numel()} elements out of bounds"
    assert slot.sentinels_intact()


def check_sums(s, y, x, tol=1e-5):
    """(n, 2, c) column sums against the stored output y: sum y and sum y * x"""
    yf, xf = y.to(f64), x.to(f64)
    for k, ref, mag in ((0, yf.sum((1, 2)), yf.abs().sum((1, 2))),
                        (1, (yf * xf).sum((1, 2)), (yf * xf).abs().sum((1, 2)))):
        assert ((s[:, k].to(f64) - ref).abs() <= tol * mag + 1e-6).all()


@pytest.mark.parametrize("off", [8, 64])
@pytest.mark.parametrize("cin,cout", [(64, 64), (64, 128), (128, 64)])   # K = 64: resident weights; 128: plain halo
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_halo_forward_bias_row_residual_colsums(geom, cin, cout, off):
    torch.manual_seed(31)
    B, H, W = GEOMETRY[geom]()
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    rowvec = torch.randn(B, cout, device=dev) * 0.3
    res = Slot(B, H, W, cout, 64, 8)
    out = Slot(B, H, W, cout, off, 72, fill=float("nan"))
    cs = ops.ColStats(B, off + cout, dev)
    ops.conv3x3_fwd(x, w, bias, rowvec=rowvec, res=res.view, out=out.view, colstats=(cs, off))
    side = bias.to(f64) + rowvec.to(f64).view(B, 1, 1, cout) + res.view.to(f64)
    ref = conv64(x, w) + side
    absref = conv64(x.abs(), w.abs()) + side.abs()
    check(out.view, ref, absref, out)
    check_sums(cs.ws.sum(0)[..., off:], out.view, out.view)


@pytest.mark.parametrize("cin", [64, 192, 320, 384])                    # K = 64; 320 columns: the plain halo grid
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_halo_dgrad_accumulate_in_place(geom, cin):
    torch.manual_seed(32)
    B, H, W = GEOMETRY[geom]()
    dy = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, 64, device=dev) / 24).bfloat16()
    dx = Slot(B, H, W, cin, 64, 8)
    prior = dx.view.to(f64)
    ops.conv3x3_dgrad(dy, w, dx.view, accumulate=True)
    ref = prior + dgrad64(dy, w, (B, H, W, cin))
    absref = prior.abs() + dgrad64(dy.abs(), w.abs(), (B, H, W, cin))
    check(dx.view, ref, absref, dx)


@pytest.mark.parametrize("cin", [64, 128, 192, 320, 384])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_halo_dgrad_fused_groupnorm_backward(geom, cin):
    torch.manual_seed(33)
    B, H, W = GEOMETRY[geom]()
    dy = torch.randn(B, H, W, 64, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, 64, device=dev) / 24).bfloat16()
    x = Slot(B, H, W, cin, 64, 64)
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = Slot(B, H, W, cin, 8, 56, fill=float("nan"))
    ws = ops.conv3x3_dgrad_gn(dy, w, dz.view, x.view, ab)
    z = x.view.to(f64) * ab[:, 0].to(f64).view(B, 1, 1, cin) + ab[:, 1].to(f64).view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    g = dgrad64(dy, w, (B, H, W, cin))
    absg = dgrad64(dy.abs(), w.abs(), (B, H, W, cin))
    silu_grad = s * (1 + z * (1 - s))
    # the sigmoid is 0.5 tanh(z / 2) + 0.5 with tanh.approx: about 2^-12 absolute, times |d silu' / d sigmoid|
    check(dz.view, g * silu_grad, absg * silu_grad.abs(), dz, extra=2.0 ** -12 * (z.abs() + 2) * g.abs())
    assert torch.equal(x.buf.view(torch.int16), x.saved.view(torch.int16))   # the side input is only read
    check_sums(ws.sum(0), dz.view, x.view)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("k", [64, 256])                                 # 1 or 4 ring stages per tile
@pytest.mark.parametrize("cin", [128, 320])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_1x1_dgrad_per_tap_ring(geom, cin, k, accumulate):
    torch.manual_seed(34)
    B, H, W = GEOMETRY[geom]()
    dy = torch.randn(B, H, W, k, device=dev).bfloat16()
    w = (torch.randn(cin, k, device=dev) / k ** 0.5).bfloat16()
    dx = Slot(B, H, W, cin, 64, 8, fill=None if accumulate else float("nan"))
    prior = dx.view.to(f64) if accumulate else torch.zeros(dx.view.shape, dtype=f64, device=dev)
    ops.conv1x1_dgrad(dy, w, dx.view, accumulate=accumulate)
    w4 = w.view(1, 1, cin, k)
    check(dx.view, prior + dgrad64(dy, w4, (B, H, W, cin)), prior.abs() + dgrad64(dy.abs(), w4.abs(), (B, H, W, cin)),
          dx)


@pytest.mark.parametrize("off", [8, 64])
@pytest.mark.parametrize("geom", sorted(GEOMETRY))
def test_1x1_forward_residual_offset(geom, off):
    torch.manual_seed(35)
    B, H, W = GEOMETRY[geom]()
    x = torch.randn(B, H, W, 192, device=dev).bfloat16()
    w = (torch.randn(192, 128, device=dev) / 192 ** 0.5).bfloat16()
    bias = torch.randn(128, device=dev) * 0.3
    res = Slot(B, H, W, 128, 8, 64)
    out = Slot(B, H, W, 128, off, 8, fill=float("nan"))
    ops.conv1x1_fwd(x, w, bias, res=res.view, out=out.view)
    side = bias.to(f64) + res.view.to(f64)
    w4 = w.view(1, 1, 192, 128)
    check(out.view, conv64(x, w4) + side, conv64(x.abs(), w4.abs()) + side.abs(), out)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("cin,k", [(64, 64), (128, 128), (320, 64)])
def test_stride2_dgrad_per_tap_parities(cin, k, accumulate):
    """four parity launches of 1, 2, 2 and 4 taps, each writing every second pixel of the slot"""
    torch.manual_seed(36)
    B, H, W = 4, 32, 32                                                  # dy; dx is 64 x 64
    dy = torch.randn(B, H, W, k, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, k, device=dev) / (3 * k ** 0.5)).bfloat16()
    dx = Slot(B, 2 * H, 2 * W, cin, 64, 8, fill=None if accumulate else float("nan"))
    prior = dx.view.to(f64) if accumulate else torch.zeros(dx.view.shape, dtype=f64, device=dev)
    ops.conv3x3_dgrad(dy, w, dx.view, stride=2, accumulate=accumulate)
    shape = (B, 2 * H, 2 * W, cin)
    check(dx.view, prior + dgrad64(dy, w, shape, 2), prior.abs() + dgrad64(dy.abs(), w.abs(), shape, 2), dx)
