"""The convolution and GEMM engines compared element by element with the float64 references of
tests/elementwise_ref.py, through every route fdx_tc_launch / fdx_tct_launch / fdx_wgrad9_launch selects, at the
UNet's own layers: C2's full batch (256 images of 64 x 64 and 32 x 32), C3's 256 x 256 levels, the gallery UNet's
1024-channel 8 x 8 and 16 x 16 layers, and the ragged and tiny edges.

Every case runs twice:
  * dense: random bf16 operands, checked against the per-element bound of the reference (the worst
    |err| / bound is printed as `WORST <case> <ratio>`);
  * exact: integer operands in {-2, ..., 2} (weights optionally scaled by a power of two), integer bias, residual
    and prior.  The case asserts that every output's sum of |terms| is below 2^24; then any f32 summation order
    is exact, so f32 outputs must equal the float64 result and bf16 outputs its bf16 rounding, bit for bit.
    This is what sees a dropped pixel block or a skipped split in a reduction of 10^6 pixels, which no
    magnitude bound can.
Outputs are channel slots of wider buffers with sentinel channels on both sides that must come back
bit-identical; outputs that are not accumulated start as NaN, accumulated ones (dgrad(accumulate=True), every
weight gradient) start from a random prior.  Each case id names its route, restated on the host from the
launch code, and the case asserts the kind of the kernel that ran last."""
import ctypes
import math

import pytest
import torch

import elementwise_ref as R
from flaxdiff_b200 import _lib, ops
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN, ptr, stream_ptr

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64
SENTINEL = -1234.0                                   # exactly representable in bf16
LO, HI = 8, 16                                       # sentinel channels left / right of a bf16 slot
KIND = {"tc": 0, "tct": 1, "wgrad9": 3}              # FDX_KERNEL_TC / TCT / WGRAD9
KINDS = ("dense", "exact")
# The ids name the route for this device's SM count; without a device the cases are only collected (and
# skipped), named for a 132-SM H100 SXM.
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def sms() -> int:
    n = _lib.load().fdx_device_sm_count()
    assert n == SMS, (n, SMS)
    return n


def report(name, frac):
    print(f"WORST {name} {frac:.3f}")


def assert_route(route):
    kind = _lib.load().fdx_last_kernel_kind()
    assert kind == KIND[route.split("-")[0]], (route, kind)


# ----------------------------------------------------------------------------------------------- routes
def launch_route(W, H, N, K, Ncols, es=1, halo=True):
    """fdx_tc_launch hands a pixels-as-M launch (forward or data gradient) to fdx_tct_launch when es = 1, Ncols
    is a multiple of 64 but not of 256 and at most 512, and W, H, K are multiples of 16, 16, 64 (fdx_tct.cu);
    the halo variant serves the standard 3x3 tap set and keeps its weights resident when K = 64 and a grid of
    whole column-block groups idles no SM that the plain grid would use.  Elsewhere fdx_tc_kernel with the
    column tile of its cost model."""
    if es == 1 and Ncols % 64 == 0 and Ncols % 256 != 0 and Ncols <= 512 and W % 16 == 0 and H % 16 == 0 \
            and K % 64 == 0:
        if not halo:
            return "tct-pertap"
        cblks = Ncols // 64
        ntiles = cblks * (W // 16) * (H // 16) * N
        if K == 64 and min(ntiles, SMS // cblks * cblks) == min(ntiles, SMS):
            return "tct-halo-resident"
        return "tct-halo-streamed"
    return f"tc-bn{R.tc_bn(Ncols)}"


def wgrad_route(H, W, stride):
    """fdx_conv3x3_wgrad: fdx_wgrad9_launch at stride 1 on power-of-two images with W >= 8 and H >= 64 / TW
    (TW = 16 for W >= 16, else 8), the generic TC_MNMN split-K launch otherwise."""
    pow2 = W >= 8 and W & (W - 1) == 0 and H & (H - 1) == 0
    if stride == 1 and pow2 and H >= 64 // (16 if W >= 16 else 8):
        return f"wgrad9-tw{16 if W >= 16 else 8}"
    return "tc-mnmn"


# ----------------------------------------------------------------------------------------------- operands
def draw(shape, kind, g, scale=1.0, dtype=torch.bfloat16):
    """dense: N(0, scale^2); exact: integers in {-2..2} times the power of two nearest to scale."""
    if kind == "exact":
        t = torch.randint(-2, 3, tuple(shape), generator=g, device=dev).float() * 2.0 ** round(math.log2(scale))
    else:
        t = torch.randn(tuple(shape), generator=g, device=dev) * scale
    return t.to(dtype)


def gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def slot(shape, fill=math.nan, dtype=torch.bfloat16):
    """Channel slot [LO, LO + C) of a wider NHWC buffer holding `fill`, its neighbours SENTINEL."""
    *lead, C = shape
    buf = torch.full((*lead, LO + C + HI), SENTINEL, dtype=dtype, device=dev)
    v = buf[..., LO:LO + C]
    v.fill_(fill)
    return buf, v


def into_slot(t):
    buf, v = slot(tuple(t.shape), dtype=t.dtype)
    v.copy_(t)
    return buf, v


def guarded_f32(t):
    """A contiguous f32 copy of t with four sentinels on either side (16-byte aligned)."""
    n = t.numel()
    buf = torch.full((n + 8,), SENTINEL, dtype=torch.float32, device=dev)
    v = buf[4:4 + n].view(t.shape)
    v.copy_(t)
    return buf, v


def assert_guard(buf, C=None):
    if C is None:                                     # guarded_f32
        ends = torch.cat([buf[:4], buf[-4:]])
        assert torch.equal(ends, torch.full_like(ends, SENTINEL)), "a kernel wrote outside its output"
    else:
        R.assert_guard_intact(buf, LO, C, SENTINEL)


def check(kind, what, got, ref, args, bf16_out):
    """dense: |got - ref| within the reference's bound; exact: bit for bit (bf16 outputs: the exact value
    rounded to bf16), given that every output's sum of |terms| is below 2^24."""
    val, delta = ref(**args)
    if kind == "exact":
        mag = ref(**{k: (v.abs() if isinstance(v, torch.Tensor) else v) for k, v in args.items()})[0]
        assert R.exact_case_ok(mag), f"{what}: the exact case's sums reach 2^24"
        want = val.to(torch.bfloat16).to(F64) if bf16_out else val
        bad = ~(got.to(F64) == want)
        if bad.any():
            i = tuple(int(j) for j in torch.nonzero(bad)[0])
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from the exact "
                                 f"result; first at {i}: got {got[i].item()!r}, exact {val[i].item()!r}")
        return
    bound = R.bf16_bound(val, delta) if bf16_out else R.f32_bound(val, delta)
    report(what, R.assert_elementwise(got, val, bound, what))


def f64(t):
    return None if t is None else t.to(F64)


# ----------------------------------------------------------------------------------------------- conv3x3 forward
# (N, H, W, Cin, Cout, stride, epilogue)
FWD = [
    (256, 64, 64, 64, 64, 1, "bias"),                  # C2 64 x 64
    (256, 32, 32, 128, 128, 1, "bias+res"),            # C2 32 x 32
    (256, 16, 16, 256, 256, 1, ""),                    # C2 16 x 16
    (2, 256, 256, 64, 64, 1, "bias"),                  # C3 256 x 256
    (4, 16, 16, 64, 128, 1, ""),
    (4, 16, 16, 64, 192, 1, ""),
    (4, 16, 16, 64, 320, 1, ""),                       # 20 tiles: resident
    (32, 16, 16, 64, 320, 1, ""),                      # 160 tiles: five column blocks do not divide the grid
    (4, 16, 16, 64, 384, 1, ""),
    (8, 16, 16, 64, 448, 1, "bias"),
    (4, 16, 16, 128, 128, 1, "bias+res+rowvec"),
    (2, 16, 16, 1024, 1024, 1, "bias"),                # gallery 16 x 16
    (4, 8, 8, 1024, 1024, 1, ""),                      # gallery 8 x 8
    (8, 8, 8, 64, 64, 1, "bias"),
    (8, 8, 8, 128, 128, 1, "res"),
    (8, 8, 8, 128, 512, 1, ""),
    (16, 2, 2, 64, 64, 1, "bias+res+rowvec"),          # 2 x 2 images: many images per tile
    (8, 32, 32, 64, 64, 2, "bias"),                    # stride 2, pad (0, 1)
    (4, 64, 64, 128, 128, 2, ""),
    (4, 15, 15, 64, 64, 2, "bias"),                    # stride 2 on odd sizes, pad (1, 1)
]


def _fwd_id(c):
    N, H, W, Ci, Co, s, epi = c
    Ho, Wo = -(-H // s), -(-W // s)
    r = launch_route(Wo, Ho, N, Ci, Co, s, s == 1)
    return f"{r}-B{N}-{H}x{W}-{Ci}to{Co}-s{s}" + (f"-{epi}" if epi else "")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", FWD, ids=[_fwd_id(c) for c in FWD])
def test_conv3x3_fwd(case, kind):
    N, H, W, Ci, Co, s, epi = case
    g = gen(1)
    Ho, Wo = -(-H // s), -(-W // s)
    x = draw((N, H, W, Ci), kind, g)
    w = draw((3, 3, Ci, Co), kind, g, 1 / math.sqrt(9 * Ci))
    bias = draw((Co,), kind, g, dtype=torch.float32) if "bias" in epi else None
    rowvec = draw((N, Co), kind, g, dtype=torch.float32) if "rowvec" in epi else None
    res = draw((N, Ho, Wo, Co), kind, g) if "res" in epi.split("+") else None
    buf, y = slot((N, Ho, Wo, Co))
    ops.conv3x3_fwd(x, w, bias=bias, rowvec=rowvec, res=res, out=y, stride=s)
    route = _fwd_id(case).split("-B")[0]
    assert_route(route)
    assert_guard(buf, Co)
    args = dict(x=f64(x), w_hwio=f64(w), stride=s, bias=f64(bias), rowvec=f64(rowvec), res=f64(res))
    check(kind, "conv3x3_fwd " + route, y, R.conv3x3_fwd_ref, args, True)


# ----------------------------------------------------------------------------------------------- conv3x3 data gradient
# (N, H, W, Cin, Cout, stride, accumulate), (H, W) of dx
DGRAD = [
    (256, 64, 64, 64, 64, 1, False),                   # C2 64 x 64
    (256, 32, 32, 128, 128, 1, True),                  # C2 32 x 32
    (8, 32, 32, 192, 64, 1, False),                    # the up path's concat inputs
    (8, 32, 32, 384, 128, 1, True),
    (8, 16, 16, 128, 128, 1, False),
    (4, 16, 16, 1024, 1024, 1, False),                 # gallery 16 x 16
    (4, 8, 8, 1024, 1024, 1, True),                    # gallery 8 x 8
    (8, 8, 8, 64, 64, 1, True),
    (16, 2, 2, 64, 128, 1, False),
    (256, 64, 64, 64, 64, 2, False),                   # C2 downsample: four parity launches of 4, 2, 2, 1 taps
    (8, 32, 32, 64, 64, 2, True),
    (8, 16, 16, 128, 128, 2, True),                    # 8 x 8 dy: pixels-as-M engine
]


def _dgrad_id(c):
    N, H, W, Ci, Co, s, acc = c
    r = launch_route(W // s, H // s, N, Co, Ci, 1, s == 1)
    return ("s2parity-" if s == 2 else "") + f"{r}-B{N}-{H}x{W}-{Ci}from{Co}" + ("-accumulate" if acc else "")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", DGRAD, ids=[_dgrad_id(c) for c in DGRAD])
def test_conv3x3_dgrad(case, kind):
    N, H, W, Ci, Co, s, acc = case
    g = gen(2)
    dy = draw((N, H // s, W // s, Co), kind, g)
    w = draw((3, 3, Ci, Co), kind, g, 1 / math.sqrt(9 * Co))
    prior = draw((N, H, W, Ci), kind, g) if acc else None
    buf, dx = into_slot(prior) if acc else slot((N, H, W, Ci))
    ops.conv3x3_dgrad(dy, w, dx, stride=s, accumulate=acc)
    route = _dgrad_id(case).split("-B")[0].replace("s2parity-", "")
    assert_route(route)
    assert_guard(buf, Ci)
    args = dict(dy=f64(dy), w_hwio=f64(w), stride=s, prior=f64(prior))
    check(kind, "conv3x3_dgrad " + _dgrad_id(case).split("-B")[0], dx, R.conv3x3_dgrad_ref, args, True)


# ----------------------------------------------------------------------------------------------- conv3x3 weight gradient
# (N, H, W, Cin, Cout, stride), (H, W) of x
WGRAD = [
    (256, 64, 64, 64, 64, 1),                          # C2 64 x 64: 2^20 pixels per weight
    (256, 32, 32, 128, 128, 1),                        # C2 32 x 32
    (2, 256, 256, 64, 64, 1),                          # C3 256 x 256
    (4, 16, 16, 1024, 1024, 1),                        # gallery 16 x 16
    (16, 8, 8, 1024, 1024, 1),                         # gallery 8 x 8
    (8, 16, 16, 64, 128, 1),
    (256, 64, 64, 64, 64, 2),                          # C2 downsample
    (8, 32, 32, 64, 128, 2),
    (4, 24, 24, 64, 64, 1),                            # not a power of two
    (8, 12, 12, 128, 64, 1),
    (16, 2, 2, 64, 64, 1),
]


def _wgrad_id(c):
    N, H, W, Ci, Co, s = c
    return f"{wgrad_route(H, W, s)}-B{N}-{H}x{W}-{Ci}x{Co}-s{s}"


def wgrad_depth(N, H, W, Ci, Co, s):
    if wgrad_route(H, W, s).startswith("wgrad9"):
        return R.wgrad9_depth(N, H, W, Ci, Co, sms())
    Ho, Wo = -(-H // s), -(-W // s)
    return R.mnmn_depth(Wo, Ho, N, Ci, Co, 9, sms())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", WGRAD, ids=[_wgrad_id(c) for c in WGRAD])
def test_conv3x3_wgrad(case, kind):
    N, H, W, Ci, Co, s = case
    g = gen(3)
    x = draw((N, H, W, Ci), kind, g)
    dy = draw((N, -(-H // s), -(-W // s), Co), kind, g)
    prior = draw((3, 3, Ci, Co), kind, g, 16.0, torch.float32)
    buf, dw = guarded_f32(prior)
    ops.conv3x3_wgrad(x, dy, dw, stride=s)
    route = wgrad_route(H, W, s)
    assert_route(route)
    assert_guard(buf)
    args = dict(x=f64(x), dy=f64(dy), depth=wgrad_depth(N, H, W, Ci, Co, s), stride=s, prior=f64(prior))
    check(kind, "conv3x3_wgrad " + route, dw, R.conv3x3_wgrad_ref, args, False)


# ----------------------------------------------------------------------------------------------- 1x1 convolutions
@pytest.mark.parametrize("kind", KINDS)
def test_conv1x1_tct_pertap(kind):
    """The residual 1x1 convolution: forward with bias and residual, data gradient accumulated; one tap, so the
    transposed engine's per-tap loads."""
    N, H, W, Ci, Co = 8, 32, 32, 128, 64
    g = gen(4)
    x = draw((N, H, W, Ci), kind, g)
    w = draw((Ci, Co), kind, g, 1 / math.sqrt(Ci))
    bias = draw((Co,), kind, g, dtype=torch.float32)
    res = draw((N, H, W, Co), kind, g)
    buf, y = slot((N, H, W, Co))
    ops.conv1x1_fwd(x, w, bias=bias, res=res, out=y)
    assert_route("tct")
    assert_guard(buf, Co)
    P = N * H * W
    gref = lambda a, b, bias=None, res=None, prior=None: R.gemm_ref(a, b, a.shape[-1] + R.EPI, bias=bias, res=res,  # noqa: E731
                                                                     prior=prior)
    check(kind, "conv1x1_fwd tct-pertap", y.reshape(P, Co), gref,
          dict(a=f64(x).reshape(P, Ci), b=f64(w), bias=f64(bias), res=f64(res).reshape(P, Co)), True)
    dy = draw((N, H, W, Co), kind, g)
    prior = draw((N, H, W, Ci), kind, g)
    buf, dx = into_slot(prior)
    ops.conv1x1_dgrad(dy, w, dx, accumulate=True)
    assert_route("tct")
    assert_guard(buf, Ci)
    check(kind, "conv1x1_dgrad tct-pertap", dx.reshape(P, Ci), gref,
          dict(a=f64(dy).reshape(P, Co), b=f64(w).T, prior=f64(prior).reshape(P, Ci)), True)


# ----------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("kind", KINDS)
def test_gemm_kk_f32_alpha(kind):
    """GEMM_KK, f32 D with alpha, ragged M (300) and leading dimensions wider than the matrices."""
    M, N, K, alpha = 300, 96, 128, 0.125
    g = gen(5)
    A = draw((M, K + 8), kind, g)
    B = draw((N, K), kind, g, 1 / math.sqrt(K))
    Dbuf = torch.full((M, 4 + N + 4), SENTINEL, dtype=torch.float32, device=dev)
    D = Dbuf[:, 4:4 + N]
    D.fill_(math.nan)
    ops.gemm(GEMM_KK, A, B, D, M, N, K, A.stride(0), B.stride(0), Dbuf.stride(0), alpha=alpha)
    assert_route("tc")
    assert R.tc_bn(N) == 128
    side = torch.cat([Dbuf[:, :4], Dbuf[:, 4 + N:]], 1)
    assert torch.equal(side, torch.full_like(side, SENTINEL))
    ref = lambda a, b: R.gemm_ref(a, b, K + R.EPI, alpha=alpha)  # noqa: E731
    check(kind, "gemm KK tc-bn128", D, ref, dict(a=f64(A[:, :K]), b=f64(B).T), False)


@pytest.mark.parametrize("kind", KINDS)
def test_gemm_kmn_bias_residual_batched(kind):
    """GEMM_KMN, bf16 D with bias and residual, N % 64 = 32, ragged M and a (2 x 3) batch of strided A, B, D
    and residual."""
    b1, b2, M, N, K = 2, 3, 77, 160, 192
    g = gen(6)
    a_ld, r_ld = K + 8, N + 8
    A = draw((b2, b1, M, a_ld), kind, g)
    B = draw((b2, b1, K, N), kind, g, 1 / math.sqrt(K))
    bias = draw((N,), kind, g, dtype=torch.float32)
    res = draw((b2, b1, M, r_ld), kind, g)
    Dbuf, D = slot((b2, b1, M, N))
    ops.gemm(GEMM_KMN, A, B, D, M, N, K, a_ld, N, Dbuf.shape[-1], b1, b2,
             a_s=(M * a_ld, b1 * M * a_ld), b_s=(K * N, b1 * K * N), d_s=(M * Dbuf.shape[-1], b1 * M * Dbuf.shape[-1]),
             bias=bias, res=res, r_ld=r_ld, r_s=(M * r_ld, b1 * M * r_ld))
    assert_route("tc")
    assert_guard(Dbuf, N)
    ref = lambda a, b, bias, res: R.gemm_ref(a, b, K + R.EPI, bias=bias, res=res)  # noqa: E731
    check(kind, f"gemm KMN tc-bn{R.tc_bn(N)}", D, ref,
          dict(a=f64(A[..., :K]), b=f64(B), bias=f64(bias), res=f64(res[..., :N])), True)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("mode", ["reduce_batch-atomic", "single-split"])
def test_gemm_mnmn(mode, kind):
    """GEMM_MNMN (D = A^T B, A [k][m], B [k][n]): reduced over a batch of 4 with split-K atomics onto a prior, and
    per batch entry with one split (no atomics)."""
    b1, M, N, K = 4, 64, 96, 4096
    g = gen(7)
    A = draw((b1, K, M), kind, g)
    B = draw((b1, K, N), kind, g, 1 / 64)
    reduce = mode != "single-split"
    lead = (M,) if reduce else (b1, M)
    if reduce:
        prior = draw(lead + (N,), kind, g, 16.0, torch.float32)
    Dbuf = torch.full(lead + (4 + N + 4,), SENTINEL, dtype=torch.float32, device=dev)
    D = Dbuf[..., 4:4 + N]
    D.copy_(prior) if reduce else D.fill_(math.nan)
    d_ld = Dbuf.shape[-1]
    ops.gemm(GEMM_MNMN, A, B, D, M, N, K, M, N, d_ld, b1, 1, d_s=(0 if reduce else M * d_ld, 0),
             atomic=reduce, reduce_batch=reduce)
    assert_route("tc")
    side = torch.cat([Dbuf[..., :4], Dbuf[..., 4 + N:]], -1)
    assert torch.equal(side, torch.full_like(side, SENTINEL))
    if reduce:
        depth = R.mnmn_depth(K, b1, 1, M, N, 1, sms(), gemm=True)
        args = dict(a=f64(A).permute(2, 0, 1).reshape(M, b1 * K), b=f64(B).reshape(b1 * K, N), prior=f64(prior))
    else:
        depth = R.mnmn_depth(K, b1, 1, M, N, 1, sms(), gemm=True, splits=1, mn_batched=True)
        assert depth == K + 2
        args = dict(a=f64(A).transpose(1, 2), b=f64(B))
    ref = lambda a, b, prior=None: R.gemm_ref(a, b, depth, prior=prior)  # noqa: E731
    check(kind, f"gemm MNMN {mode} tc-mnmn", D, ref, args, False)


# ----------------------------------------------------------------------------------------------- sub-pixel upsample
@pytest.mark.parametrize("kind", KINDS)
def test_upconv_pack_bit_exact(kind):
    """upconv_pack_kernel equals its host restatement bit for bit; its rounding is within PACK of the exact
    tap sums' magnitudes (printed as the worst ratio)."""
    g = gen(8)
    w = draw((3, 3, 256, 128), kind, g, 1 / 48, torch.float32)
    got = ops.upconv3x3_pack(w)
    want = R.upconv_pack_ref(w)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    ex = torch.zeros(16, 256, 128, dtype=F64, device=dev)
    ex_abs = torch.zeros_like(ex)
    for ph in range(4):
        for ky in range(3):
            for kx in range(3):
                i = ph * 4 + R.up_slot(ph >> 1, ky) * 2 + R.up_slot(ph & 1, kx)
                ex[i] += w[ky, kx].to(F64)
                ex_abs[i] += w[ky, kx].to(F64).abs()
    report("upconv3x3_pack", R.assert_elementwise(got, ex, R.PACK * ex_abs, "upconv pack"))


UPCONV = [(8, 16, 16, 128, 128), (32, 32, 32, 64, 64), (4, 8, 8, 256, 256), (2, 128, 128, 64, 64)]


def _up_id(c, what):
    N, h, w, Ci, Co = c
    r = {"fwd": launch_route(w, h, N, Ci, Co, halo=False), "dgrad": f"tc-bn{R.tc_bn(Ci)}", "wgrad": "tc-mnmn"}[what]
    return f"{r}-B{N}-{h}x{w}-{Ci}to{Co}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", UPCONV, ids=[_up_id(c, "fwd") for c in UPCONV])
def test_upconv3x3_fwd(case, kind):
    """Four parity launches of 4 taps each, with the bias, against nearest 2x + conv3x3 with the f32 weights."""
    N, h, w_, Ci, Co = case
    g = gen(9)
    x = draw((N, h, w_, Ci), kind, g)
    w = draw((3, 3, Ci, Co), kind, g, 1 / math.sqrt(9 * Ci), torch.float32)
    bias = draw((Co,), kind, g, dtype=torch.float32)
    buf, y = slot((N, 2 * h, 2 * w_, Co))
    ops.upconv3x3_fwd(x, ops.upconv3x3_pack(w), bias, y)
    route = _up_id(case, "fwd").split("-B")[0]
    assert_route(route)
    assert_guard(buf, Co)
    check(kind, "upconv3x3_fwd " + route, y, R.upconv_fwd_ref, dict(x=f64(x), w_hwio=f64(w), bias=f64(bias)), True)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", UPCONV, ids=[_up_id(c, "dgrad") for c in UPCONV])
def test_upconv3x3_dgrad_accumulate(case, kind):
    """One launch of 16 taps reading dY at every other pixel (es = 2: the pixels-as-M engine), onto a prior."""
    N, h, w_, Ci, Co = case
    g = gen(10)
    dy = draw((N, 2 * h, 2 * w_, Co), kind, g)
    w = draw((3, 3, Ci, Co), kind, g, 1 / math.sqrt(9 * Co), torch.float32)
    prior = draw((N, h, w_, Ci), kind, g)
    buf, dx = into_slot(prior)
    ops.upconv3x3_dgrad(dy, ops.upconv3x3_pack(w), dx, accumulate=True)
    route = _up_id(case, "dgrad").split("-B")[0]
    assert_route(route)
    assert_guard(buf, Ci)
    check(kind, "upconv3x3_dgrad " + route, dx, R.upconv_dgrad_ref, dict(dy=f64(dy), w_hwio=f64(w), prior=f64(prior)),
          True)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", UPCONV, ids=[_up_id(c, "wgrad") for c in UPCONV])
def test_upconv3x3_wgrad_fold(case, kind):
    """A TC_MNMN launch of 16 taps over the low-resolution pixels, folded onto the nine taps of a prior."""
    N, h, w_, Ci, Co = case
    g = gen(11)
    x = draw((N, h, w_, Ci), kind, g)
    dy = draw((N, 2 * h, 2 * w_, Co), kind, g)
    prior = draw((3, 3, Ci, Co), kind, g, 16.0, torch.float32)
    buf, dw = guarded_f32(prior)
    ops.upconv3x3_wgrad(x, dy, dw)
    assert_route("tc")
    assert_guard(buf)
    depth = R.upconv_wgrad_depth(N, h, w_, Ci, Co, sms())
    check(kind, "upconv3x3_wgrad tc-mnmn", dw, R.upconv_wgrad_ref,
          dict(x=f64(x), dy=f64(dy), depth=depth, prior=f64(prior)), False)


# ----------------------------------------------------------------------------------------------- 3-channel convolutions
C3CH = [(256, 64, 64, 64), (2, 256, 256, 128), (3, 10, 12, 64)]


def _c3_id(c):
    N, H, W, C = c
    return f"tc-bn{R.tc_bn(C)}-B{N}-{H}x{W}-{C}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", C3CH, ids=[_c3_id(c) for c in C3CH])
def test_conv_in(case, kind):
    """conv_in 3 -> C: im2col3 (bit for bit), a GEMM_KMN of K = 27 with the bias into a channel slot, and the
    weight and bias gradients by a GEMM_MNMN reduce over every pixel onto priors."""
    N, H, W, C = case
    g = gen(12)
    x = draw((N, H, W, 3), kind, g)
    w = draw((3, 3, 3, C), kind, g, 1 / 6, torch.float32)
    bias = draw((C,), kind, g, dtype=torch.float32)
    assert torch.equal(ops.im2col3(x, +1, True).view(torch.int16), R.im2col3_ref(x, +1, True).view(torch.int16))
    buf, y = slot((N, H, W, C))
    ops.conv_in_fwd(x, w, bias, y)
    assert_route("tc")
    assert_guard(buf, C)
    check(kind, "conv_in_fwd tc", y, R.conv_in_fwd_ref, dict(x=f64(x), w_hwio=f64(w), bias=f64(bias)), True)
    dy = draw((N, H, W, C), kind, g)
    pw, pb = draw((3, 3, 3, C), kind, g, 16.0, torch.float32), draw((C,), kind, g, 16.0, torch.float32)
    bw, dw = guarded_f32(pw)
    bb, db = guarded_f32(pb)
    ops.conv_in_wgrad(x, dy, dw, db)
    assert_route("tc")
    assert_guard(bw)
    assert_guard(bb)
    depth = R.mnmn_depth(N * H * W, 1, 1, 32, C, 1, sms(), gemm=True) + 1
    for i, (name, got) in enumerate((("dw", dw), ("dbias", db))):
        ref = lambda x, dy, dw_prior, db_prior, i=i: R.conv_in_wgrad_ref(x, dy, depth, dw_prior, db_prior)[i]  # noqa: E731
        check(kind, f"conv_in_wgrad {name} tc-mnmn", got, ref,
              dict(x=f64(x), dy=f64(dy), dw_prior=f64(pw), db_prior=f64(pb)), False)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", C3CH, ids=[_c3_id(c) for c in C3CH])
def test_conv_out(case, kind):
    """conv_out C -> 3: the f32 column GEMM + col2im3 (bit for bit against its restatement) forward, the data
    gradient from im2col3 of the f32 loss gradient (bit for bit) and the weight and bias gradients onto priors."""
    N, H, W, C = case
    g = gen(13)
    x = draw((N, H, W, C), kind, g)
    w = draw((3, 3, C, 3), kind, g, 1 / math.sqrt(9 * C), torch.float32)
    bias = draw((3,), kind, g, dtype=torch.float32)
    y = ops.conv_out_fwd(x, w, bias)
    assert_route("tc")
    check(kind, "conv_out_fwd tc", y, R.conv_out_fwd_ref, dict(x=f64(x), w_hwio=f64(w), bias=f64(bias)), False)
    # col2im3 alone, on random f32 columns
    col = draw((N * H * W, 32), kind, g, dtype=torch.float32)
    yc = torch.empty((N, H, W, 3), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().fdx_col2im3x3_c3(ptr(col), ptr(bias), ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W),
                                            ptr(yc), stream_ptr()), "col2im3x3_c3")
    assert torch.equal(yc, R.col2im3_ref(col, bias, N, H, W))
    dF = draw((N, H, W, 3), kind, g, 1.0, torch.float32)
    col = ops.im2col3(dF, -1, False)
    assert torch.equal(col.view(torch.int16), R.im2col3_ref(dF, -1, False).view(torch.int16))
    buf, dx = slot((N, H, W, C))
    ops.conv_out_dgrad(dF, w, dx, col=col)
    assert_route("tc")
    assert_guard(buf, C)
    check(kind, "conv_out_dgrad tc", dx, R.conv_out_dgrad_ref, dict(dF=f64(dF), w_hwio=f64(w)), True)
    pw, pb = draw((3, 3, C, 3), kind, g, 16.0, torch.float32), draw((3,), kind, g, 16.0, torch.float32)
    bw, dw = guarded_f32(pw)
    bb, db = guarded_f32(pb)
    ops.conv_out_wgrad(x, dF, dw, db, col=col)
    assert_route("tc")
    assert_guard(bw)
    assert_guard(bb)
    depth = R.mnmn_depth(N * H * W, 1, 1, C, 32, 1, sms(), gemm=True) + 1
    for i, (name, got) in enumerate((("dw", dw), ("dbias", db))):
        ref = lambda x, dF, dw_prior, db_prior, i=i: R.conv_out_wgrad_ref(x, dF, depth, dw_prior, db_prior)[i]  # noqa: E731
        check(kind, f"conv_out_wgrad {name} tc-mnmn", got, ref,
              dict(x=f64(x), dF=f64(dF), dw_prior=f64(pw), db_prior=f64(pb)), False)
