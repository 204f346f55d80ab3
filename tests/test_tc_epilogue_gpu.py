"""The tap-GEMM engine (fdx_tc_kernel) in every instantiation: column tiles of 64, 128 and 256 in the forward,
data-gradient and weight-gradient modes, each epilogue (plain bf16, fused GroupNorm backward, column sums, f32,
f32 reductions), and the epilogue's edge cases: a last 64-column chunk without its second half, a column count
that is not a multiple of the tile, tiles with rows past the image, an odd number of 64-deep K chunks at the
64-column tile, and tap pairing in the weight gradient.  The shapes are ones the transposed engine declines
(multiples of 256 columns, 8 x 8 and 24 x 24 images, stride 2, 768 columns, GEMMs).  Each launch is checked to
have run fdx_tc_kernel, and its result against fp32 torch."""
import ctypes

import pytest
import torch
import torch.nn.functional as Fnn

from flaxdiff_b200 import _lib, ops
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

BF16_TOL, F32_TOL = 5e-3, 1e-4


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def last_kernel():
    lib = _lib.load()
    lib.fdx_kernel_kind_name.restype = ctypes.c_char_p
    return lib.fdx_kernel_kind_name(lib.fdx_last_kernel_kind()).decode()


def ran_tc():
    torch.cuda.synchronize()
    assert last_kernel() == "fdx_tc_kernel"


def conv_ref(x, w, stride=1):
    # NHWC / HWIO; SAME padding as flax: stride 1 pads (1, 1), stride 2 on even sizes (0, 1)
    xn = x.float().permute(0, 3, 1, 2)
    xn = Fnn.pad(xn, (1, 1, 1, 1) if stride == 1 else (0, 1, 0, 1))
    return Fnn.conv2d(xn, w.float().permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def rand_w(cin, cout):
    return (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()


# (B, H, W, Cin, Cout, stride): 256 and 512 columns -> BN 256; 128 columns on 8 x 8 -> BN 128; 64 columns on 8 x 8
# with K = 192 -> BN 64 and 27 K chunks; 320 columns at stride 2 -> BN 128, last tile half full.  B = 3 on 8 x 8
# images leaves the second image of the last tile past the batch.
FWD = [(2, 16, 16, 128, 256, 1), (3, 8, 8, 256, 512, 1), (3, 8, 8, 64, 128, 1), (3, 8, 8, 192, 64, 1),
       (2, 32, 32, 64, 320, 2), (2, 32, 32, 128, 256, 2)]


@pytest.mark.parametrize("B,H,W,cin,cout,stride", FWD)
def test_conv_forward_bias_rowvec_residual(B, H, W, cin, cout, stride):
    torch.manual_seed(10)
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = rand_w(cin, cout)
    bias = torch.randn(cout, device=dev) * 0.3
    rowvec = torch.randn(B, cout, device=dev) * 0.3
    res = torch.randn(B, H // stride, W // stride, cout, device=dev).bfloat16()
    y = ops.conv3x3_fwd(x, w, bias, rowvec, res, stride=stride)
    ran_tc()
    ref = conv_ref(x, w, stride) + bias + rowvec[:, None, None, :] + res.float()
    assert rel(y, ref) < BF16_TOL
    y2 = ops.conv3x3_fwd(x, w, bias, rowvec, res, stride=stride)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)


@pytest.mark.parametrize("cout", [256, 512])
def test_conv_forward_column_sums(cout):
    torch.manual_seed(11)
    B, H, cin = 2, 16, 128
    x = torch.randn(B, H, H, cin, device=dev).bfloat16()
    w = rand_w(cin, cout)
    cs = ops.ColStats(B, cout, dev)
    y = torch.empty(B, H, H, cout, device=dev, dtype=torch.bfloat16)
    ops.conv3x3_fwd(x, w, out=y, colstats=(cs, 0))
    ran_tc()
    assert rel(y, conv_ref(x, w)) < BF16_TOL
    assert rel(ops.groupnorm_stats_from_cols(cs, 32, 0, cout), ops.groupnorm_stats(y, 32)) < 1e-5


# (B, H, W, Cin = columns, Cout = K, stride): 256 columns -> BN 256; 768 columns -> three 256 tiles; 128 and
# 64 columns on 8 x 8; K = 192 at 64 columns -> 27 K chunks; stride 2 (four parity launches).
DGRAD = [(2, 16, 16, 256, 128, 1), (2, 16, 16, 768, 64, 1), (3, 8, 8, 128, 192, 1), (3, 8, 8, 64, 192, 1),
         (2, 32, 32, 256, 64, 2)]


@pytest.mark.parametrize("B,H,W,cin,cout,stride", DGRAD)
def test_conv_dgrad_accumulate(B, H, W, cin, cout, stride):
    torch.manual_seed(12)
    x = torch.zeros(B, H, W, cin, device=dev, requires_grad=True)
    w = rand_w(cin, cout)
    y = conv_ref(x, w, stride)
    dy = torch.randn_like(y).bfloat16()
    y.backward(dy.float())
    dx = torch.randn(B, H, W, cin, device=dev).bfloat16()
    prior = dx.float().clone()
    ops.conv3x3_dgrad(dy.contiguous(), w, dx, stride=stride, accumulate=True)
    ran_tc()
    assert rel(dx, prior + x.grad) < BF16_TOL
    dx1 = torch.zeros_like(dx)
    dx2 = torch.zeros_like(dx)
    ops.conv3x3_dgrad(dy.contiguous(), w, dx1, stride=stride)
    ops.conv3x3_dgrad(dy.contiguous(), w, dx2, stride=stride)
    torch.cuda.synchronize()
    assert torch.equal(dx1, dx2)


# (H, Cin = columns, Cout): BN 256 at 256 and 512 columns; 24 x 24 images for BN 128 and BN 64 (27 K chunks)
@pytest.mark.parametrize("H,cin,cout", [(16, 256, 64), (16, 512, 128), (24, 128, 64), (24, 64, 192)])
def test_dgrad_fused_groupnorm_backward(H, cin, cout):
    torch.manual_seed(13)
    B = 2
    dy = torch.randn(B, H, H, cout, device=dev).bfloat16()
    w = rand_w(cin, cout)
    x = torch.randn(B, H, H, cin, device=dev).bfloat16()
    ab = torch.randn(B, 2, cin, device=dev) * 0.5
    dz = torch.empty(B, H, H, cin, device=dev, dtype=torch.bfloat16)
    ws = ops.conv3x3_dgrad_gn(dy, w, dz, x, ab)
    ran_tc()
    xg = torch.zeros(B, H, H, cin, device=dev, requires_grad=True)
    conv_ref(xg, w).backward(dy.float())
    z = x.float() * ab[:, 0].view(B, 1, 1, cin) + ab[:, 1].view(B, 1, 1, cin)
    s = torch.sigmoid(z)
    assert rel(dz, xg.grad * s * (1 + z * (1 - s))) < 1e-2
    sums = ws.sum(0)                                   # [B][2][cin]: sum dz, sum dz * x per (image, channel)
    dzf = dz.float()
    assert rel(sums[:, 0], dzf.sum((1, 2))) < 1e-4
    assert rel(sums[:, 1], (dzf * x.float()).sum((1, 2))) < 1e-4


def test_conv1x1_odd_k_chunks_at_64_columns():
    torch.manual_seed(14)
    B, H, W, cin, cout = 3, 8, 8, 192, 64           # forward K = 192: three 64-deep chunks, BN 64
    x = torch.randn(B, H, W, cin, device=dev).bfloat16()
    w = (torch.randn(cin, cout, device=dev) / cin ** 0.5).bfloat16()
    bias = torch.randn(cout, device=dev) * 0.3
    y = ops.conv1x1_fwd(x, w, bias)
    ran_tc()
    assert rel(y, x.float() @ w.float() + bias) < BF16_TOL
    dy = torch.randn(B, H, W, cin, device=dev).bfloat16()   # data gradient 64 columns <- 192 (K = 192)
    w2 = (torch.randn(cout, cin, device=dev) / cin ** 0.5).bfloat16()
    dx = torch.zeros(B, H, W, cout, device=dev, dtype=torch.bfloat16)
    ops.conv1x1_dgrad(dy, w2, dx)
    ran_tc()
    assert rel(dx, dy.float() @ w2.float().t()) < BF16_TOL


# (B, H, Cin = rows, Cout = columns): BN 256 with tap pairing (Cin = 64), BN 128, BN 64 with a half-empty
# second row block (Cin = 192); all stride 2, split-K with f32 reductions.
@pytest.mark.parametrize("B,H,cin,cout", [(2, 32, 64, 256), (2, 32, 128, 128), (4, 16, 192, 64)])
def test_conv_wgrad_stride2(B, H, cin, cout):
    torch.manual_seed(15)
    x = torch.randn(B, H, H, cin, device=dev).bfloat16()
    w = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).requires_grad_(True)
    y = conv_ref(x, w, 2)
    dy = torch.randn_like(y).bfloat16()
    y.backward(dy.float())
    dw = torch.zeros(3, 3, cin, cout, device=dev)
    ops.conv3x3_wgrad(x, dy.contiguous(), dw, stride=2)
    ran_tc()
    assert rel(dw, w.grad) < F32_TOL


@pytest.mark.parametrize("M,N,K", [(300, 96, 192), (300, 288, 320), (77, 32, 64)])
def test_gemm_kmn_bf16_half_chunks(M, N, K):
    # N % 64 == 32: the last 64-column chunk has no second half; 288 columns leave the last 128 tile mostly empty
    torch.manual_seed(16)
    A = torch.randn(M, K, device=dev).bfloat16()
    Bm = torch.randn(K, N, device=dev).bfloat16()
    bias = torch.randn(N, device=dev)
    res = torch.randn(M, N, device=dev).bfloat16()
    D = ops.linear_fwd(A, Bm, bias=bias, res=res)
    ran_tc()
    assert rel(D, A.float() @ Bm.float() + bias + res.float()) < BF16_TOL


@pytest.mark.parametrize("M,N,K", [(300, 64, 192), (300, 256, 320), (129, 768, 128)])
def test_gemm_kk_f32(M, N, K):
    torch.manual_seed(17)
    A = torch.randn(M, K, device=dev).bfloat16()
    Bm = torch.randn(N, K, device=dev).bfloat16()
    D = torch.empty(M, N, device=dev)
    ops.gemm(GEMM_KK, A, Bm, D, M, N, K, K, K, N, alpha=0.5)
    ran_tc()
    assert rel(D, 0.5 * A.float() @ Bm.float().t()) < F32_TOL
    D2 = torch.empty_like(D)
    ops.gemm(GEMM_KK, A, Bm, D2, M, N, K, K, K, N, alpha=0.5)
    torch.cuda.synchronize()
    assert torch.equal(D, D2)


@pytest.mark.parametrize("M,N,K", [(192, 96, 1000), (64, 256, 4096), (128, 128, 640)])
def test_gemm_mnmn_f32_split_k(M, N, K):
    torch.manual_seed(18)
    A = torch.randn(K, M, device=dev).bfloat16()
    Bm = torch.randn(K, N, device=dev).bfloat16()
    D = torch.zeros(M, N, device=dev)
    ops.gemm(GEMM_MNMN, A, Bm, D, M, N, K, M, N, N, atomic=True, reduce_batch=True)
    ran_tc()
    assert rel(D, A.float().t() @ Bm.float()) < F32_TOL
    D1 = torch.zeros(M, N, device=dev)          # plain f32 stores (one split)
    ops.gemm(GEMM_MNMN, A, Bm, D1, M, N, K, M, N, N)
    ran_tc()
    assert rel(D1, A.float().t() @ Bm.float()) < F32_TOL
    D2 = torch.zeros(M, N, device=dev)
    ops.gemm(GEMM_MNMN, A, Bm, D2, M, N, K, M, N, N)
    torch.cuda.synchronize()
    assert torch.equal(D1, D2)
