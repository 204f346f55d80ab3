"""fdx_gemm_cat, the GEMM whose A operand comes from two row matrices: bit for bit fdx_gemm on the materialised
torch.cat([A0, A1], 1) - at K0 / K1 in {64, 768, 1536}, N in {32, 768, 3072}, M from one row to SimpleUDiT-B/2's
262144 tokens, with bias and residual on and off and bf16 and f32 output - bitwise repeatable, and the split-weight
float32 projection [x | x] x [W_hi; W_lo] against float64."""
import itertools

import pytest
import torch

from flaxdiff_b200 import ops
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
KS = (64, 768, 1536)
NS = (32, 768, 3072)


def _both(mode, A0, A1, Bm, N, out_dtype, bias, res):
    M, K0 = A0.shape
    K = K0 + A1.shape[1]
    b_ld = K if mode == GEMM_KK else N
    r_ld = N if res is not None else 0
    want = torch.empty((M, N), dtype=out_dtype, device=dev)
    ops.gemm(mode, torch.cat([A0, A1], 1), Bm, want, M, N, K, K, b_ld, N, bias=bias, res=res, r_ld=r_ld)
    got = torch.full((M, N), float("nan"), dtype=out_dtype, device=dev)
    ops.gemm_cat(mode, A0, A1, Bm, got, M, N, K, K0, K0, A1.shape[1], b_ld, N, bias=bias, res=res, r_ld=r_ld)
    return got, want


@pytest.mark.parametrize("M", [1, 127, 129, 8191, 262144])
def test_bitwise_equal_to_gemm_on_the_concatenation(M):
    g = torch.Generator(device=dev).manual_seed(M)
    A = {k: torch.randn(M, k, generator=g, device=dev).bfloat16() for k in KS}
    A1 = {k: torch.randn(M, k, generator=g, device=dev).bfloat16() for k in KS}
    bad = []
    for K0, K1 in itertools.product(KS, KS):
        K = K0 + K1
        for N in NS:
            W = (torch.randn(K, N, generator=g, device=dev) / K ** 0.5).bfloat16()
            bias = torch.randn(N, generator=g, device=dev)
            res = torch.randn(M, N, generator=g, device=dev).bfloat16()
            mode = GEMM_KMN if (K0 + N) % 2 == 0 else GEMM_KK
            Bm = W if mode == GEMM_KMN else W.t().contiguous()
            for out_dtype, b, r in itertools.product((torch.bfloat16, torch.float32), (None, bias), (None, res)):
                got, want = _both(mode, A[K0], A1[K1], Bm, N, out_dtype, b, r)
                if not torch.equal(got, want):
                    bad.append((K0, K1, N, mode, str(out_dtype), b is not None, r is not None,
                                (got.float() - want.float()).abs().max().item()))
            del W, res
    assert not bad, bad[:10]


@pytest.mark.parametrize("mode", [GEMM_KK, GEMM_KMN])
def test_both_modes_at_the_up_dense_shape_and_bitwise_repeats(mode):
    g = torch.Generator(device=dev).manual_seed(7)
    M, F = 8192, 768
    x, skip = (torch.randn(M, F, generator=g, device=dev).bfloat16() for _ in range(2))
    W = (torch.randn(2 * F, F, generator=g, device=dev) / (2 * F) ** 0.5).bfloat16()
    Bm = W if mode == GEMM_KMN else W.t().contiguous()
    bias = torch.randn(F, generator=g, device=dev)
    got, want = _both(mode, x, skip, Bm, F, torch.bfloat16, bias, None)
    assert torch.equal(got, want)
    again, _ = _both(mode, x, skip, Bm, F, torch.bfloat16, bias, None)
    assert torch.equal(got, again)
    # and it is the Dense over [x, skip]
    ref = torch.cat([x, skip], 1).double() @ W.double() + bias.double()
    assert ((got.double() - ref).abs() / (ref.abs() + 1e-2)).max().item() < 2e-2


def test_strided_sources():
    """A0 and A1 as column slices of wider buffers (row stride > width), as the model never needs but the entry point
    allows."""
    g = torch.Generator(device=dev).manual_seed(3)
    M, K0, K1, N = 1000, 128, 192, 96
    buf0 = torch.randn(M, K0 + 64, generator=g, device=dev).bfloat16()
    buf1 = torch.randn(M, K1 + 128, generator=g, device=dev).bfloat16()
    A0, A1 = buf0[:, 64:], buf1[:, :K1]
    W = torch.randn(K0 + K1, N, generator=g, device=dev).bfloat16()
    want = torch.empty((M, N), dtype=torch.float32, device=dev)
    ops.gemm(GEMM_KMN, torch.cat([A0, A1], 1), W, want, M, N, K0 + K1, K0 + K1, N, N)
    got = torch.empty_like(want)
    ops.gemm_cat(GEMM_KMN, A0, A1, W, got, M, N, K0 + K1, K0, buf0.stride(0), buf1.stride(0), N, N)
    assert torch.equal(got, want)


def _split_case(positive: bool):
    """x bf16 [M, F]; W f32 with bits below bf16: W = a + a * u * 2^-10 (a bf16, u in [0.5, 1]) rounds to a, so W_hi
    alone misses a 2^-10-relative part of every weight.  With positive x and W that error adds up over K."""
    g = torch.Generator(device=dev).manual_seed(11 + positive)
    M, F, N = 4096, 768, 32
    x = torch.randn(M, F, generator=g, device=dev)
    x = (x.abs() if positive else x).bfloat16()
    a = torch.randn(F, N, generator=g, device=dev)
    a = (a.abs() if positive else a).bfloat16().float()
    u = 0.5 + 0.5 * torch.rand(F, N, generator=g, device=dev)
    W = a + a * u * 2.0 ** -10
    w_hi = ops.cast_f32_bf16(W.contiguous())
    w_lo = ops.cast_f32_bf16((W - w_hi.float()).contiguous())
    ref = x.double() @ W.double()
    scale = x.double().abs() @ W.double().abs()
    return x, W, w_hi, w_lo, ref, scale


@pytest.mark.parametrize("positive", [True, False])
def test_split_weight_projection_reproduces_float32(positive):
    x, W, w_hi, w_lo, ref, scale = _split_case(positive)
    M, F = x.shape
    N = W.shape[1]
    y = torch.empty((M, N), dtype=torch.float32, device=dev)
    ops.gemm_cat(GEMM_KMN, x, x, torch.cat([w_hi, w_lo], 0), y, M, N, 2 * F, F, F, F, N, N)
    err = ((y.double() - ref).abs() / scale).max().item()
    assert err <= 1e-4, err
    if positive:
        # W_hi alone misses the part below bf16: the same bound fails, so the check tells the two apart
        y1 = torch.empty_like(y)
        ops.gemm(GEMM_KMN, x, w_hi, y1, M, N, F, F, N, N)
        err1 = ((y1.double() - ref).abs() / scale).max().item()
        assert err1 > 1e-4, err1
