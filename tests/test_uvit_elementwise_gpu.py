"""UViT's kernels (fdx_uvit.cu) element by element against float64, through the C ABI: the sequence assembly forward
(bit for bit) and backward (the split rows bit for bit, the position gradient within a derived bound and bitwise on
rerun), the head's LayerNorm(64) + swish / mish forward and backward, and the 6-channel im2col (bit for bit).  Outputs
are NaN-prefilled and guarded by sentinel rows, so a row that is skipped or written past its end shows."""
import math

import pytest
import torch

from flaxdiff_b200 import ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
BF = torch.bfloat16


def _guarded(rows, cols, dtype):
    """(buffer with one sentinel row either side, NaN-filled interior view)."""
    buf = torch.full((rows + 2, cols), 7.0, dtype=dtype, device=dev)
    buf[1:-1] = float("nan")
    return buf, buf[1:-1]


@pytest.mark.parametrize("B,N,T,F", [(1, 1, 0, 64), (5, 37, 77, 768), (256, 256, 0, 64), (1, 4096, 77, 1536),
                                     (5, 256, 77, 1024), (256, 37, 77, 128)])
def test_assembly_forward_is_exact(B, N, T, F):
    g = torch.Generator(device=dev).manual_seed(B * 7 + N)
    patch = torch.randn(B * N, F, generator=g, device=dev).to(BF)
    pos = torch.randn(N + 3, F, generator=g, device=dev)
    tim = torch.randn(B, F, generator=g, device=dev).to(BF)
    txt = torch.randn(B * T, F, generator=g, device=dev).to(BF) if T else None
    L = N + 1 + T
    buf, out = _guarded(B * L, F, BF)
    from flaxdiff_b200._lib import check, load, ptr, stream_ptr
    check(load().fdx_uvit_assemble_fwd(ptr(patch), ptr(pos), ptr(tim), ptr(txt), B, N, T, F, ptr(out),
                                       stream_ptr()))
    ref = torch.empty(B, L, F, dtype=torch.float64, device=dev)
    ref[:, :N] = patch.view(B, N, F).double() + pos[:N].double()
    ref[:, N] = tim.double()
    if T:
        ref[:, N + 1:] = txt.view(B, T, F).double()
    # f32(bf16) + f32 is exact in float64's rounding to f32 then bf16 except at double-rounding ties: compare with the
    # f32 sum rounded once to bf16, which is what the kernel computes
    ref16 = ref.clone()
    ref16[:, :N] = (patch.view(B, N, F).float() + pos[:N]).double()
    assert torch.equal(out.view(B, L, F), ref16.to(torch.float32).to(BF))
    assert (buf[0] == 7).all() and (buf[-1] == 7).all()
    assert torch.equal(ops.uvit_assemble_fwd(patch, pos, tim, txt, B, N, T), out)


@pytest.mark.parametrize("B,N,T,F", [(1, 1, 0, 64), (5, 37, 77, 768), (256, 256, 0, 64), (256, 1024, 0, 768),
                                     (3, 4096, 77, 128)])
def test_assembly_backward_split_and_position_gradient(B, N, T, F):
    g = torch.Generator(device=dev).manual_seed(B + N + F)
    L = N + 1 + T
    dx = torch.randn(B * L, F, generator=g, device=dev).to(BF)
    dpos0 = torch.randn(N, F, generator=g, device=dev)
    dpos = dpos0.clone()
    dpatch, dtime, dtext = ops.uvit_assemble_bwd(dx, B, N, T, dpos)
    d3 = dx.view(B, L, F)
    assert torch.equal(dpatch.view(B, N, F), d3[:, :N])
    assert torch.equal(dtime, d3[:, N].float())
    if T:
        assert torch.equal(dtext.view(B, T, F), d3[:, N + 1:])
    ref = dpos0.double() + d3[:, :N].double().sum(0)
    # f32 sums of B bf16 terms plus the initial value: each addition rounds by at most 2^-24 of the running sum,
    # which is at most sum |terms| (the derived bound)
    bound = (B + 1) * 2.0 ** -24 * (dpos0.double().abs() + d3[:, :N].double().abs().sum(0))
    assert ((dpos.double() - ref).abs() <= bound + 1e-30).all()
    again = dpos0.clone()
    ops.uvit_assemble_bwd(dx, B, N, T, again)
    assert torch.equal(again, dpos)


def _act(z, act):
    if act == ops.ACT_MISH:
        return z * torch.tanh(torch.nn.functional.softplus(z))
    return z * torch.sigmoid(z)


@pytest.mark.parametrize("act", [ops.ACT_SILU, ops.ACT_MISH])
@pytest.mark.parametrize("B,HW", [(1, 64), (256, 64), (4, 256), (1, 512)])
def test_head_norm_forward_and_backward(act, B, HW):
    g = torch.Generator(device=dev).manual_seed(B + HW + act)
    P = B * HW * HW
    x = (torch.rand(P, 64, generator=g, device=dev) * 200 - 100).to(BF)
    x[::3] = (torch.randn(x[::3].shape, generator=g, device=dev) * 0.5).to(BF)    # O(1) rows too
    gamma = torch.randn(64, generator=g, device=dev)
    beta = torch.randn(64, generator=g, device=dev)
    dy = torch.randn(P, 64, generator=g, device=dev).to(BF)
    eps = 1e-5
    y = ops.uvit_head_norm_fwd(x, gamma, beta, eps, act)
    xd = x.double().requires_grad_(True)
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    z = (xd - mu) / torch.sqrt(var + eps) * gamma.double() + beta.double()
    yr = _act(z, act)
    # bf16 output: half an ulp of the result plus the f32 arithmetic's slack (|y| 2^-20 and an absolute 1e-5)
    tol = yr.detach().abs() * (2.0 ** -8 + 2.0 ** -18) + 1e-5
    assert ((y.double() - yr.detach()).abs() <= tol).all()
    dgamma = torch.zeros(64, device=dev)
    dbeta = torch.zeros(64, device=dev)
    dx = ops.uvit_head_norm_bwd(x, dy, gamma, beta, eps, act, dgamma, dbeta)
    gx, = torch.autograd.grad(yr, xd, dy.double())
    zz = z.detach().requires_grad_(True)
    gz, = torch.autograd.grad(_act(zz, act), zz, dy.double())
    xh = (z.detach() - beta.double()) / gamma.double()
    rg, rb = (gz * xh).sum(0), gz.sum(0)
    scale = (gz.abs() * gamma.double().abs()).sum(-1, keepdim=True) / 64 * (1 / torch.sqrt(var.detach() + eps))
    assert ((dx.double() - gx).abs() <= gx.abs() * 2.0 ** -8 + 2e-3 * scale + 1e-6).all()
    s = (gz.abs() * (1 + xh.abs())).sum(0)
    assert ((dgamma.double() - rg).abs() <= 1e-4 * s + 1e-6).all()
    assert ((dbeta.double() - rb).abs() <= 1e-4 * s + 1e-6).all()
    dg2, db2 = torch.zeros(64, device=dev), torch.zeros(64, device=dev)
    assert torch.equal(ops.uvit_head_norm_bwd(x, dy, gamma, beta, eps, act, dg2, db2), dx)
    assert torch.equal(dg2, dgamma) and torch.equal(db2, dbeta)


@pytest.mark.parametrize("f32_0,f32_1", [(False, True), (True, False), (True, True), (False, False)])
@pytest.mark.parametrize("n,h,w", [(1, 1, 1), (2, 7, 5), (3, 64, 64)])
def test_im2col_c6_is_exact(f32_0, f32_1, n, h, w):
    g = torch.Generator(device=dev).manual_seed(n * h + w)
    a = torch.randn(n, h, w, 3, generator=g, device=dev)
    b = torch.randn(n, h, w, 3, generator=g, device=dev)
    a = a if f32_0 else a.to(BF)
    b = b if f32_1 else b.to(BF)
    col = ops.im2col3_c6(a, b)
    ref = torch.zeros(n, h, w, 64, dtype=BF, device=dev)
    pa = torch.nn.functional.pad(a.to(BF).permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    pb = torch.nn.functional.pad(b.to(BF).permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    for t in range(9):
        ky, kx = t // 3, t % 3
        ref[..., t * 3:t * 3 + 3] = pa[:, ky:ky + h, kx:kx + w]
        ref[..., 32 + t * 3:32 + t * 3 + 3] = pb[:, ky:ky + h, kx:kx + w]
    assert torch.equal(col.view(n, h, w, 64), ref)
    assert math.isfinite(col.float().sum().item())
