"""fdx_ssm.cu's kernels element by element against float64: the discretisation and its backward, the sequence-parallel
scan and adjoint scan in both directions, and the row permutation.  Lengths cover one token, one chunk +- 1 and 4096
tokens (256^2 at patch 4); state counts 16, 64 and 128, with the slowest decay (n = 0, dt = 0.001, |Abar| ~ 0.9995) and
the fastest (n = N - 1, dt = 0.1) present in every case.  Every kernel is also run twice and compared bit for bit."""
import math

import pytest
import torch

from flaxdiff_b200 import ops

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
F64 = torch.float64


def _leaves(N, F, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(N, dtype=F64)
    log_dt = torch.empty(N, dtype=F64).uniform_(math.log(0.001), math.log(0.1), generator=g)
    log_dt[0], log_dt[-1] = math.log(0.001), math.log(0.1)
    P = {"log_A_real": torch.log(n + 0.5), "A_imag": math.pi * n, "log_dt": log_dt,
         "B_re": torch.randn(N, F, generator=g, dtype=F64) / N ** 0.5,
         "B_im": torch.randn(N, F, generator=g, dtype=F64) / N ** 0.5,
         "C_re": torch.randn(F, N, generator=g, dtype=F64) / F ** 0.5,
         "C_im": torch.randn(F, N, generator=g, dtype=F64) / F ** 0.5}
    return {k: v.float() for k, v in P.items()}


def _disc64(P):
    p = {k: v.double() for k, v in P.items()}
    dt = p["log_dt"].exp()
    A = torch.complex(-p["log_A_real"].exp(), p["A_imag"])
    Ab = torch.exp(A * dt)
    Bb = ((Ab - 1) / (A + 1e-8))[:, None] * torch.complex(p["B_re"], p["B_im"])
    return A * dt, Ab, Bb


def _discretize(Ps, N, F):
    nd = len(Ps)
    wb = torch.empty((F, 2 * nd * N), dtype=torch.bfloat16, device=dev)
    adt = torch.empty(2 * nd * N, dtype=torch.float32, device=dev)
    wcs = []
    for d, P in enumerate(Ps):
        wc = torch.empty((2 * N, F), dtype=torch.bfloat16, device=dev)
        ops.ssm_discretize({k: v.to(dev) for k, v in P.items()}, N, F, wb, 2 * d * N, wc, adt)
        wcs.append(wc)
    return wb, wcs, adt


def _close(got, ref, tol):
    got, ref = got.double().cpu(), ref.double().cpu()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-30
    assert err <= tol * scale, (err, scale, tol)


@pytest.mark.parametrize("N,F", [(16, 64), (64, 768), (128, 256)])
def test_discretize_forward(N, F):
    Ps = [_leaves(N, F, 1), _leaves(N, F, 2)]
    wb, wcs, adt = _discretize(Ps, N, F)
    wb2, wcs2, adt2 = _discretize(Ps, N, F)
    assert torch.equal(wb, wb2) and torch.equal(adt, adt2) and all(torch.equal(a, b) for a, b in zip(wcs, wcs2))
    for d, P in enumerate(Ps):
        adt64, _, Bb = _disc64(P)
        c = 2 * d * N
        g = (Bb.abs() / torch.complex(P["B_re"].double(), P["B_im"].double()).abs().clamp_min(1e-30))[:, :1]
        # f32 rounding of g B relative to its terms |g| (|B_re| + |B_im|), where they cancel; bf16 rounding of the rest
        terms = g * (P["B_re"].double().abs() + P["B_im"].double().abs())
        for got, ref in ((wb[:, c:c + N].T, Bb.real), (wb[:, c + N:c + 2 * N].T, Bb.imag)):
            err = (got.double().cpu() - ref).abs()
            assert (err <= 2 ** -8 * ref.abs() + 2e-6 * terms).all(), (err / (ref.abs() + 1e-30)).max()
        assert torch.equal(wcs[d][:N].cpu(), P["C_re"].T.bfloat16())
        assert torch.equal(wcs[d][N:].cpu(), (-P["C_im"]).T.bfloat16())
        _close(adt[c:c + N], adt64.real, 1e-6)
        _close(adt[c + N:c + 2 * N] * math.pi, adt64.imag, 1e-6)


@pytest.mark.parametrize("N,F,parts", [(16, 64, 1), (64, 768, 37), (128, 256, 300)])
def test_discretize_backward(N, F, parts):
    P = _leaves(N, F, 3)
    g = torch.Generator().manual_seed(4)
    dwb = torch.randn(2 * N, F, generator=g)
    dwc = torch.randn(2 * N, F, generator=g)
    dab = torch.randn(parts, 2 * N, generator=g)
    dgb = torch.randn(parts, 2 * N, generator=g)
    outs = []
    for _ in range(2):
        G = {k: torch.zeros_like(v, device=dev) for k, v in P.items()}
        ops.ssm_discretize_bwd({k: v.to(dev) for k, v in P.items()}, G, N, F, dwb.to(dev), 0, dwc.to(dev),
                               dab.to(dev), dgb.to(dev))
        outs.append(G)
    assert all(torch.equal(outs[0][k], outs[1][k]) for k in P)
    # the kernel's contract: dAbar = sum of dab; d(g) = sum of dgb / conj(g) (dgb sums lambda conj(Bu), Bu = g u B^T);
    # dBbar = dwb reaches B only (g's share comes through dgb)
    Pd = {k: v.double().requires_grad_(True) for k, v in P.items()}
    _, Ab, _ = _disc64(Pd)
    A = torch.complex(-Pd["log_A_real"].exp(), Pd["A_imag"])
    gfun = (Ab - 1) / (A + 1e-8)
    K = torch.complex(dgb.double().sum(0)[:N], dgb.double().sum(0)[N:]) / gfun.detach().conj()
    Bfix = gfun.detach()[:, None] * torch.complex(Pd["B_re"], Pd["B_im"])
    S = dab.double().sum(0)
    loss = (S[:N] * Ab.real + S[N:] * Ab.imag).sum() + (K.real * gfun.real + K.imag * gfun.imag).sum() \
        + (dwb[:N].double() * Bfix.real).sum() + (dwb[N:].double() * Bfix.imag).sum() \
        + (dwc[:N].double() * Pd["C_re"].T).sum() - (dwc[N:].double() * Pd["C_im"].T).sum()
    loss.backward()
    for k in P:
        _close(outs[0][k], Pd[k].grad, 1e-5)


def _scan64(bu, adt, B, L, N, nd):
    """f64 states of the recurrence with Abar = exp(adt) (adt's imaginary part in half-turns)."""
    S2 = 2 * nd * N
    a = adt.double().cpu()
    x = bu.double().cpu().view(B, L, S2)
    out = torch.zeros_like(x)
    for d in range(nd):
        c = 2 * d * N
        Ab = torch.exp(torch.complex(a[c:c + N], a[c + N:c + 2 * N] * math.pi))
        u = torch.complex(x[..., c:c + N], x[..., c + N:c + 2 * N])
        if d == 1:
            u = u.flip(1)
        h = torch.zeros(B, N, dtype=torch.complex128)
        hs = []
        for t in range(L):
            h = Ab * h + u[:, t]
            hs.append(h)
        X = torch.stack(hs, 1)
        if d == 1:
            X = X.flip(1)
        out[..., c:c + N], out[..., c + N:c + 2 * N] = X.real, X.imag
    return out.view(B * L, S2)


def _adjoint64(dx, x, bu, adt, B, L, N, nd):
    """f64 lambda and the sums over (sample, token) of lambda_k conj(x_{k-1}) and lambda_k conj(bu_k) per state, from
    the f32 states x."""
    S2 = 2 * nd * N
    a = adt.double().cpu()
    g = dx.double().cpu().view(B, L, S2)
    xs = x.double().cpu().view(B, L, S2)
    bs = bu.double().cpu().view(B, L, S2)
    lam_out = torch.zeros_like(g)
    dab = torch.zeros(S2, dtype=F64)
    dgb = torch.zeros(S2, dtype=F64)
    for d in range(nd):
        c = 2 * d * N
        Ab = torch.exp(torch.complex(a[c:c + N], a[c + N:c + 2 * N] * math.pi))
        gg = torch.complex(g[..., c:c + N], g[..., c + N:c + 2 * N])
        xx = torch.complex(xs[..., c:c + N], xs[..., c + N:c + 2 * N])
        bb = torch.complex(bs[..., c:c + N], bs[..., c + N:c + 2 * N])
        if d == 1:
            gg, xx, bb = gg.flip(1), xx.flip(1), bb.flip(1)
        lam = torch.zeros(B, N, dtype=torch.complex128)
        lams = [None] * L
        for t in range(L - 1, -1, -1):
            lam = gg[:, t] + Ab.conj() * lam
            lams[t] = lam
        Lm = torch.stack(lams, 1)
        xprev = torch.cat([torch.zeros_like(xx[:, :1]), xx[:, :-1]], 1)
        s = (Lm * xprev.conj()).sum((0, 1))
        sg = (Lm * bb.conj()).sum((0, 1))
        dgb[c:c + N], dgb[c + N:c + 2 * N] = sg.real, sg.imag
        if d == 1:
            Lm = Lm.flip(1)
        lam_out[..., c:c + N], lam_out[..., c + N:c + 2 * N] = Lm.real, Lm.imag
        dab[c:c + N], dab[c + N:c + 2 * N] = s.real, s.imag
    return lam_out.view(B * L, S2), dab, dgb


SCANS = [  # B, L, N, ndir, chunk
    (2, 1, 16, 2, 8), (2, 63, 16, 2, 64), (3, 65, 64, 2, 64), (2, 64, 128, 1, 64), (1, 4096, 64, 2, 64),
    (1, 4096, 128, 1, 100), (2, 4096, 16, 2, 512), (4, 1000, 64, 2, None),
]


@pytest.mark.parametrize("B,L,N,nd,chunk", SCANS)
def test_scan_and_adjoint(B, L, N, nd, chunk):
    F = 64
    chunk = chunk or ops.ssm_chunk(B, L, nd * N, dev)
    Ps = [_leaves(N, F, 5 + d) for d in range(nd)]
    _, _, adt = _discretize(Ps, N, F)
    S2 = 2 * nd * N
    g = torch.Generator(device=dev).manual_seed(6)
    bu = torch.randn(B * L, S2, generator=g, device=dev)
    ref = _scan64(bu, adt, B, L, N, nd)
    x, x16 = ops.ssm_scan(bu, adt, B, N, nd, chunk)
    x_b, x16_b = ops.ssm_scan(bu, adt, B, N, nd, chunk)
    x_in = bu.clone()
    ops.ssm_scan(x_in, adt, B, N, nd, chunk, out=x_in)             # in place
    assert torch.equal(x, x_b) and torch.equal(x16, x16_b) and torch.equal(x, x_in)
    assert torch.equal(x16, x.bfloat16())
    _close(x, ref, 2e-5)
    dx = torch.randn(B * L, S2, generator=g, device=dev)
    lam16, dab, dgb = ops.ssm_scan_bwd(dx, x, bu, adt, B, N, nd, chunk)
    lam16_b, dab_b, dgb_b = ops.ssm_scan_bwd(dx, x, bu, adt, B, N, nd, chunk)
    assert torch.equal(lam16, lam16_b) and torch.equal(dab, dab_b) and torch.equal(dgb, dgb_b)
    lam_ref, dab_ref, dgb_ref = _adjoint64(dx, x, bu, adt, B, L, N, nd)
    _close(lam16, lam_ref, 2 ** -8 + 2e-5)
    _close(dab.double().sum(0), dab_ref, 1e-4)
    _close(dgb.double().sum(0), dgb_ref, 1e-4)


@pytest.mark.parametrize("dtype,width", [(torch.bfloat16, 56), (torch.float32, 32), (torch.bfloat16, 768)])
def test_permute_rows(dtype, width):
    B, L = 3, 24
    idx = torch.randperm(L, generator=torch.Generator().manual_seed(7)).to(torch.int32)
    src = torch.randn(B * L, width, device=dev).to(dtype)
    got = ops.permute_rows(src, idx.to(dev))
    want = src.view(B, L, width)[:, idx.long().to(dev)].reshape(B * L, width)
    assert torch.equal(got, want)
