"""Float64 references of the memory-bound kernels (GroupNorm, RMSNorm, GEGLU, column sums, nearest 2x upsample)
and of the fused attention, and an element-wise comparator whose tolerance is derived, element by element, from the kernels' arithmetic.

Every reference takes the same bf16 values the kernel reads (as float64 tensors, on any device) and returns the
exact result together with `delta`: a first-order bound on how far the kernel's f32 arithmetic can be from it
before the output is stored.  The backwards are written in closed form (no autograd), so they run in float64 on
the GPU at N = 256.

Tolerance model (used by every element-wise test):
  * bf16 output, got = bf16(v) with |v - ref| <= delta:
        |got - ref| <= ulp_bf16(ref) + (1 + 2^-8) * delta                                           (k = 1)
    Round to nearest gives |bf16(v) - v| <= ulp(v)/2 <= 2^-8 |v| <= 2^-8 (|ref| + delta), and 2^-8 |ref| < ulp(ref)
    (bf16 has 8 significant bits).  One ulp is the output rounding; nothing else is allowed for free.
  * f32 output: |got - ref| <= 2^-24 (|ref| + delta) + delta.
  * delta collects the known error sources, each bounded where it arises:
      - f32 sums:  |fl(sum t) - sum t| <= gamma(D) * sum |t|, D the longest chain of dependent additions
        (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 4.4), gamma(D) = D u / (1 - D u),
        u = 2^-24.  D is counted from the kernel's loop structure where it is stated below, and otherwise taken
        as the number of terms, which bounds every summation order.
      - tanh.approx.f32 (f2_tanh in fdx_common.cuh, gelu_tanh_f in fdx_geglu.cu): relative error at most
        2^-10.987 (PTX ISA, tanh); TANH below rounds that up to 2^-10.9.  SiLU is h (1 + tanh h) with h = z/2, so
        its error is |h tanh h| TANH, about |h| 2^-11 for z << 0 where the output itself is near 0.
      - rsqrtf: at most 2 ulp (CUDA C Programming Guide, Mathematical Functions), i.e. 4u relative.
      - individual f32 roundings: u relative each; the count per formula is stated where it is used.
      - the statistics a normalisation divides by: their relative error propagates through mean / rstd.
    These are per-element bounds: the terms that involve a whole group (GroupNorm) or pixel (RMSNorm) are
    means over that unit, i.e. epsilon * s with s the unit's scale.  Constants come from this derivation; if a
    kernel exceeds its bound, that is a finding to explain, not a reason to widen the bound.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as Fnn

U32 = 2.0 ** -24             # unit roundoff of f32
U_BF16 = 2.0 ** -8           # unit roundoff of bf16 (8 significant bits)
TANH = 2.0 ** -10.9          # relative error bound of tanh.approx.f32 (documented 2^-10.987)
RSQRT = 4 * U32              # rsqrtf: 2 ulp of the result
# bf16 x bf16 products are exact in f32; the tensor cores may add with truncation instead of rounding, so every
# addition of the convolution's K-long accumulation counts 2u.
TC_ADD = 2 * U32


def gamma(depth) -> float:
    d = float(depth) * U32
    return d / (1.0 - d)


def ulp_bf16(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |ref| (2^(e-7) for |ref| in [2^e, 2^(e+1)); constant below the smallest normal)."""
    a = ref.abs().to(torch.float64).clamp_min(2.0 ** -126)
    _, e = torch.frexp(a)                     # a = m 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(a), (e - 8).to(torch.int32))


def bf16_bound(ref: torch.Tensor, delta) -> torch.Tensor:
    return ulp_bf16(ref) + (1 + U_BF16) * delta


def f32_bound(ref: torch.Tensor, delta) -> torch.Tensor:
    return U32 * (ref.abs() + delta) + delta


def assert_elementwise(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> float:
    """Fail if any element of `got` is not finite or lies outside |got - ref| <= bound.  Returns the worst
    |got - ref| / bound, so that callers can report how close a kernel comes to its bound."""
    g = got.detach().to(torch.float64)
    r = ref.detach().to(device=g.device, dtype=torch.float64)
    b = torch.as_tensor(bound, dtype=torch.float64, device=g.device).expand_as(r)
    assert g.shape == r.shape, (what, tuple(g.shape), tuple(r.shape))
    err = (g - r).abs()
    frac = torch.where(err == 0, torch.zeros_like(err), err / b)     # an exact element is 0 x even a zero bound
    bad = ~(err <= b) | ~torch.isfinite(g)            # NaN compares false: an unwritten NaN-prefilled element fails
    nbad = int(bad.sum())
    worst = torch.where(torch.isfinite(frac), frac, torch.full_like(frac, math.inf))
    if nbad:
        i = int(torch.argmax(torch.where(bad, worst, torch.zeros_like(worst))))
    else:
        i = int(torch.argmax(worst))
    if g.numel() == 0:
        return 0.0
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), tuple(g.shape))) if g.dim() else ()
    gi, ri, bi = g.reshape(-1)[i].item(), r.reshape(-1)[i].item(), b.reshape(-1)[i].item()
    ei = abs(gi - ri) if math.isfinite(gi) else math.inf
    ulps = ei / ulp_bf16(torch.tensor(ri, dtype=torch.float64)).item()
    assert nbad == 0, (f"{what}: {nbad} of {g.numel()} elements outside the bound; worst at {idx}: got {gi!r}, "
                       f"ref {ri!r}, |err| = {ei:.4g} = {ulps:.3g} bf16 ulp = {ei / bi:.3g} x its bound {bi:.4g}")
    return float(worst.max()) if worst.numel() else 0.0


# ----------------------------------------------------------------------------------------------- GroupNorm
def _g(t: torch.Tensor, G: int) -> torch.Tensor:
    """(N, H, W, C) -> (N, HW, G, C/G)."""
    return t.reshape(t.shape[0], -1, G, t.shape[-1] // G)


def _gmean(t: torch.Tensor) -> torch.Tensor:
    """Mean over the (pixel, channel-in-group) unit of a grouped tensor, kept for broadcasting."""
    return t.mean((1, 3), keepdim=True)


def gn_stats_ref(x: torch.Tensor, G: int):
    """fdx_groupnorm_stats: [N][G] (sum, sum of squares) -> (value, delta).  gn_stats_kernel gives each thread
    ceil(HW C/(8 G) / 256) 16-byte vectors of 8 serial additions, then a 5-level warp tree and the 8 warps in
    order: D = 8 ceil(HW C / (2048 G)) + 13.  bf16 squares are exact in f32."""
    xg = _g(x, G)
    n_items = xg.shape[1] * xg.shape[3] // 8
    D = 8 * math.ceil(n_items / 256) + 13
    val = torch.stack([xg.sum((1, 3)), (xg * xg).sum((1, 3))], -1)
    delta = gamma(D) * torch.stack([xg.abs().sum((1, 3)), (xg * xg).sum((1, 3))], -1)
    return val, delta


class GnFwd:
    """Closed-form GroupNorm (flax: f32 statistics, var = max(0, E[x^2] - E[x]^2), y = (x - mean) rstd gamma + beta)
    with optional SiLU, and the f32 error of the statistics the kernels derive from fdx_groupnorm_stats."""

    def __init__(self, x, gamma_, beta_, G: int, eps: float, silu: bool):
        self.G, self.silu, self.shape = G, silu, x.shape
        N, H, W, C = x.shape
        self.HW, self.cpg = H * W, C // G
        xg = _g(x, G)
        self.xg = xg
        self.gam = gamma_.reshape(1, 1, G, -1).to(torch.float64)
        self.bet = beta_.reshape(1, 1, G, -1).to(torch.float64)
        mu = _gmean(xg)
        ex2 = _gmean(xg * xg)
        var = (ex2 - mu * mu).clamp_min(0)
        self.mu, self.r = mu, 1.0 / torch.sqrt(var + eps)
        self.xh = (xg - mu) * self.r
        self.z = self.gam * self.xh + self.bet
        # statistics: mean = s/cnt (1 rounding), var = q/cnt - mean^2 (3 roundings), rstd (2 ulp):
        #   dmu <= (D+1) u mean|x|,   drstd/rstd <= (D+3) u (E[x^2] + mean^2) / (var + eps) + 5u
        # D covers both producers of the sums: gn_stats_kernel (gn_stats_ref) and the per-channel column sums
        # of fdx_groupnorm_apply_cols (each rounded once to f32, then 4 slots x ceil(cpg/32) per lane and a
        # 5-level warp tree)
        D = max(8 * math.ceil(self.HW * self.cpg / 8 / 256) + 13, 4 * math.ceil(self.cpg / 32) + 6)
        self.dmu = gamma(D + 1) * _gmean(xg.abs())
        self.rho_r = gamma(D + 3) * (ex2 + mu * mu) / (var + eps) + RSQRT + U32
        self.dxh = self.r * ((xg - mu).abs() * self.rho_r + self.dmu)      # error of the kernel's normalised x
        # z = fma(x, a, b) with a = rstd gamma and b = beta - mean a: 3 roundings on |a|(|x| + |mean|) + |beta|
        self.dz = self.gam.abs() * self.dxh + 3 * U32 * (self.gam.abs() * self.r * (xg.abs() + mu.abs()) +
                                                         self.bet.abs())
        h = 0.5 * self.z
        self.h, self.t = h, torch.tanh(h)

    def forward(self):
        """-> (y, delta) as (N, H, W, C).  y = h (1 + tanh h) is one fma on the approximate tanh."""
        if not self.silu:
            return self.z.reshape(self.shape), self.dz.reshape(self.shape)
        y = self.h * (1 + self.t)
        sig = 0.5 * (1 + self.t)
        dsilu = sig * (1 + self.h * (1 - self.t))
        delta = dsilu.abs() * self.dz + (self.h * self.t).abs() * TANH + U32 * y.abs()
        return y.reshape(self.shape), delta.reshape(self.shape)


def gn_forward_ref(x, gamma_, beta_, G, eps, silu):
    return GnFwd(x, gamma_, beta_, G, eps, silu).forward()


def gn_backward_ref(x, dy, gamma_, beta_, G, eps, silu, dy_delta=None):
    """Closed-form GroupNorm(+SiLU) backward -> dict of (value, delta) for dx, dgamma, dbeta and the per-image /
    total column sums of dx.  `dy_delta` is a per-element bound on the error of the dy the kernel sees (the fused
    path's convolution data gradient and its bf16 rounding).

        dz = dy silu'(z),  g = gamma dz,  dx = rstd (g - mean_g(g) - xhat mean_g(g xhat))
        dbeta = sum_{n,p} dz,  dgamma = sum_{n,p} dz xhat
    """
    f = GnFwd(x, gamma_, beta_, G, eps, silu)
    N = x.shape[0]
    dyg = _g(dy, G)
    gam_a, r = f.gam.abs(), f.r
    if silu:
        sig = 0.5 * (1 + f.t)
        dsilu = sig * (1 + f.h * (1 - f.t))
        dz = dyg * dsilu
        # silu'(z) = (1+t)/2 (1 + h(1-t)): d silu'/dt = 1/2 - h t, |silu''| <= 1/2, then 6 roundings on the
        # pair arithmetic (each <= u (1 + 2|h|) |dy|)
        e_dz = dyg.abs() * ((0.5 - f.h * f.t).abs() * f.t.abs() * TANH + 0.5 * f.dz + 6 * U32 * (1 + 2 * f.h.abs()))
    else:
        dsilu = torch.ones_like(dyg)
        dz = dyg
        e_dz = torch.zeros_like(dyg)
    if dy_delta is not None:
        e_dz = e_dz + dsilu.abs() * _g(dy_delta, G)
    g = f.gam * dz
    m1, m2 = _gmean(g), _gmean(g * f.xh)
    dx = r * (g - m1 - f.xh * m2)
    # the kernel forms x*c2 and c3 = mean*c2 - rstd*m1 separately: its absolute-value scale of xhat is
    # rstd (|x| + |mean|), plus the statistics' error
    xa = r * (f.xg.abs() + f.mu.abs()) + f.dxh
    ga = gam_a * dz.abs()
    # f32 sums of pass 1 (S0 = sum dz, S1 = sum dz x per image and channel, any arrangement: at most HW terms in
    # a chain plus the row / CTA / cluster / slot reductions), the group sums over cpg channels and the ~16
    # scalar roundings of c2, c3 and the two fmas
    rows = max(1, 256 // (x.shape[-1] // 8))
    gb = gamma(f.HW + 2 * rows + 2 * f.cpg + 80) + f.rho_r
    e_g = gam_a * e_dz
    d_dx = (r * (e_g + _gmean(e_g) + xa * _gmean(e_g * xa))                 # error of dz
            + r * (f.dxh * _gmean((g * f.xh).abs()) + f.xh.abs() * _gmean(ga * f.dxh))   # statistics
            + gb * r * (ga + _gmean(ga) + xa * _gmean(ga * xa)))            # f32 roundings and sums
    dx_abs = r * (ga + _gmean(ga) + xa * _gmean(ga * xa))
    out = {}
    shp = x.shape

    def ug(t):
        return t.reshape(shp)

    out["dx"] = (ug(dx), ug(d_dx))
    # dgamma / dbeta: per-image sums as above, then the sum over N images (atomics or the finalize kernel)
    gr = gamma(f.HW + 2 * rows + N + 128)
    out["dbeta"] = (dz.sum((0, 1)).reshape(-1), (e_dz.sum((0, 1)) + gr * dz.abs().sum((0, 1))).reshape(-1))
    out["dgamma"] = ((dz * f.xh).sum((0, 1)).reshape(-1),
                     (e_dz * xa + dz.abs() * f.dxh).sum((0, 1)).reshape(-1) +
                     ((gr + f.rho_r) * dz.abs() * xa).sum((0, 1)).reshape(-1))
    # column sums of dx before any addend and before the bf16 rounding
    ci = dx.sum(1).reshape(N, -1)
    d_ci = (d_dx.sum(1) + gamma(f.HW + 2 * rows + 64) * dx_abs.sum(1)).reshape(N, -1)
    out["csum_img"] = (ci, d_ci)
    out["csum_tot"] = (ci.sum(0), d_ci.sum(0) + gamma(N + 64) * (dx_abs.sum(1).reshape(N, -1)).sum(0))
    return out


# ----------------------------------------------------------------------------------------------- convolutions
# The convolution and GEMM engines (fdx_tc.cu, fdx_tct.cu, fdx_wgrad9.cu, fdx_upconv.cu, the 3-channel paths of
# ops.py).  Every reference returns (value, delta) with delta = depth TC_ADD mag: mag is the same operation on
# |inputs| (the sum of |terms| of each output), depth the longest chain of f32 additions the kernel makes:
#   * the K-long accumulation of one tile (9 Cin taps forward, taps x Cout data gradient, the pixels of one split
#     of a weight gradient), counted from the launch code below;
#   * EPI = 16 further roundings: the epilogue's alpha, bias, row vector, residual or prior.  A split-K reduction
#     adds one level per split (red.global.add / atomics in any order) and a prior that is accumulated onto, one.
# Where an operand is rounded to bf16 before the tensor cores read it (the packed sub-pixel weights, the master
# weights of the 3-channel convolutions, conv_out's loss gradient), delta has U_BF16 on that operand explicitly.
# The references run in float64 on the device, over chunks of `chunk` images.
EPI = 16


def _pads(stride: int, H: int, W: int):
    """flax SAME for a 3x3 kernel, low side (the high side is 1): (1, 1) at stride 1; at stride 2, 0 on even and
    1 on odd sizes (fdx_api_tc.cu)."""
    if stride == 1:
        return 1, 1
    return (0 if H % 2 == 0 else 1), (0 if W % 2 == 0 else 1)


def _conv(x, w_hwio, stride):
    """float64 3x3 SAME cross-correlation, NHWC x HWIO -> NHWC."""
    ph, pw = _pads(stride, x.shape[1], x.shape[2])
    xp = Fnn.pad(x.to(torch.float64).permute(0, 3, 1, 2), (pw, 1, ph, 1))
    return Fnn.conv2d(xp, w_hwio.to(torch.float64).permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def _dconv(dy, w_hwio, stride, H, W):
    """Adjoint of _conv onto an (H, W) input."""
    ph, pw = _pads(stride, H, W)
    d = dy.to(torch.float64).permute(0, 3, 1, 2)
    full = Fnn.conv_transpose2d(d, w_hwio.to(torch.float64).permute(3, 2, 0, 1), stride=stride)
    return full[:, :, ph:ph + H, pw:pw + W].permute(0, 2, 3, 1)


def _chunks(N, chunk):
    return [slice(i, min(N, i + chunk)) for i in range(0, N, chunk)]


def _plus(val, mag, *terms):
    """Add epilogue terms (bias, row vector, residual, prior; None skipped) to a value and its magnitude."""
    for t in terms:
        if t is not None:
            t = t.to(torch.float64)
            val, mag = val + t, mag + t.abs()
    return val, mag


def conv3x3_fwd_ref(x, w_hwio, stride: int = 1, bias=None, rowvec=None, res=None, chunk: int = 64):
    """fdx_conv3x3_fwd: y = conv(x, w) + bias + rowvec[n] + res, NHWC / HWIO.  One accumulator chains all nine
    taps: depth 9 Cin + EPI."""
    N = x.shape[0]
    val = torch.cat([_conv(x[s], w_hwio, stride) for s in _chunks(N, chunk)])
    mag = torch.cat([_conv(x[s].abs(), w_hwio.abs(), stride) for s in _chunks(N, chunk)])
    rv = None if rowvec is None else rowvec.reshape(N, 1, 1, -1)
    val, mag = _plus(val, mag, bias, rv, res)
    return val, (9 * x.shape[-1] + EPI) * TC_ADD * mag


def conv3x3_dgrad_ref(dy, w_hwio, stride: int = 1, prior=None, chunk: int = 64):
    """d/dx of a 3x3 SAME cross-correlation (HWIO weights), NHWC -> (value, delta of the tensor-core engine).
    Stride 1: one launch of K = 9 Cout.  Stride 2 (even input sizes): four output-parity launches with 4, 2, 2
    and 1 taps, the longest K = 4 Cout.  `prior`: the bf16 dx that accumulate=True adds to."""
    N, Ho, Wo, Cout = dy.shape
    H, W = Ho * stride, Wo * stride
    val = torch.cat([_dconv(dy[s], w_hwio, stride, H, W) for s in _chunks(N, chunk)])
    mag = torch.cat([_dconv(dy[s].abs(), w_hwio.abs(), stride, H, W) for s in _chunks(N, chunk)])
    val, mag = _plus(val, mag, prior)
    K = (9 if stride == 1 else 4) * Cout
    return val, (K + EPI) * TC_ADD * mag


def _wgrad(x, dy, stride, absolute, chunk):
    """sum over images and output pixels of x[n, s oy + ky - ph, s ox + kx - pw, ci] dy[n, oy, ox, co]."""
    N, Ho, Wo, Co = dy.shape
    Ci = x.shape[-1]
    ph, pw = _pads(stride, x.shape[1], x.shape[2])
    out = torch.zeros(3, 3, Ci, Co, dtype=torch.float64, device=dy.device)
    for s in _chunks(N, chunk):
        xs, d = x[s].to(torch.float64), dy[s].to(torch.float64).reshape(-1, Co)
        if absolute:
            xs, d = xs.abs(), d.abs()
        xp = Fnn.pad(xs, (0, 0, pw, 1, ph, 1))
        for ky in range(3):
            for kx in range(3):
                tap = xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
                out[ky, kx] += tap.reshape(-1, Ci).T @ d
    return out


def conv3x3_wgrad_ref(x, dy, depth: int, stride: int = 1, prior=None, chunk: int = 16):
    """fdx_conv3x3_wgrad: dw (f32 HWIO) = prior + sum_pixels x (shifted by the tap) dy.  `depth` from
    wgrad9_depth or mnmn_depth (it includes the prior)."""
    val, mag = _plus(_wgrad(x, dy, stride, False, chunk), _wgrad(x, dy, stride, True, chunk), prior)
    return val, depth * TC_ADD * mag


def split_count(sms: int, base_tiles: int, kblocks: int) -> int:
    """The wave-aware split-K count of fdx_tc.cu (TC_MNMN) and fdx_wgrad9.cu: the split whose tile total fills
    w = 1..4 waves of `sms` SMs best, more waves only for > 3 % more fill; at most one split per pixel block."""
    best, splits = -1.0, 1
    for w in range(1, 5):
        sp = min(max(1, (sms * w) // base_tiles), kblocks)
        tiles = base_tiles * sp
        eff = tiles / (math.ceil(tiles / sms) * sms)
        if eff > best + 0.03:
            best, splits = eff, sp
    return min(splits, kblocks)


def wgrad9_depth(N: int, H: int, W: int, Cin: int, Cout: int, sms: int) -> int:
    """fdx_wgrad9_launch: 64-pixel blocks (TW = 16 for W >= 16, else 8), split over the pixel blocks; each split
    chains 64 products per block, then one red.global.add per split onto the prior."""
    TW = 16 if W >= 16 else 8
    kblocks = (W // TW) * (H // (64 // TW)) * N
    splits = split_count(sms, math.ceil(Cin / 64) * math.ceil(Cout / 64), kblocks)
    return 64 * math.ceil(kblocks / splits) + splits + 1


def _pow2_floor(v: int) -> int:
    return 1 << (max(1, v).bit_length() - 1)


def tc_bn(ncols: int) -> int:
    """fdx_tc_launch's column tile: the first of 256 / 128 / 64 minimising ceil(ncols / bn) (bn + 64)."""
    return min((256, 128, 64), key=lambda bn: math.ceil(ncols / bn) * (bn + 64))


def mnmn_depth(W: int, H: int, N: int, M: int, Ncols: int, ntaps: int, sms: int, gemm: bool = False,
               b_view: bool = False, splits: int = 0, mn_batched: bool = False) -> int:
    """fdx_tc_launch in TC_MNMN (the generic weight gradient and the GEMM_MNMN reductions): 64-row pixel tiles
    (a TW x TH x TN box for convolutions, 64 rows of K for GEMMs), split over the pixel blocks (`splits` 0 =
    the wave-aware count); depth = rows per split + one level per split + the prior."""
    if gemm:
        TW, TH, TN = 64, 1, 1
    else:
        TW = _pow2_floor(min(W, 16))
        TH = _pow2_floor(min(H, 64 // TW))
        TN = 64 // TW // TH
    nxb, nyb, nnb = math.ceil(W / TW), math.ceil(H / TH), math.ceil(N / TN)
    tpp = 2 if (M <= 64 and ntaps > 1 and not b_view) else 1
    base = math.ceil(ntaps / tpp) * math.ceil(M / 128) * math.ceil(Ncols / tc_bn(Ncols))
    kblocks = nxb if mn_batched else nxb * nyb * nnb
    nbz = nyb * nnb if mn_batched else 1
    sp = split_count(sms, base * nbz, kblocks) if splits <= 0 else min(splits, kblocks)
    return 64 * math.ceil(kblocks / sp) + sp + 1


def gemm_ref(a, b, depth: int, alpha: float = 1.0, bias=None, res=None, prior=None):
    """fdx_gemm: D = alpha a @ b + bias + res (+ the prior of an atomic D), a (..., M, K), b (..., K, N) float64
    views of the operands in any GEMM_KK / GEMM_KMN / GEMM_MNMN layout.  depth: K + EPI, or mnmn_depth."""
    a, b = a.to(torch.float64), b.to(torch.float64)
    val, mag = _plus(alpha * (a @ b), abs(alpha) * (a.abs() @ b.abs()), bias, res, prior)
    return val, depth * TC_ADD * mag


# sub-pixel upsample convolution (fdx_upconv.cu): output parity (py, px) reads low-resolution row
# i + (slot - 1 + py) through the sum of the 3x3 taps that land on the same source pixel
def up_slot(parity: int, k: int) -> int:
    return (1 if k >= 1 else 0) if parity == 0 else (1 if k == 2 else 0)


def upconv_pack_ref(w_hwio):
    """upconv_pack_kernel restated: per parity (py, px), the f32 taps added in (ky, kx) order into slot
    (up_slot(py, ky), up_slot(px, kx)) from +0, then rounded to bf16 (round to nearest even) -> bf16 [16][Cin][Cout]."""
    t = w_hwio.to(torch.float32)
    out = []
    for ph in range(4):
        py, px = ph >> 1, ph & 1
        acc = [torch.zeros_like(t[0, 0]) for _ in range(4)]
        for ky in range(3):
            for kx in range(3):
                s = up_slot(py, ky) * 2 + up_slot(px, kx)
                acc[s] = acc[s] + t[ky, kx]
        out += acc
    return torch.stack(out).to(torch.bfloat16)


# the packed weight: fl(sum of <= 4 f32 taps) rounded to bf16 is within PACK times the sum of the taps' |w|
# of the exact tap sum (u_bf16 on the sum, gamma(3) on the f32 additions)
PACK = U_BF16 + gamma(3) * (1 + U_BF16)


def upconv_fwd_ref(x, w_hwio, bias=None, chunk: int = 16):
    """fdx_upconv3x3_fwd = conv3x3(nearest 2x(x)) + bias with the f32 master weights; each parity launch chains
    4 taps x Cin products of the packed bf16 weights (PACK on the weight operand)."""
    up = upsample2x_ref(x.to(torch.float64))
    val, mag = conv3x3_fwd_ref(up, w_hwio, 1, chunk=chunk)[0], conv3x3_fwd_ref(up.abs(), w_hwio.abs(), chunk=chunk)[0]
    val, mag = _plus(val, mag, bias)
    return val, ((4 * x.shape[-1] + EPI) * TC_ADD * (1 + PACK) + PACK) * mag


def upconv_dgrad_ref(dy, w_hwio, prior=None, chunk: int = 16):
    """fdx_upconv3x3_dgrad: the adjoint of upconv_fwd_ref onto the low-resolution x (one launch of 16 taps,
    K = 16 Cout), plus the bf16 prior of accumulate=True."""
    val = upsample2x_bwd_ref(conv3x3_dgrad_ref(dy, w_hwio, chunk=chunk)[0])
    mag = upsample2x_bwd_ref(conv3x3_dgrad_ref(dy.abs(), w_hwio.abs(), chunk=chunk)[0])
    val, mag = _plus(val, mag, prior)
    return val, ((16 * dy.shape[-1] + EPI) * TC_ADD * (1 + PACK) + PACK) * mag


def upconv_wgrad_depth(N: int, h: int, w: int, Cin: int, Cout: int, sms: int) -> int:
    """fdx_upconv3x3_wgrad: a TC_MNMN launch of 16 taps over the low-resolution pixels (B a stride-2 view), then
    upconv_fold_kernel adds the 4 parity slabs of each tap from 0 and adds that onto the prior."""
    return mnmn_depth(w, h, N, Cin, Cout, 16, sms, b_view=True) + 4


def upconv_wgrad_ref(x, dy, depth: int, prior=None, chunk: int = 16):
    """d/dw of upconv_fwd_ref (f32 HWIO) = prior + the 3x3 weight gradient of the upsampled x."""
    return conv3x3_wgrad_ref(upsample2x_ref(x.to(torch.float64)), dy, depth, prior=prior, chunk=chunk)


# 3-channel first and last convolutions (ops.conv_in_* / conv_out_*): im2col3 + one tensor-core GEMM (+ col2im3)
def im2col3_ref(src, sgn: int, ones_col: bool):
    """fdx_im2col3x3_c3: col[p][3 t + k] = src[p + sgn d(t)][k] (0 outside the image) as bf16 (round to nearest
    even from the f32 / bf16 source), column 27 = 1 with ones_col, columns 28..31 = 0 -> (N H W, 32) bf16."""
    N, H, W, _ = src.shape
    sp = Fnn.pad(src.to(torch.float32), (0, 0, 1, 1, 1, 1))
    cols = []
    for ky in range(3):
        for kx in range(3):
            oy, ox = 1 + sgn * (ky - 1), 1 + sgn * (kx - 1)
            cols.append(sp[:, oy:oy + H, ox:ox + W])
    extra = torch.zeros(N, H, W, 5, dtype=torch.float32, device=src.device)
    if ones_col:
        extra[..., 0] = 1
    return torch.cat(cols + [extra], -1).reshape(N * H * W, 32).to(torch.bfloat16)


def col2im3_ref(col, bias, N: int, H: int, W: int):
    """fdx_col2im3x3_c3 restated in f32: y[p][k] = bias[k], then + col[p + d(t)][3 t + k] for the taps inside the
    image in (ky, kx) order -> (N, H, W, 3) f32."""
    c = Fnn.pad(col.to(torch.float32).reshape(N, H, W, 32), (0, 0, 1, 1, 1, 1))
    inside = Fnn.pad(torch.ones(N, H, W, 1, dtype=torch.bool, device=col.device), (0, 0, 1, 1, 1, 1))
    y = bias.to(torch.float32).reshape(1, 1, 1, 3).expand(N, H, W, 3).clone()
    for ky in range(3):
        for kx in range(3):
            t = ky * 3 + kx
            ok = inside[:, ky:ky + H, kx:kx + W]
            y = torch.where(ok, y + c[:, ky:ky + H, kx:kx + W, 3 * t:3 * t + 3], y)
    return y


def conv_in_fwd_ref(x, w_hwio, bias, chunk: int = 64):
    """ops.conv_in_fwd: bf16 im2col of x (exact) times bf16(w) (U_BF16 on the weights), K = 27, with the bias."""
    val, d = conv3x3_fwd_ref(x, w_hwio, 1, bias=bias, chunk=chunk)
    mag = d / ((9 * x.shape[-1] + EPI) * TC_ADD)
    return val, ((27 + EPI) * TC_ADD * (1 + U_BF16) + U_BF16) * mag


def conv_in_wgrad_ref(x, dy, depth: int, dw_prior=None, db_prior=None, chunk: int = 16):
    """ops.conv_in_wgrad: im2col(x)^T dY (with the ones column for the bias) by a GEMM_MNMN reduce over the pixels
    into a zeroed f32 (32, Cout), then added onto the priors: depth = mnmn_depth + 1."""
    dw = conv3x3_wgrad_ref(x, dy, depth, prior=dw_prior, chunk=chunk)
    s = dy.to(torch.float64).sum((0, 1, 2))
    db = _plus(s, dy.to(torch.float64).abs().sum((0, 1, 2)), db_prior)
    return dw, (db[0], depth * TC_ADD * db[1])


def conv_out_fwd_ref(x, w_hwio, bias, chunk: int = 64):
    """ops.conv_out_fwd: GEMM (pixels x Cin)(Cin x 27) of bf16(w) into f32 columns (K = Cin), then col2im3 adds
    the bias and the nine taps' columns in f32 (10 more levels)."""
    val, d = conv3x3_fwd_ref(x, w_hwio, 1, bias=bias, chunk=chunk)
    mag = d / ((9 * x.shape[-1] + EPI) * TC_ADD)
    return val, ((x.shape[-1] + EPI + 10) * TC_ADD * (1 + U_BF16) + U_BF16) * mag


def conv_out_dgrad_ref(dF, w_hwio, chunk: int = 64):
    """ops.conv_out_dgrad: im2col of dF rounded to bf16 (U_BF16 on dF) times bf16(w) (U_BF16 on w), K = 27."""
    val, d = conv3x3_dgrad_ref(dF, w_hwio, 1, chunk=chunk)
    mag = d / ((27 + EPI) * TC_ADD)
    rho = 2 * U_BF16 + U_BF16 ** 2
    return val, ((27 + EPI) * TC_ADD * (1 + rho) + rho) * mag


def conv_out_wgrad_ref(x, dF, depth: int, dw_prior=None, db_prior=None, chunk: int = 16):
    """ops.conv_out_wgrad: x^T im2col(dF) (dF rounded to bf16: U_BF16) by a GEMM_MNMN reduce into a zeroed f32
    (Cin, 32), then added onto the prior (depth = mnmn_depth + 1); the bias gradient is fdx_colsum over the
    bf16 centre-tap columns (depth: the number of pixels, which bounds any order) plus the prior."""
    val, d = conv3x3_wgrad_ref(x, dF, depth, prior=dw_prior, chunk=chunk)
    mag = d / (depth * TC_ADD)
    dw = (val, (depth * TC_ADD * (1 + U_BF16) + U_BF16) * mag)
    f = dF.to(torch.float64)
    P = f.numel() // f.shape[-1]
    s, m = _plus(f.sum((0, 1, 2)), f.abs().sum((0, 1, 2)), db_prior)
    return dw, (s, (gamma(P + 1) * (1 + U_BF16) + U_BF16) * m)


def exact_case_ok(mag) -> bool:
    """Precondition of the exact integer cases: with integer operands and every output's sum of |terms| below
    2^24, every partial sum is an integer of at most 24 bits, so any f32 summation order, truncating or
    rounding, is exact."""
    return bool((mag < 2.0 ** 24).all())


def assert_guard_intact(buf, lo: int, C: int, sentinel: float):
    """The channels of an NHWC buffer outside the slot [lo, lo + C) still hold `sentinel`, bit for bit."""
    side = torch.cat([buf[..., :lo], buf[..., lo + C:]], -1)
    ref = torch.full_like(side, sentinel)
    bits = torch.int16 if side.element_size() == 2 else torch.int32
    assert torch.equal(side.view(bits), ref.view(bits)), "a kernel wrote outside its channel slot"


def conv_gn_backward_ref(x, dy, w_hwio, gamma_, beta_, G, eps):
    """d/dx of conv3x3(silu(groupnorm(x))) given dy = d/d(conv output).  The data gradient reaches the GroupNorm
    backward as bf16: either da itself (two-pass path) or dz = da silu'(z) (fused epilogue) is rounded, so the
    input error is the engine's plus 2^-8 (|da| + its error), scaled by |silu'| <= 1.1 -- the same bound either way."""
    da, e_da = conv3x3_dgrad_ref(dy, w_hwio)
    return gn_backward_ref(x, da, gamma_, beta_, G, eps, True, dy_delta=e_da + U_BF16 * 1.1 * (da.abs() + e_da))


# ----------------------------------------------------------------------------------------------- RMSNorm
def rms_forward_ref(x, scale, eps):
    """y = x rstd scale, rstd = 1/sqrt(mean_c x^2 + eps) per pixel -> (value, delta).
    rms_fwd_kernel: per lane ceil(C/256) vectors of 8 serial squares, then a 5-level warp tree:
    D = 8 ceil(C/256) + 5; q/C and + eps (2 roundings), rsqrtf, then two products."""
    C = x.shape[-1]
    q = (x * x).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(q + eps)
    y = x * r * scale
    rho = gamma(8 * math.ceil(C / 256) + 5 + 2) / 2 + RSQRT + 2 * U32
    return y, rho * y.abs()


def rms_backward_ref(x, dy, scale, eps, npix_per_sweep: int):
    """dx = rstd (g - xhat mean_c(g xhat)), g = dy scale, xhat = x rstd;  dscale = sum_p dy xhat.
    -> dict of (value, delta).  rms_bwd_kernel sums mean_c(g xhat) like the forward sums x^2 (D as above, plus
    the division by C); dscale is a per-warp serial sum over ceil(npix / npix_per_sweep) pixels, 8 warps through
    shared-memory atomics and one global atomic per block (npix_per_sweep / 8 of them)."""
    C = x.shape[-1]
    q = (x * x).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(q + eps)
    xh = x * r
    g = dy * scale
    m = (g * xh).mean(-1, keepdim=True)
    dx = r * (g - xh * m)
    rho = gamma(8 * math.ceil(C / 256) + 5 + 2) / 2 + RSQRT + U32
    gc = gamma(8 * math.ceil(C / 256) + 5 + 1)
    d_dx = (rho + gc + 4 * U32) * r * (g.abs() + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
    npix = x.numel() // C
    ds = (dy * xh).reshape(-1, C).sum(0)
    D = math.ceil(npix / npix_per_sweep) + 8 + npix_per_sweep // 8 + 1
    d_ds = (gamma(D) + rho + U32) * (dy * xh).abs().reshape(-1, C).sum(0)
    return {"dx": (dx, d_dx), "dscale": (ds, d_ds)}


# ----------------------------------------------------------------------------------------------- GEGLU
GELU_C, GELU_A = math.sqrt(2 / math.pi), 0.044715


def _gelu_parts(b):
    inner = GELU_C * (b + GELU_A * b ** 3)
    t = torch.tanh(inner)
    # the f32 argument: b^3 (2 roundings), a b^3, the add, the product by c: 5 roundings on |inner|-scale terms
    d_inner = 5 * U32 * GELU_C * (b.abs() + GELU_A * b.abs() ** 3)
    dt = TANH * t.abs() + (1 - t * t) * d_inner                    # error of the kernel's t
    return inner, t, dt


def geglu_forward_ref(u):
    """u = [lin | gel] (rows, 2 inner) -> g = lin * 0.5 gel (1 + tanh(c (gel + 0.044715 gel^3))) (jax.nn.gelu,
    approximate=True), with delta: |lin| 0.5 |gel| dt from tanh, plus 3 roundings of the products."""
    inner = u.shape[1] // 2
    a, b = u[:, :inner], u[:, inner:]
    _, t, dt = _gelu_parts(b)
    gl = 0.5 * b * (1 + t)
    val = a * gl
    delta = a.abs() * 0.5 * b.abs() * dt + 3 * U32 * (a * 0.5 * b).abs() * (1 + t.abs())
    return val, delta


def geglu_backward_ref(u, dg):
    """du = [dg gelu(gel) | dg lin gelu'(gel)], gelu'(b) = (1+t)/2 + b (1-t^2) c (1 + 3 a b^2) / 2, with delta."""
    inner = u.shape[1] // 2
    a, b = u[:, :inner], u[:, inner:]
    _, t, dt = _gelu_parts(b)
    k = GELU_C * (1 + 3 * GELU_A * b * b)
    gl = 0.5 * b * (1 + t)
    gp = 0.5 * (1 + t) + 0.5 * b * (1 - t * t) * k
    d_lin = dg * gl
    d_gel = dg * a * gp
    e_lin = dg.abs() * 0.5 * b.abs() * dt + 3 * U32 * (dg * 0.5 * b).abs() * (1 + t.abs())
    # d gelu'/dt = 1/2 - b t k; the ~10 roundings of the derivative formula on its absolute-value form
    gp_abs = 0.5 * (1 + t.abs()) + 0.5 * b.abs() * (1 + t * t) * k
    e_gel = (dg * a).abs() * ((0.5 - b * t * k).abs() * dt + 12 * U32 * gp_abs)
    return torch.cat([d_lin, d_gel], 1), torch.cat([e_lin, e_gel], 1)


# ----------------------------------------------------------------------------------------------- streaming
def colsum_ref(x, per_image: bool):
    x = x.to(torch.float64)
    return x.sum((1, 2)) if per_image else x.sum((0, 1, 2))


def upsample2x_ref(x):
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2)


def upsample2x_bwd_ref(dy):
    """Adjoint of nearest 2x: each input pixel receives the sum of its 2x2 output block."""
    N, H2, W2, C = dy.shape
    return dy.to(torch.float64).reshape(N, H2 // 2, 2, W2 // 2, 2, C).sum((2, 4))


# ----------------------------------------------------------------------------------------------- attention
# ex2.approx.ftz.f32: at most 2 ulp of the result over the full range (PTX ISA, ex2; the figure behind __expf's
# 2 + 1.173 |x| ulp in the CUDA C Programming Guide), i.e. 4u relative.  Subnormal results flush to 0: an absolute
# error below FTZ on a weight that is at most 1 against a row sum that is at least 1.
EX2 = 4 * U32
FTZ = 2.0 ** -126
LOGF = 2 * U32               # logf: 1 ulp (CUDA C Programming Guide, Mathematical Functions), 2u relative


def _attn_rows(q, k, v, dO, sc):
    """One (image, head) and a chunk of its query rows: q, dO (R, dh), k, v (Lk, dh), float64.  -> dict of the
    exact forward / backward pieces and their bounds; dk / dv are this chunk's share of the sums over queries."""
    R, dh = q.shape
    Lk = k.shape[0]
    nblk = math.ceil(Lk / 128)
    Lkp = 128 * nblk                     # keys of the zero-filled key blocks: the depth of every sum over keys
    ka, va = k.abs(), v.abs()
    S = q @ k.T
    t = sc * S
    tmax = t.amax(1, keepdim=True)
    e = torch.exp(t - tmax)
    lsum = e.sum(1, keepdim=True)
    lse = tmax + torch.log(lsum)
    P = e / lsum
    O = P @ v
    # S = Q K^T: exact bf16 products, an f32 wgmma chain of dh additions
    es = sc * dh * TC_ADD * (q.abs() @ ka.T)
    # Relative error of each key's weight 2^x, x = fmaf(s, scale_log2, -m), shared by the numerator (acc) and the
    # denominator (l):
    #   S error (es); scale_log2 = fl(scale fl(log2 e)) is 2u off, on |t|; the fma rounds once on
    #   |x| <= log2e (tmax - t), m being the running maximum (m <= the final one, t log2e <= m); ex2: EX2.
    #   corr = ex2(m_old - m_new) scales acc and l by the same factor: its error is a relative error of the weights
    #   of the earlier blocks' keys, shared by numerator and denominator, and is counted here once -- EX2 per
    #   block and the rounding of m_old - m_new, whose sum over the later blocks is <= log2e (tmax - t).
    eta = es + 2 * U32 * t.abs() + 2 * U32 * (tmax - t) + nblk * EX2
    Pe = P * eta
    # O = sum bf16(p) v / sum p (l from the unrounded p):
    #   a weight error moves O by sum_k P_k eta_k (v_k - O) <= (P eta) |v| + |O| sum_k P eta;
    #   P rounded to bf16 for the PV MMA only: U_BF16 sum P |v| (the dominant term);
    #   PV accumulated by wgmma over every key of every block (Lkp terms, TC_ADD each) and the acc * corr + O_j
    #   chain across blocks (gamma(nblk));  l: an f32 sum of <= Lkp terms, the block combine and two quad
    #   shuffles (dh = 128), relative gamma(Lkp + nblk + 2) since every term is positive;
    #   1 / l and acc * inv: 2u.  Flushed weights: FTZ per key.
    eps_l = gamma(Lkp + nblk + 2)
    spa = P @ va
    d_o = (Pe @ va + O.abs() * Pe.sum(1, keepdim=True)
           + (U_BF16 + TC_ADD * Lkp + gamma(nblk) + eps_l + 2 * U32) * spa + FTZ * Lk * va.amax(0))
    # lse = m ln2 + logf(l): m's own rounding cancels against the -m inside every exponent; the weight errors
    # (without the bf16 rounding) and l's sum error move log l; logf 1 ulp of log l; fl(ln 2) and the product m ln2
    # 2u on |tmax| (the f32 rounding of the sum is f32_bound's)
    d_lse = Pe.sum(1) + eps_l + LOGF * torch.log(lsum).squeeze(1) + 2 * U32 * tmax.abs().squeeze(1)
    out = {"o": (O, d_o), "lse": (lse.squeeze(1), d_lse)}
    if dO is None:
        return out
    # D = rowsum(dO o O) from the kernel's bf16 O (its bound ob), a serial f32 fma chain of dh terms
    ob = bf16_bound(O, d_o)
    dOa = dO.abs()
    D = (dO * O).sum(1, keepdim=True)
    e_D = (dOa * ob).sum(1, keepdim=True) + gamma(dh) * (dOa * (O.abs() + ob)).sum(1, keepdim=True)
    # dP = dO V^T: an f32 wgmma chain of dh additions
    dP = dO @ v.T
    e_dP = dh * TC_ADD * (dOa @ va.T)
    # P recomputed from the kernel's lse: p = ex2(fmaf(s, scale_log2, -fl(lse fl(log2 e)))); relative error from S,
    # scale_log2 (2u |t|), the kernel's lse (its f32 bound), fl(log2 e) and the product (2u |lse|), the fma's one
    # rounding on |x| = log2e |t - lse| and ex2; plus FTZ absolute
    lse_b = f32_bound(lse, d_lse.unsqueeze(1))
    eps_p = es + 2 * U32 * t.abs() + lse_b + 2 * U32 * lse.abs() + U32 * (t - lse).abs() + EX2
    ep = P * eps_p + FTZ
    # dS = p fmaf(dP, scale, -fl(D scale)): exact dS = P g, g = scale (dP - D); the fma and the product round once
    # each; dS rounded to bf16 for the output GEMMs
    g = sc * (dP - D)
    e_g = sc * (e_dP + e_D + U32 * D.abs()) + U32 * g.abs()
    dS = P * g
    e_dS = ep * g.abs() + P * e_g + U32 * dS.abs()
    dSa = dS.abs() + e_dS
    e_dSb = e_dS + U_BF16 * dSa
    # the output GEMMs: dQ = dS K accumulates over every key block (Lkp terms); dK = dS^T Q and dV = bf16(P)^T dO
    # over every query tile -- their depth is added by the caller, which knows L; here the sums of |terms|
    Pa = P + ep
    e_Pb = ep + U_BF16 * Pa
    out["dq"] = (dS @ k, e_dSb @ ka + TC_ADD * Lkp * (dSa @ ka))
    out["dk"] = (dS.T @ q, e_dSb.T @ q.abs(), dSa.T @ q.abs())
    out["dv"] = (P.T @ dO, e_Pb.T @ dOa, Pa.T @ dOa)
    return out


def attention_ref(q, k, v, heads: int, dh: int, scale: float, d_o=None, max_elems: int = 1 << 22):
    """Closed-form float64 softmax attention of fdx_attention_fwd / _bwd (o = softmax(q k^T scale) v per (image,
    head); dS = P o (dP - D) scale, dQ = dS K, dK = dS^T Q, dV = P^T dO).  q, d_o: (B, L, heads dh), k, v: (B, Lk,
    heads dh), the bf16 values as float64 on any device; `scale` as the f32 the kernel receives.  Runs per (image,
    head) in chunks of at most `max_elems` (query, key) pairs.  -> dict of (value, delta): o (B, L, HD), lse (B,
    heads, L) and, with d_o, dq (B, L, HD), dk, dv (B, Lk, HD).  Compare o, dq, dk, dv with bf16_bound, lse with
    f32_bound."""
    B, L, HD = q.shape
    Lk = k.shape[1]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    Lp = 128 * math.ceil(L / 128)       # queries of the zero-filled query tiles: the depth of the sums over queries
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=q.device)  # noqa: E731
    res = {"o": (z(B, L, HD), z(B, L, HD)), "lse": (z(B, heads, L), z(B, heads, L))}
    if d_o is not None:
        res.update({n: (z(B, r, HD), z(B, r, HD)) for n, r in (("dq", L), ("dk", Lk), ("dv", Lk))})
    R = max(1, max_elems // Lk)
    for b in range(B):
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            kh, vh = k[b, :, cs], v[b, :, cs]
            acc = {n: [z(Lk, dh), z(Lk, dh), z(Lk, dh)] for n in ("dk", "dv")} if d_o is not None else {}
            for r0 in range(0, L, R):
                rs = slice(r0, min(L, r0 + R))
                out = _attn_rows(q[b, rs, cs], kh, vh, None if d_o is None else d_o[b, rs, cs], sc)
                for n in ("o", "dq") if d_o is not None else ("o",):
                    res[n][0][b, rs, cs], res[n][1][b, rs, cs] = out[n]
                res["lse"][0][b, h, rs], res["lse"][1][b, h, rs] = out["lse"]
                for n in acc:
                    for i in range(3):
                        acc[n][i] += out[n][i]
            for n in acc:
                val, err, mag = acc[n]
                res[n][0][b, :, cs], res[n][1][b, :, cs] = val, err + TC_ADD * Lp * mag
    return res


# ----------------------------------------------------------------------------------------------- training step
# The kernels that run once per step over every parameter (csrc/fdx_optim.cu), the time embedding
# (csrc/fdx_misc.cu) and the diffusion / loss / sampler streams (csrc/fdx_stream.cu).  Conventions as above;
# in addition:
#   * deltas here EXCLUDE the output's own rounding (f32_bound adds it); an intermediate that the kernel rounds
#     and reuses enters downstream with its delta + u |value| (`_full`).
#   * each product or sum of a formula rounds once (u on its absolute value); with FMA contraction some of
#     these roundings disappear, so the same bound covers the fused and the unfused form.
#   * TINY: one rounding into the subnormal range (the library is built without flush-to-zero) is off by at
#     most 2^-150 absolute; every rounding of a value that can be that small adds TINY.
#   * sqrtf is correctly rounded (no fast-math); sinf / cosf / tanhf are within 2 ulp (CUDA C Programming
#     Guide, Mathematical Functions); atomics add in any order, so each atomic on an address is one level of
#     summation depth.
TINY = 2.0 ** -149
TANHF = 4 * U32              # tanhf: 2 ulp of a result in [-1, 1], i.e. 4u relative


def ulp_f32(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of f32 numbers at |ref| (2^(e-24) for |ref| in [2^(e-1), 2^e); 2^-149 below the smallest normal)."""
    a = ref.abs().to(torch.float64).clamp_min(2.0 ** -126)
    _, e = torch.frexp(a)
    return torch.ldexp(torch.ones_like(a), (e - 24).to(torch.int32))


def f32(x: float) -> float:
    """x rounded to f32 (round to nearest), as a Python float."""
    return float(torch.tensor(x, dtype=torch.float32))


def _full(val, delta):
    """Error of an intermediate the kernel rounded to f32 and then reads again."""
    return delta + U32 * val.abs() + TINY


def adam_ref(p, g, m, v, *, lr, b1, b2, eps, wd, bc1, bc2, mul, rho_mul=0.0):
    """One optax adam / adamw step (scale_by_adam -> add_decayed_weights -> -lr) as adam_kernel evaluates it:
        gj = g mul;  m' = b1 m + (1 - b1) gj;  v' = b2 v + (1 - b2) gj gj
        t = (m'/bc1) / (sqrt(v'/bc2) + eps) + wd p;  p' = p - lr t
    p, g, m, v: float64 tensors of the f32 values; the hyperparameters are the f32 values the kernel uses
    (lr, b1, b2, eps, wd, bc1, bc2); `mul` the exact gradient multiplier (grad_scale / loss scale times the
    clip factor) and rho_mul the relative error of the kernel's f32 multiplier.  1 - b is exact for b in
    [0.5, 1] (Sterbenz).  -> dict of (value, delta) for p, m, v and t (LAMB's update u, before -lr)."""
    c1, c2 = 1.0 - b1, 1.0 - b2
    gj = g * mul
    e_gj = (U32 + rho_mul) * gj.abs() + TINY
    m1 = b1 * m + c1 * gj
    e_m = U32 * ((b1 * m).abs() + (c1 * gj).abs()) + c1 * e_gj + 2 * TINY
    v1 = b2 * v + c2 * gj * gj
    e_v = U32 * (b2 * v + 2 * c2 * gj * gj) + 2 * c2 * gj.abs() * e_gj + 3 * TINY
    mh, vh = m1 / bc1, v1 / bc2
    e_mh = _full(m1, e_m) / bc1 + U32 * mh.abs() + TINY
    e_vh = _full(v1, e_v) / bc2 + U32 * vh + TINY
    s = torch.sqrt(vh)
    e_s = torch.where(s > 0, e_vh / (2 * s.clamp_min(1e-300)), torch.sqrt(e_vh)) + U32 * s
    den = s + eps
    e_den = e_s + U32 * den
    q = mh / den
    e_q = e_mh / den + q.abs() * e_den / den + U32 * q.abs() + TINY
    t = q + wd * p
    e_t = e_q + U32 * (wd * p).abs()
    p1 = p - lr * t
    e_p = lr * _full(t, e_t) + U32 * lr * t.abs()
    return {"p": (p1, e_p), "m": (m1, e_m), "v": (v1, e_v), "t": (t, e_t)}


def ema_ref(ema, p, decay, e_p=None):
    """TrainState.apply_ema: ema' = decay ema + (1 - decay) p (decay and 1 - decay as the kernel's f32 values);
    e_p: delta of the p the kernel reads (the fused step's p' before its rounding), None when p is exact."""
    c = f32(1.0 - decay)
    val = decay * ema + c * p
    delta = U32 * ((decay * ema).abs() + (c * p).abs()) + 2 * TINY
    if e_p is not None:
        delta = delta + c * _full(p, e_p)
    return val, delta


def sumsq_ref(g, mul, depth: int):
    """fdx_grad_stats' out[0] = sum (g mul)^2 over a buffer, with a summation depth `depth`; the kernel's
    product g fl(mul) and the square add 3u relative to each (positive) term, the multiplier's rounding 1u."""
    x = g * mul
    val = (x * x).sum()
    return val, gamma(depth + 4) * val


def grad_stats_depth(n: int, sms: int) -> int:
    """grad_stats_kernel: grid = min(ceil(n/4/256), 8 SMs) blocks of 256 threads; each thread adds one float4
    (a 4-term chain) per grid-stride iteration to its running sum, then a warp tree (5), the 8 warps' tree (5)
    and one atomic per block."""
    n4 = n // 4
    blocks = max(1, min(math.ceil(n4 / 256), 8 * sms))
    iters = math.ceil(n4 / (blocks * 256))
    return 4 + iters + 10 + blocks


def lamb_ref(p, g, m, v, seg_start, seg_len, *, lr, b1, b2, eps, wd, bc1, bc2, mul, rho_mul=0.0):
    """optax.lamb over a flat buffer of segments [seg_start, seg_start + seg_len) (tensor slots, 64-aligned,
    zero gaps): u = adam's t, ratio = ||p|| / ||u|| per segment (1 where either is 0), p' = p - lr ratio u.
    lamb_pass1_kernel sums each segment's p^2 and u^2 as 4-term fmaf chains, then a warp tree (5) and one
    atomic per warp when the warp's 128 elements lie in one segment, per thread otherwise: at most
    ceil(len/128) + 1 single-segment warps, 2 x 32 threads of warps that straddle a boundary and 32 of the
    partial last warp.  -> dict of (value, delta) for p, m, v, u, and the per-segment norms (sum p^2, sum u^2)."""
    r = adam_ref(p, g, m, v, lr=lr, b1=b1, b2=b2, eps=eps, wd=wd, bc1=bc1, bc2=bc2, mul=mul, rho_mul=rho_mul)
    u, e_u = r["t"]
    e_uf = _full(u, e_u)
    nseg = seg_start.numel()
    seg = torch.repeat_interleave(torch.arange(nseg, device=p.device), seg_len)

    def ssum(x):
        return torch.zeros(nseg, dtype=torch.float64, device=p.device).index_add_(0, seg, x)

    D = torch.tensor([9 + math.ceil(int(n) / 128) + 1 + 96 for n in seg_len.tolist()], dtype=torch.float64,
                     device=p.device)
    gD = D * U32 / (1 - D * U32)
    np2, nu2 = ssum(p * p), ssum(u * u)
    e_np2 = gD * np2
    e_nu2 = gD * nu2 + 2 * ssum(u.abs() * e_uf)
    pn, un = torch.sqrt(np2), torch.sqrt(nu2)
    one = (pn == 0) | (un == 0)
    ratio = torch.where(one, torch.ones_like(pn), pn / torch.where(one, torch.ones_like(un), un))
    rel = torch.where(one, torch.zeros_like(pn),
                      e_np2 / (2 * np2.clamp_min(1e-300)) + e_nu2 / (2 * nu2.clamp_min(1e-300)) + 3 * U32)
    a, rel_a = (lr * ratio)[seg], (rel + U32)[seg]
    p1 = p - a * u
    e_p = a * e_uf + (a * u).abs() * (rel_a + U32)
    return {"p": (p1, e_p), "m": r["m"], "v": r["v"], "u": (u, e_u), "np2": (np2, e_np2), "nu2": (nu2, e_nu2)}


# time embedding: gelu(tanh) with tanhf and the f32 constants of fdx_misc.cu
GELU_K = math.sqrt(2 / math.pi)


def gelu_f32_ref(x):
    """gelu_tanh(x) = 0.5 x (1 + tanhf(k (x + a x^3))) -> (value, delta, t, e_t): the argument carries 7
    roundings (x^3: 2, a x^3, the sum, k ( ), the f32 constants k and a) on k (|x| + a |x|^3)."""
    inner = GELU_K * (x + GELU_A * x ** 3)
    t = torch.tanh(inner)
    e_in = 7 * U32 * GELU_K * (x.abs() + GELU_A * x.abs() ** 3)
    e_t = TANHF * t.abs() + (1 - t * t) * e_in
    y = 0.5 * x * (1 + t)
    return y, 0.5 * x.abs() * (e_t + U32 * (1 + t).abs()), t, e_t


def gelu_grad_f32_ref(x):
    """gelu_tanh_grad: 0.5 (1 + t) + 0.5 x (1 - t^2) k (1 + 3 a x^2) -> (value, delta incl. its own rounding):
    the error of t times d/dt = 1/2 - x t K, and 12 roundings on the absolute-value form."""
    _, _, t, e_t = gelu_f32_ref(x)
    K = GELU_K * (1 + 3 * GELU_A * x * x)
    gp = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * K
    gp_abs = 0.5 * (1 + t.abs()) + 0.5 * x.abs() * (1 + t * t) * K
    return gp, (0.5 - x * t * K).abs() * e_t + 12 * U32 * gp_abs


def time_phase_f32(t, freqs):
    """The kernel's phase: fl(t fl(fl(2 pi) f)), in f32 (one correctly rounded product each) -> (B, D/2)."""
    w = torch.tensor(2 * math.pi, dtype=torch.float32, device=freqs.device) * freqs.to(torch.float32)
    return t.to(torch.float32)[:, None] * w[None, :]


def time_embed_fwd_ref(ph, four, h1, h2, W1, b1, W2, b2):
    """FourierEmbedding + TimeProjection, each stage from the f32 values the kernel stored before it (four, h1,
    h2: float64 of the kernel's outputs).  Dense: a serial chain of D fmas onto the bias (gamma(D)).
    -> dict of (value, bound): 'four' is bounded by 2 ulp of the float64 sine / cosine of the f32 phase; the
    others are (value, delta) for f32_bound."""
    D = W1.shape[0]
    ph = ph.to(torch.float64)
    fr = torch.cat([torch.sin(ph), torch.cos(ph)], 1)
    out = {"four": (fr, 2 * ulp_f32(fr))}
    out["h1"] = (b1 + four @ W1, gamma(D) * (b1.abs() + four.abs() @ W1.abs()))
    g1, e_g1 = gelu_f32_ref(h1)[:2]
    out["h2"] = (b2 + g1 @ W2, gamma(D) * (b2.abs() + g1.abs() @ W2.abs()) + _full(g1, e_g1) @ W2.abs())
    out["emb"] = gelu_f32_ref(h2)[:2]
    return out


def wgrad_small_depth(B: int) -> int:
    """dense_wgrad_small_kernel: batch slices bs = 16 / 4 / 1 for B >= 64 / >= 8 / < 8, a serial chain over
    ceil(B / bs) samples each, then bs atomics onto the prior value."""
    bs = 16 if B >= 64 else (4 if B >= 8 else 1)
    return math.ceil(B / bs) + bs + 1


def time_embed_bwd_ref(demb, four, h1, h2, dh1, dh2, W2, dW1_0, db1_0, dW2_0, db2_0):
    """Backward of the time MLP, each stage from the kernel's stored f32 inputs (dh1, dh2: its workspaces):
        dh2 = demb gelu'(h2);  dh1 = (dh2 W2^T) gelu'(h1);  dW2 += gelu(h1)^T dh2;  dW1 += four^T dh1;  db += sum_b
    -> dict of (value, delta) for dh2, dh1, dW1, db1, dW2, db2."""
    D, B = W2.shape[0], demb.shape[0]
    gp2, e_gp2 = gelu_grad_f32_ref(h2)
    gp1, e_gp1 = gelu_grad_f32_ref(h1)
    out = {"dh2": (demb * gp2, demb.abs() * e_gp2)}
    da1 = dh2 @ W2.T
    e_da1 = gamma(D) * (dh2.abs() @ W2.abs().T)
    out["dh1"] = (da1 * gp1, gp1.abs() * e_da1 + da1.abs() * e_gp1)
    g1, e_g1 = gelu_f32_ref(h1)[:2]
    gw = gamma(wgrad_small_depth(B))
    out["dW2"] = (dW2_0 + g1.T @ dh2, gw * (dW2_0.abs() + g1.abs().T @ dh2.abs()) + _full(g1, e_g1).T @ dh2.abs())
    out["db2"] = (db2_0 + dh2.sum(0), gw * (db2_0.abs() + dh2.abs().sum(0)))
    out["dW1"] = (dW1_0 + four.T @ dh1, gw * (dW1_0.abs() + four.abs().T @ dh1.abs()))
    out["db1"] = (db1_0 + dh1.sum(0), gw * (db1_0.abs() + dh1.abs().sum(0)))
    return out


def diffuse_ref(x0, eps, alpha, sigma, normalize: bool, kind: int):
    """forward_diffusion + get_target of diffuse_forward_kernel: x = (x0 - 127.5) / 127.5 (one rounding) or x0;
    x_t = a x + s eps; target x / eps / (a eps - s x) rsqrtf(a^2 + s^2).  x0, eps: (B, E) float64; alpha,
    sigma: (B,) the f32 values.  -> dict of (value, delta) for x_t and target."""
    a, s = alpha[:, None], sigma[:, None]
    x = (x0 - 127.5) / 127.5 if normalize else x0
    e_x = U32 * x.abs() if normalize else torch.zeros_like(x)
    xt = a * x + s * eps
    out = {"x_t": (xt, a.abs() * e_x + U32 * ((a * x).abs() + (s * eps).abs()))}
    if kind == 0:
        out["target"] = (x, torch.zeros_like(x))      # the normalising division is the output's own rounding
    elif kind == 1:
        out["target"] = (eps, torch.zeros_like(eps))
    else:
        inv = 1.0 / torch.sqrt(a * a + s * s)
        rho = gamma(3) / 2 + RSQRT
        d = a * eps - s * x
        e_d = U32 * ((a * eps).abs() + (s * x).abs() + d.abs()) + s.abs() * e_x
        out["target"] = (d * inv, inv * e_d + (d * inv).abs() * rho)
    return out


def loss_ref(F, x_t, target, c_out, c_skip, weight, depth: int):
    """optax.l2_loss weighted and averaged (loss_kernel): d = c_out F + c_skip x_t - target (4 roundings on the
    absolute-value sum), loss = sum 0.5 w d^2 / (B E), dF = w c_out d / (B E) with g = fl(fl(w c_out) fl(1/(BE)))
    (3u).  The loss adds, per positive term, 4 roundings of the float4's squares, the product by w, the product by
    1/(BE) and its rounding, and `depth` levels of summation.  -> dict of (value, delta) for loss and dF."""
    B, E = F.shape
    co, cs, w = c_out[:, None], c_skip[:, None], weight[:, None]
    d = co * F + cs * x_t - target
    e_d = gamma(4) * ((co * F).abs() + (cs * x_t).abs() + target.abs())
    g = w * co / (B * E)
    term = 0.5 * w * d * d / (B * E)
    loss = term.sum()
    e_loss = gamma(depth + 7) * loss + (w * d.abs() * e_d).sum() / (B * E)
    return {"loss": (loss, e_loss), "dF": (g * d, g.abs() * e_d + 3 * U32 * (g * d).abs())}


def affine_ref(inputs, coef):
    """sum_k coef[k, b] in_k as a serial chain of n_in fmas from 0 (affine_kernel) -> (value, delta)."""
    val = sum(c[:, None] * x for c, x in zip(coef, inputs))
    mag = sum((c[:, None] * x).abs() for c, x in zip(coef, inputs))
    return val, gamma(len(inputs)) * mag
