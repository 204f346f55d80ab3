"""Thin Python wrappers over the libfdx C-ABI (one function per entry point).

Tensors are NHWC bf16 activations / HWIO conv kernels exactly as the reference's flax
modules store them (flaxdiff/models/common.py:166-172).  No arithmetic happens in
Python: each wrapper marshals pointers, shapes and the current CUDA stream.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN, act, check, load, ptr, stream_ptr


def _opt_act(t: Optional[torch.Tensor], name: str):
    return None if t is None else act(t, name)


# --------------------------------------------------------------------------- conv
COLSTATS_SLOTS = 4
COLSTATS_MIN_PIXELS = 128     # the engines accumulate fused per-image sums on images of >= 128 pixels


class ColStats:
    """Per-(image, channel) sum / sum-of-squares workspace of one activation BUFFER, filled by the epilogues
    of the convolutions that write into it (each at its channel offset) and turned into GroupNorm
    statistics by groupnorm_stats_from_cols."""

    def __init__(self, n: int, channels: int, device, slots: int = COLSTATS_SLOTS):
        self.ws = torch.zeros((slots, n, 2, channels), dtype=torch.float32, device=device)
        self.n, self.channels, self.slots = n, channels, slots

    def desc(self, channel_offset: int = 0):
        return _lib.fdx_colstats(self.ws.data_ptr() + 4 * channel_offset, self.slots, self.channels)


def groupnorm_stats_from_cols(cs: ColStats, groups: int, c0: int = 0, channels: Optional[int] = None) -> torch.Tensor:
    """fdx_groupnorm_stats' output for channels [c0, c0 + channels) of the buffer, from its epilogue sums."""
    channels = cs.channels - c0 if channels is None else channels
    stats = torch.empty((cs.n, groups, 2), dtype=torch.float32, device=cs.ws.device)
    check(load().fdx_groupnorm_stats_from_cols(ptr(cs.ws), cs.slots, cs.n, cs.channels, c0, channels, groups,
                                               ptr(stats), stream_ptr()), "groupnorm_stats_from_cols")
    return stats


def conv3x3_fwd(x: torch.Tensor, w_hwio: torch.Tensor, bias: Optional[torch.Tensor] = None,
                rowvec: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, stride: int = 1, colstats=None) -> torch.Tensor:
    """3x3 SAME conv, NHWC bf16, HWIO bf16 weights; out = conv + bias + rowvec[n] + res.
    colstats = (ColStats, channel offset): also accumulate the output's per-image channel sums."""
    n, h, w, cin = x.shape
    cout = w_hwio.shape[-1]
    assert w_hwio.dtype == torch.bfloat16 and w_hwio.is_contiguous()
    assert tuple(w_hwio.shape) == (3, 3, cin, cout), (w_hwio.shape, cin, cout)
    ho, wo = (h + stride - 1) // stride, (w + stride - 1) // stride
    if out is None:
        out = torch.empty((n, ho, wo, cout), dtype=torch.bfloat16, device=x.device)
    if colstats is not None:
        d = colstats[0].desc(colstats[1])
        check(load().fdx_conv3x3_fwd_stats(act(x, "x"), ptr(w_hwio), ptr(bias), ptr(rowvec), _opt_act(res, "res"),
                                           act(out, "out"), stride, d, stream_ptr()), "conv3x3_fwd_stats")
        return out
    check(load().fdx_conv3x3_fwd(act(x, "x"), ptr(w_hwio), ptr(bias), ptr(rowvec), _opt_act(res, "res"),
                                 act(out, "out"), stride, stream_ptr()), "conv3x3_fwd")
    return out


def conv3x3_dgrad(dy: torch.Tensor, w_hwio: torch.Tensor, dx: torch.Tensor, stride: int = 1,
                  accumulate: bool = False) -> torch.Tensor:
    check(load().fdx_conv3x3_dgrad(act(dy, "dy"), ptr(w_hwio), act(dx, "dx"), stride, int(accumulate),
                                   stream_ptr()), "conv3x3_dgrad")
    return dx


def conv3x3_wgrad(x: torch.Tensor, dy: torch.Tensor, dw_hwio: torch.Tensor, stride: int = 1) -> torch.Tensor:
    """Accumulates d(loss)/dw (f32 HWIO) into dw_hwio."""
    assert dw_hwio.dtype == torch.float32 and dw_hwio.is_contiguous()
    check(load().fdx_conv3x3_wgrad(act(x, "x"), act(dy, "dy"), ptr(dw_hwio), stride, stream_ptr()), "conv3x3_wgrad")
    return dw_hwio


def conv1x1_fwd(x: torch.Tensor, w_io: torch.Tensor, bias: Optional[torch.Tensor] = None,
                res: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """1x1 conv in convolution geometry: x NHWC bf16, w_io bf16 [Cin, Cout] (flax (1,1,Cin,Cout))."""
    n, h, w, cin = x.shape
    cout = w_io.shape[-1]
    assert w_io.dtype == torch.bfloat16 and w_io.is_contiguous() and w_io.numel() == cin * cout
    if out is None:
        out = torch.empty((n, h, w, cout), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_conv1x1_fwd(act(x, "x"), ptr(w_io), ptr(bias), _opt_act(res, "res"),
                                 act(out, "out"), stream_ptr()), "conv1x1_fwd")
    return out


def conv1x1_dgrad(dy: torch.Tensor, w_io: torch.Tensor, dx: torch.Tensor, accumulate: bool = False) -> torch.Tensor:
    check(load().fdx_conv1x1_dgrad(act(dy, "dy"), ptr(w_io), act(dx, "dx"), int(accumulate), stream_ptr()),
          "conv1x1_dgrad")
    return dx


# --------------------------------------------------------------------------- gemm
def gemm(mode: int, A: torch.Tensor, B: torch.Tensor, D: torch.Tensor, M: int, N: int, K: int,
         a_ld: int, b_ld: int, d_ld: int, batch1: int = 1, batch2: int = 1,
         a_s=(0, 0), b_s=(0, 0), d_s=(0, 0), alpha: float = 1.0,
         bias: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
         r_ld: int = 0, r_s=(0, 0), atomic: bool = False, reduce_batch: bool = False) -> torch.Tensor:
    """Generic (batched) bf16 GEMM on the tensor-core engine; see include/fdx.h fdx_gemm_desc."""
    g = _gemm_desc(mode, A, B, D, M, N, K, a_ld, b_ld, d_ld, batch1, batch2, a_s, b_s, d_s, alpha, bias, res, r_ld,
                   r_s, atomic, reduce_batch)
    check(load().fdx_gemm(g, stream_ptr()), "gemm")
    return D


def _gemm_desc(mode, A, B, D, M, N, K, a_ld, b_ld, d_ld, batch1, batch2, a_s, b_s, d_s, alpha, bias, res, r_ld, r_s,
               atomic, reduce_batch):
    g = _lib.fdx_gemm_desc()
    g.mode = mode
    g.M, g.N, g.K = M, N, K
    g.batch1, g.batch2 = batch1, batch2
    g.A, g.a_ld, g.a_s1, g.a_s2 = ptr(A), a_ld, a_s[0], a_s[1]
    g.B, g.b_ld, g.b_s1, g.b_s2 = ptr(B), b_ld, b_s[0], b_s[1]
    g.D, g.d_ld, g.d_s1, g.d_s2 = ptr(D), d_ld, d_s[0], d_s[1]
    g.d_f32 = int(D.dtype == torch.float32)
    g.d_atomic = int(atomic)
    g.reduce_batch = int(reduce_batch)
    g.alpha = alpha
    g.bias = ptr(bias)
    g.res, g.r_ld, g.r_s1, g.r_s2 = ptr(res), r_ld, r_s[0], r_s[1]
    return g


def gemm_cat(mode: int, A0: torch.Tensor, A1: torch.Tensor, B: torch.Tensor, D: torch.Tensor, M: int, N: int, K: int,
             K0: int, a_ld: int, a1_ld: int, b_ld: int, d_ld: int, bias: Optional[torch.Tensor] = None,
             res: Optional[torch.Tensor] = None, r_ld: int = 0) -> torch.Tensor:
    """gemm (KK or KMN, batch 1) with A = [A0 | A1] along k - k < K0 from A0, the rest from A1 - without writing the
    concatenation; bit for bit gemm on torch.cat([A0, A1], 1).  See include/fdx.h fdx_gemm_cat."""
    g = _gemm_desc(mode, A0, B, D, M, N, K, a_ld, b_ld, d_ld, 1, 1, (0, 0), (0, 0), (0, 0), 1.0, bias, res, r_ld,
                   (0, 0), False, False)
    check(load().fdx_gemm_cat(g, ptr(A1), a1_ld, K0, stream_ptr()), "gemm_cat")
    return D


def linear_cat_fwd(x0: torch.Tensor, x1: torch.Tensor, w_kn: torch.Tensor, bias: Optional[torch.Tensor] = None,
                   out_dtype=torch.bfloat16) -> torch.Tensor:
    """y = [x0 | x1] @ w (+ bias): a Dense over the concatenation of two row matrices, w [K0 + K1, N]."""
    M, K0 = x0.shape
    K = K0 + x1.shape[1]
    assert x1.shape[0] == M and w_kn.shape[0] == K and x0.stride(1) == 1 and x1.stride(1) == 1 and w_kn.is_contiguous()
    N = w_kn.shape[1]
    out = torch.empty((M, N), dtype=out_dtype, device=x0.device)
    return gemm_cat(GEMM_KMN, x0, x1, w_kn, out, M, N, K, K0, x0.stride(0), x1.stride(0), N, N, bias=bias)


def linear_fwd(x2d: torch.Tensor, w_kn: torch.Tensor, out: Optional[torch.Tensor] = None,
               bias: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None,
               out_dtype=torch.bfloat16) -> torch.Tensor:
    """y[m][n] = x[m][k] @ w[k][n] (flax Dense kernel layout (in, out)); x row stride may exceed K."""
    M, K = x2d.shape
    Kw, N = w_kn.shape
    assert K == Kw and x2d.stride(1) == 1 and w_kn.is_contiguous()
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x2d.device)
    return gemm(GEMM_KMN, x2d, w_kn, out, M, N, K, x2d.stride(0), N, out.stride(0), bias=bias,
                res=res, r_ld=(res.stride(0) if res is not None else 0))


# --------------------------------------------------------------------------- norms
# Activation codes of the GroupNorm entry points' `act` argument.  The wrappers take the code or a bool, so that
# the positional True / False of existing callers keep meaning silu / none.
ACT_NONE, ACT_SILU, ACT_MISH = 0, 1, 2


def _act_code(a) -> int:
    code = int(a)
    if code not in (ACT_NONE, ACT_SILU, ACT_MISH):
        raise ValueError(f"activation code {a!r}: expected 0 (none), 1 (silu) or 2 (mish)")
    return code


def groupnorm_stats(x: torch.Tensor, groups: int) -> torch.Tensor:
    stats = torch.empty((x.shape[0], groups, 2), dtype=torch.float32, device=x.device)
    check(load().fdx_groupnorm_stats(act(x, "x"), groups, ptr(stats), stream_ptr()), "groupnorm_stats")
    return stats


def groupnorm_apply(x, groups, stats, gamma, beta, eps: float, act_fn, out=None) -> torch.Tensor:
    """y = act_fn(GroupNorm(x)); act_fn = ACT_NONE / ACT_SILU / ACT_MISH (or False / True)."""
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_groupnorm_apply(act(x, "x"), groups, ptr(stats), ptr(gamma), ptr(beta), eps, _act_code(act_fn),
                                     act(out, "out"), stream_ptr()), "groupnorm_apply")
    return out


def groupnorm_apply_cols(x, groups, cs: "ColStats", c0: int, gamma, beta, eps: float, act_fn, out=None):
    """groupnorm_apply with the statistics read from the producers' epilogue column sums (no stats_from_cols
    launch) -> (y, stats[N][groups][2] for the backward)."""
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    stats = torch.empty((cs.n, groups, 2), dtype=torch.float32, device=x.device)
    check(load().fdx_groupnorm_apply_cols(act(x, "x"), groups, ptr(cs.ws), cs.slots, cs.channels, c0, ptr(gamma),
                                          ptr(beta), eps, _act_code(act_fn), act(out, "out"), ptr(stats),
                                          stream_ptr()), "groupnorm_apply_cols")
    return out, stats


def groupnorm_bwd(x, dy, groups, stats, gamma, beta, eps, act_fn, dgamma, dbeta, dx,
                  accumulate: bool = False, csum_img=None, csum_tot=None, addend=None) -> torch.Tensor:
    """dx (+)= d/dx act_fn(GroupNorm(x)); `addend`: dx = d/dx + addend (another tensor of the same shape)."""
    code = _act_code(act_fn)
    red = torch.empty(2 * x.shape[0] * groups, dtype=torch.float32, device=x.device)
    if addend is not None:
        assert not accumulate
        check(load().fdx_groupnorm_bwd_add(act(x, "x"), act(dy, "dy"), groups, ptr(stats), ptr(gamma), ptr(beta),
                                           eps, code, ptr(red), ptr(dgamma), ptr(dbeta), act(dx, "dx"),
                                           act(addend, "addend"), ptr(csum_img), ptr(csum_tot), stream_ptr()),
              "groupnorm_bwd_add")
        return dx
    check(load().fdx_groupnorm_bwd(act(x, "x"), act(dy, "dy"), groups, ptr(stats), ptr(gamma), ptr(beta), eps,
                                   code, ptr(red), ptr(dgamma), ptr(dbeta), act(dx, "dx"), int(accumulate),
                                   ptr(csum_img), ptr(csum_tot), stream_ptr()), "groupnorm_bwd")
    return dx


GN_FUSE_SLOTS = 8
GN_FUSE_MIN_PIXELS = 128    # fdx_conv3x3_dgrad_gn fuses on images of >= 128 pixels
# Mish fuses by default only on images of at most 16 x 16 pixels: at 32^2 and 64^2 its epilogue (an exponential and a
# reciprocal per element) made the fused backward 2-5 % slower than the two passes on an H100 SXM (DESIGN 3.2).
GN_FUSE_MISH_MAX_PIXELS = 256


def groupnorm_coeffs(stats, gamma, beta, hw: int, eps: float) -> torch.Tensor:
    """ab[n][0][c] = rstd*gamma_c, ab[n][1][c] = beta_c - mean*rstd*gamma_c (f32)."""
    n, groups = stats.shape[0], stats.shape[1]
    c = gamma.numel()
    ab = torch.empty((n, 2, c), dtype=torch.float32, device=stats.device)
    check(load().fdx_groupnorm_coeffs(ptr(stats), ptr(gamma), ptr(beta), n, hw, c, groups, eps, ptr(ab),
                                      stream_ptr()), "groupnorm_coeffs")
    return ab


def conv3x3_dgrad_gn(dy: torch.Tensor, w_hwio: torch.Tensor, dz: torch.Tensor, x: torch.Tensor,
                     ab: torch.Tensor, slots: int = GN_FUSE_SLOTS, act_fn=ACT_SILU) -> torch.Tensor:
    """Stride-1 data gradient with the first pass of GroupNorm(+activation) backward fused into its epilogue:
    writes dz = dgrad * act'(a x + b) and returns the per-slot sums workspace for groupnorm_bwd_dz.  act_fn =
    ACT_SILU or ACT_MISH; mish runs on the transposed engine only (_gn_fuse_default) and raises elsewhere."""
    n, c = dz.shape[0], dz.shape[-1]
    ws = torch.empty((slots, n, 2, c), dtype=torch.float32, device=dz.device)
    check(load().fdx_conv3x3_dgrad_gn_act(act(dy, "dy"), ptr(w_hwio), act(dz, "dz"), act(x, "x"), ptr(ab), ptr(ws),
                                          slots, _act_code(act_fn), stream_ptr()), "conv3x3_dgrad_gn")
    return ws


def groupnorm_bwd_dz(x, dz, groups, stats, gamma, eps, ws_slots, dgamma, dbeta, dx,
                     accumulate: bool = False, csum_img=None, csum_tot=None, addend=None) -> torch.Tensor:
    if addend is not None:
        assert not accumulate, "groupnorm_bwd_dz: addend and accumulate are exclusive"
        check(load().fdx_groupnorm_bwd_dz_add(act(x, "x"), act(dz, "dz"), groups, ptr(stats), ptr(gamma), eps,
                                              ptr(ws_slots), ws_slots.shape[0], None, ptr(dgamma), ptr(dbeta),
                                              act(dx, "dx"), act(addend, "addend"), ptr(csum_img), ptr(csum_tot),
                                              stream_ptr()), "groupnorm_bwd_dz_add")
        return dx
    check(load().fdx_groupnorm_bwd_dz(act(x, "x"), act(dz, "dz"), groups, ptr(stats), ptr(gamma), eps, ptr(ws_slots),
                                      ws_slots.shape[0], None, ptr(dgamma), ptr(dbeta), act(dx, "dx"),
                                      int(accumulate), ptr(csum_img), ptr(csum_tot), stream_ptr()),
          "groupnorm_bwd_dz")
    return dx


def _gn_fuse_default(x: torch.Tensor, dy: torch.Tensor) -> bool:
    """The fused first pass is the default where the data gradient runs on the transposed engine (eight epilogue
    warps hide the silu' arithmetic; DESIGN 3.2): Cin = 64 ... 512 not a multiple of 256, 16-aligned images."""
    cin, h, w = x.shape[-1], x.shape[1], x.shape[2]
    return (cin % 64 == 0 and cin % 256 != 0 and cin <= 512 and dy.shape[-1] % 64 == 0 and h % 16 == 0 and
            w % 16 == 0 and h * w >= GN_FUSE_MIN_PIXELS)


def conv_dgrad_groupnorm_bwd(dy, w_hwio, x, groups, stats, gamma, beta, eps, dgamma, dbeta, dx,
                             accumulate: bool = False, csum_img=None, csum_tot=None,
                             fused: Optional[bool] = None, addend=None, act_fn=ACT_SILU) -> torch.Tensor:
    """d/dx of conv3x3(act_fn(groupnorm(x))) given dy = d/d(conv output): the data gradient with the first pass
    of the GroupNorm backward in its epilogue (dz = dy * act'(z), sum dz, sum dz*x) where that convolution runs
    on the transposed engine, then ONE pass over x and dz; elsewhere data gradient + the two-pass GroupNorm
    backward.  SiLU: `fused=True` fuses wherever an image has >= 128 pixels (also on the pixels-as-M engine),
    `fused=False` never.  Mish has a fused epilogue on the transposed engine only: by default it fuses where
    _gn_fuse_default holds on images of at most GN_FUSE_MISH_MAX_PIXELS, `fused=True` wherever _gn_fuse_default
    holds; every other shape takes the two passes."""
    code = _act_code(act_fn)
    da = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    if code == ACT_MISH:
        small = x.shape[1] * x.shape[2] <= GN_FUSE_MISH_MAX_PIXELS
        fused = fused is not False and _gn_fuse_default(x, dy) and (fused is True or small)
    elif fused is None:
        fused = _gn_fuse_default(x, dy)
    if fused and x.shape[1] * x.shape[2] >= GN_FUSE_MIN_PIXELS:
        ab = groupnorm_coeffs(stats, gamma, beta, x.shape[1] * x.shape[2], eps)
        ws = conv3x3_dgrad_gn(dy, w_hwio, da, x, ab, act_fn=code)
        return groupnorm_bwd_dz(x, da, groups, stats, gamma, eps, ws, dgamma, dbeta, dx, accumulate,
                                csum_img=csum_img, csum_tot=csum_tot, addend=addend)
    conv3x3_dgrad(dy, w_hwio, da)
    return groupnorm_bwd(x, da, groups, stats, gamma, beta, eps, code, dgamma, dbeta, dx, accumulate,
                         csum_img=csum_img, csum_tot=csum_tot, addend=addend)


def rmsnorm_fwd(x, scale, eps: float, out=None) -> torch.Tensor:
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_rmsnorm_fwd(act(x, "x"), ptr(scale), eps, act(out, "out"), stream_ptr()), "rmsnorm_fwd")
    return out


def rmsnorm_bwd(x, dy, scale, eps, dx, dscale, accumulate: bool = False) -> torch.Tensor:
    check(load().fdx_rmsnorm_bwd(act(x, "x"), act(dy, "dy"), ptr(scale), eps, act(dx, "dx"), int(accumulate),
                                 ptr(dscale), stream_ptr()), "rmsnorm_bwd")
    return dx


# --------------------------------------------------------------------------- streaming
TARGET_X0, TARGET_EPS, TARGET_V = 0, 1, 2


def diffuse_forward(x0: torch.Tensor, eps: torch.Tensor, alpha, sigma, c_in, normalize: bool,
                    target_kind: int):
    """-> (x_t f32, target f32, model_in bf16); x0 may be uint8 or f32, shape (B, ...)."""
    B = x0.shape[0]
    E = x0.numel() // B
    assert x0.is_contiguous() and eps.is_contiguous() and eps.dtype == torch.float32
    assert x0.dtype in (torch.uint8, torch.float32)
    x_t = torch.empty(tuple(x0.shape), dtype=torch.float32, device=x0.device)
    target = torch.empty_like(x_t)
    model_in = torch.empty(tuple(x0.shape), dtype=torch.bfloat16, device=x0.device)
    check(load().fdx_diffuse_forward(ptr(x0), int(x0.dtype == torch.uint8), ptr(eps), ptr(_f32c(alpha)),
                                     ptr(_f32c(sigma)), ptr(_f32c(c_in)), B, E, int(normalize), target_kind,
                                     ptr(x_t), ptr(target), ptr(model_in), stream_ptr()), "diffuse_forward")
    return x_t, target, model_in


def _f32c(t: torch.Tensor) -> torch.Tensor:
    t = t.reshape(-1)
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.to(torch.float32).contiguous()
    return t


def loss_fwd_bwd(F: torch.Tensor, x_t, target, c_out, c_skip, weight, want_grad: bool = True):
    """-> (loss scalar tensor f32[1], dF f32 or None)."""
    B = F.shape[0]
    E = F.numel() // B
    loss = torch.empty(1, dtype=torch.float32, device=F.device)
    dF = torch.empty_like(F) if want_grad else None
    check(load().fdx_loss_fwd_bwd(ptr(F), ptr(x_t), ptr(target), ptr(_f32c(c_out)), ptr(_f32c(c_skip)),
                                  ptr(_f32c(weight)), B, E, ptr(loss), ptr(dF), stream_ptr()), "loss_fwd_bwd")
    return loss, dF


def affine_combine(inputs, coef1: torch.Tensor, coef2: Optional[torch.Tensor] = None,
                   want_out1: bool = True, bf16_scale: Optional[torch.Tensor] = None,
                   want_bf16: bool = False, clip=None):
    """out1 = sum_i coef1[i,b]*in_i; out2 = sum_i coef2[i,b]*in_i; bf16 = bf16(out1*scale[b])."""
    n_in = len(inputs)
    x = inputs[0]
    B = x.shape[0]
    E = x.numel() // B
    for t in inputs:
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape
    coef1 = coef1.to(torch.float32).contiguous()
    assert coef1.shape == (n_in, B), (coef1.shape, n_in, B)
    if coef2 is not None:
        coef2 = coef2.to(torch.float32).contiguous()
    arr = (ctypes.c_void_p * n_in)(*[t.data_ptr() for t in inputs])
    out1 = torch.empty_like(x) if want_out1 else None
    out2 = torch.empty_like(x) if coef2 is not None else None
    outb = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    lo, hi = (clip if clip is not None else (0.0, 0.0))
    check(load().fdx_affine_combine(n_in, arr, ptr(coef1), ptr(coef2),
                                    ptr(_f32c(bf16_scale)) if bf16_scale is not None else ptr(None),
                                    B, E, ptr(out1), ptr(out2), ptr(outb), int(clip is not None), lo, hi,
                                    stream_ptr()), "affine_combine")
    return out1, out2, outb


# --------------------------------------------------------------------------- jax.random's threefry streams
def _random(entry: str, key, shape, dtype, device, out, *args):
    """Common part of the random_* wrappers.  `key`: two host ints, or a (2,) int32 CUDA tensor holding the two
    words (read by the kernel when it runs: the form a captured graph takes)."""
    shape = (shape,) if isinstance(shape, int) else tuple(int(d) for d in shape)
    if any(d < 0 for d in shape):
        raise _lib.FdxError(f"{entry}: negative dimension in shape {shape}")
    n = 1
    for d in shape:
        n *= d
    if out is None:
        device = torch.device("cuda" if device is None else device)
        if device.type != "cuda":
            raise _lib.FdxError(f"{entry}: expected a CUDA device (flaxdiff_b200 has no CPU path)")
        out = torch.empty(shape, dtype=dtype, device=device)
    elif out.dtype != dtype or out.numel() != n or not out.is_contiguous():
        raise _lib.FdxError(f"{entry}: out must be a contiguous {dtype} tensor of {n} elements")
    if isinstance(key, torch.Tensor):
        if key.dtype != torch.int32 or key.numel() != 2 or not key.is_contiguous():
            raise _lib.FdxError(f"{entry}: a device key is a contiguous (2,) int32 tensor")
        k0, k1, key_dev = 0, 0, ptr(key)
    else:
        k0, k1, key_dev = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF, ptr(None)
    check(getattr(load(), "fdx_" + entry)(k0, k1, key_dev, n, *args, ptr(out), stream_ptr()), entry)
    return out


def random_bits(key, shape, device=None, out=None) -> torch.Tensor:
    """jax.random.bits(key, shape, uint32); the words are returned in an int32 tensor (same bits)."""
    return _random("random_bits", key, shape, torch.int32, device, out)


def random_uniform(key, shape, minval: float = 0.0, maxval: float = 1.0, device=None, out=None) -> torch.Tensor:
    """jax.random.uniform(key, shape, float32, minval, maxval)."""
    return _random("random_uniform", key, shape, torch.float32, device, out, minval, maxval)


def random_normal(key, shape, device=None, out=None) -> torch.Tensor:
    """jax.random.normal(key, shape, float32)."""
    return _random("random_normal", key, shape, torch.float32, device, out)


def random_randint(key, shape, minval: int, maxval: int, device=None, out=None) -> torch.Tensor:
    """jax.random.randint(key, shape, minval, maxval, int32), minval < maxval."""
    return _random("random_randint", key, shape, torch.int32, device, out, int(minval), int(maxval))


def adamw_ema_step(p, g, m, v, ema, shadow, lr, b1, b2, eps, weight_decay, step, ema_decay,
                   grad_scale: float = 1.0, gnorm_sq=None, clip_norm: float = 0.0, dyn=None):
    check(load().fdx_adamw_ema_step(ptr(p), ptr(g), ptr(m), ptr(v), ptr(ema), ptr(shadow), p.numel(), lr, b1, b2,
                                    eps, weight_decay, step, ema_decay, grad_scale, ptr(gnorm_sq), clip_norm,
                                    ptr(dyn), stream_ptr()), "adamw_ema_step")


def optimizer_step(kind: int, p, g, m, v, ema, shadow, lr, b1, b2, eps, weight_decay, step, ema_decay=0.999,
                   grad_scale: float = 1.0, gstats=None, clip_norm: float = 0.0, dyn=None, dynscale=None,
                   seg_offsets=None, seg_norms=None, u_ws=None):
    """fdx_optimizer_step: adam / adamw / lamb update (+ optional EMA, bf16 shadow refresh, global-norm clip,
    DynamicScale unscale-and-skip) over the flat buffers.  `ema=None` = TrainState.apply_gradients alone."""
    d = _lib.fdx_opt_desc()
    d.kind = kind
    d.p, d.g, d.m, d.v = ptr(p), ptr(g), ptr(m), ptr(v)
    d.ema, d.shadow_bf16, d.n = ptr(ema), ptr(shadow), p.numel()
    d.lr, d.b1, d.b2, d.eps, d.weight_decay = lr, b1, b2, eps, weight_decay
    d.step, d.ema_decay, d.grad_scale = step, ema_decay, grad_scale
    d.gstats, d.clip_norm, d.dyn_lr_bc, d.dynscale = ptr(gstats), clip_norm, ptr(dyn), ptr(dynscale)
    if seg_offsets is not None:
        assert seg_offsets.dtype == torch.int64
        d.seg_offsets, d.nseg = ptr(seg_offsets), seg_offsets.numel()
        d.seg_norms, d.u_ws = ptr(seg_norms), ptr(u_ws)
    check(load().fdx_optimizer_step(d, stream_ptr()), "optimizer_step")


def ema_update(ema: torch.Tensor, p: torch.Tensor, decay: float):
    """ema = decay * ema + (1 - decay) * p over the flat buffers (TrainState.apply_ema)."""
    check(load().fdx_ema_update(ptr(ema), ptr(p), p.numel(), decay, stream_ptr()), "ema_update")


def grad_stats(g: torch.Tensor, dynscale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """-> f32[2] = (sum (g / dynscale[0])^2 or sum g^2, number of non-finite elements of g).  Pass the same
    DynamicScale state as to optimizer_step: its clip reads the norm with the loss scale removed."""
    out = torch.empty(2, dtype=torch.float32, device=g.device)
    check(load().fdx_grad_stats(ptr(g), g.numel(), ptr(dynscale), ptr(out), stream_ptr()), "grad_stats")
    return out


def sumsq(g: torch.Tensor) -> torch.Tensor:
    return grad_stats(g)


def dynscale_update(state3: torch.Tensor, gstats: torch.Tensor, growth_factor=2.0, backoff_factor=0.5,
                    growth_interval=2000, minimum_scale=1.1754943508222875e-38):
    check(load().fdx_dynscale_update(ptr(state3), ptr(gstats), growth_factor, backoff_factor, growth_interval,
                                     minimum_scale, stream_ptr()), "dynscale_update")


# --------------------------------------------------------------------------- data-parallel exchange
class Comm:
    """fdx_comm handle: NCCL communicator bound inside libfdx (one per process).  `unique_id()` on rank 0,
    broadcast the 128 bytes by any side channel, then `Comm(rank, world, id)` on every rank."""

    @staticmethod
    def unique_id() -> bytes:
        buf = ctypes.create_string_buffer(128)
        check(load().fdx_comm_unique_id(buf), "comm_unique_id")
        return buf.raw

    def __init__(self, rank: int, world: int, uid: bytes):
        assert len(uid) == 128
        self._h = ctypes.c_void_p()
        check(load().fdx_comm_init(ctypes.byref(self._h), rank, world, ctypes.create_string_buffer(uid, 128)),
              "comm_init")
        self.rank, self.world = rank, world

    def allreduce_avg_(self, buf: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """In-place mean over ranks of a contiguous f32 CUDA tensor (a bucket of the flat gradient buffer)."""
        assert buf.dtype == torch.float32 and buf.is_contiguous()
        st = ctypes.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
        check(load().fdx_comm_allreduce_avg(self._h, ptr(buf), buf.numel(), st), "comm_allreduce_avg")
        return buf

    def destroy(self):
        if self._h:
            check(load().fdx_comm_destroy(self._h), "comm_destroy")
            self._h = ctypes.c_void_p()


def nccl_version() -> int:
    return int(load().fdx_comm_nccl_version())


def cast_f32_bf16(src: torch.Tensor, dst: Optional[torch.Tensor] = None) -> torch.Tensor:
    assert src.dtype == torch.float32 and src.is_contiguous()
    if dst is None:
        dst = torch.empty(tuple(src.shape), dtype=torch.bfloat16, device=src.device)
    check(load().fdx_cast_f32_bf16(ptr(src), ptr(dst), src.numel(), stream_ptr()), "cast_f32_bf16")
    return dst


def upsample2x(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_upsample2x(act(x, "x"), act(out, "out"), stream_ptr()), "upsample2x")
    return out


def upsample2x_bwd(dy: torch.Tensor, dx: torch.Tensor, accumulate: bool = False) -> torch.Tensor:
    check(load().fdx_upsample2x_bwd(act(dy, "dy"), act(dx, "dx"), int(accumulate), stream_ptr()), "upsample2x_bwd")
    return dx


def act_add(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    check(load().fdx_act_add(act(a, "a"), act(b, "b"), act(out, "out"), stream_ptr()), "act_add")
    return out


def colsum(x: torch.Tensor, per_image: bool, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        shape = (x.shape[0], x.shape[-1]) if per_image else (x.shape[-1],)
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    check(load().fdx_colsum(act(x, "x"), ptr(out), int(per_image), stream_ptr()), "colsum")
    return out


# --------------------------------------------------------------------------- upsample + conv (sub-pixel)
def upconv3x3_pack(w_hwio: torch.Tensor) -> torch.Tensor:
    """bf16 [16][Cin][Cout] parity/tap-summed weights of nearest-2x + conv3x3 from the f32 HWIO kernel."""
    assert w_hwio.dtype == torch.float32 and w_hwio.is_contiguous() and w_hwio.shape[:2] == (3, 3)
    cin, cout = w_hwio.shape[2], w_hwio.shape[3]
    weff = torch.empty((16, cin, cout), dtype=torch.bfloat16, device=w_hwio.device)
    check(load().fdx_upconv3x3_pack(ptr(w_hwio), cin, cout, ptr(weff), stream_ptr()), "upconv3x3_pack")
    return weff


def upconv3x3_fwd(x: torch.Tensor, weff: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                  colstats=None) -> torch.Tensor:
    """out[B,2h,2w,Cout] = conv3x3_SAME(nearest2x(x)) + bias, without the upsampled tensor."""
    if colstats is not None:
        d = colstats[0].desc(colstats[1])
        check(load().fdx_upconv3x3_fwd_stats(act(x, "x"), ptr(weff), ptr(bias), act(out, "out"), d, stream_ptr()),
              "upconv3x3_fwd_stats")
        return out
    check(load().fdx_upconv3x3_fwd(act(x, "x"), ptr(weff), ptr(bias), act(out, "out"), stream_ptr()),
          "upconv3x3_fwd")
    return out


def upconv3x3_dgrad(dy: torch.Tensor, weff: torch.Tensor, dx: torch.Tensor, accumulate: bool = False) -> torch.Tensor:
    check(load().fdx_upconv3x3_dgrad(act(dy, "dy"), ptr(weff), act(dx, "dx"), int(accumulate), stream_ptr()),
          "upconv3x3_dgrad")
    return dx


def upconv3x3_wgrad(x: torch.Tensor, dy: torch.Tensor, dw_hwio: torch.Tensor) -> torch.Tensor:
    """Accumulates d(loss)/dw of the 3x3 kernel (f32 HWIO) into dw_hwio."""
    assert dw_hwio.dtype == torch.float32 and dw_hwio.is_contiguous()
    ws = torch.empty((16, x.shape[-1], dy.shape[-1]), dtype=torch.float32, device=x.device)
    check(load().fdx_upconv3x3_wgrad(act(x, "x"), act(dy, "dy"), ptr(ws), ptr(dw_hwio), stream_ptr()),
          "upconv3x3_wgrad")
    return dw_hwio


# --------------------------------------------------------------------------- 3-channel convs
def conv_in_fwd(x_bf16: torch.Tensor, w: torch.Tensor, bias, out: torch.Tensor,
                w_bf16: Optional[torch.Tensor] = None) -> torch.Tensor:
    """conv_in 3->Cout as im2col (K = 27 padded to 32) + one tensor-core GEMM with the bias fused."""
    n, h, w_, c = x_bf16.shape
    assert c == 3 and x_bf16.dtype == torch.bfloat16 and x_bf16.is_contiguous()
    cout = out.shape[-1]
    col = im2col3(x_bf16, +1, False)
    wb = w_bf16 if w_bf16 is not None else cast_f32_bf16(w)
    gemm(GEMM_KMN, col, wb, out, n * h * w_, cout, 27, 32, cout, out.stride(2), bias=bias)
    return out


def conv_in_fwd_direct(x_bf16: torch.Tensor, w: torch.Tensor, bias, out: torch.Tensor) -> torch.Tensor:
    """Workspace-free CUDA-core variant (fdx_conv_in_fwd)."""
    n, h, w_, c = x_bf16.shape
    assert c == 3 and x_bf16.dtype == torch.bfloat16 and x_bf16.is_contiguous()
    assert w.dtype == torch.float32 and w.is_contiguous()
    check(load().fdx_conv_in_fwd(ptr(x_bf16), n, h, w_, ptr(w), ptr(bias), act(out, "out"), stream_ptr()),
          "conv_in_fwd")
    return out


def im2col3(src: torch.Tensor, sgn: int, ones_col: bool) -> torch.Tensor:
    n, h, w, c = src.shape
    assert c == 3 and src.is_contiguous() and src.dtype in (torch.float32, torch.bfloat16)
    col = torch.empty((n * h * w, 32), dtype=torch.bfloat16, device=src.device)
    check(load().fdx_im2col3x3_c3(ptr(src), int(src.dtype == torch.float32), sgn, n, h, w, int(ones_col), ptr(col),
                                  stream_ptr()), "im2col3x3_c3")
    return col


def conv_in_wgrad(x_bf16, dy, dw, dbias):
    """dW[t][cs][co] (+ bias row) = im2col(x)^T @ dY on the tensor cores; accumulates into dw / dbias."""
    n, h, w, cout = dy.shape
    P = n * h * w
    col = im2col3(x_bf16, +1, True)
    tmp = torch.zeros((32, cout), dtype=torch.float32, device=dy.device)
    gemm(GEMM_MNMN, col, dy, tmp, 32, cout, P, 32, dy.stride(2), cout, atomic=True, reduce_batch=True)
    dw.view(27, cout).add_(tmp[:27])
    if dbias is not None:
        dbias.add_(tmp[27])


def conv_in_wgrad_direct(x_bf16, dy, dw, dbias):
    """Workspace-free CUDA-core variant (fdx_conv_in_wgrad)."""
    check(load().fdx_conv_in_wgrad(ptr(x_bf16), act(dy, "dy"), ptr(dw), ptr(dbias), stream_ptr()), "conv_in_wgrad")


def conv_out_fwd(x: torch.Tensor, w: torch.Tensor, bias) -> torch.Tensor:
    """conv_out Cin->3: one tensor-core GEMM (pixels x Cin)(Cin x 27, padded to 32) with f32 output, then the
    col2im scatter that adds the nine taps' partial sums and the bias."""
    n, h, w_, cin = x.shape
    wr = torch.zeros((cin, 32), dtype=torch.float32, device=x.device)
    wr[:, :27] = w.reshape(9, cin, 3).permute(1, 0, 2).reshape(cin, 27)       # [ci][(t,k)]
    col = torch.empty((n * h * w_, 32), dtype=torch.float32, device=x.device)
    gemm(GEMM_KMN, x, cast_f32_bf16(wr), col, n * h * w_, 32, cin, x.stride(2), 32, 32)
    return col2im3(col, bias, n, h, w_)


def col2im3(col: torch.Tensor, bias, n: int, h: int, w: int) -> torch.Tensor:
    """y f32 (n, h, w, 3) = bias + the nine taps' partial sums of col f32 [n*h*w, 32] (column t*3+k), SAME padding."""
    y = torch.empty((n, h, w, 3), dtype=torch.float32, device=col.device)
    check(load().fdx_col2im3x3_c3(ptr(col), ptr(bias), n, h, w, ptr(y), stream_ptr()), "col2im3x3_c3")
    return y


def conv_out_fwd_direct(x: torch.Tensor, w: torch.Tensor, bias) -> torch.Tensor:
    """Workspace-free CUDA-core variant (fdx_conv_out_fwd)."""
    n, h, w_, c = x.shape
    y = torch.empty((n, h, w_, 3), dtype=torch.float32, device=x.device)
    check(load().fdx_conv_out_fwd(act(x, "x"), ptr(w), ptr(bias), ptr(y), stream_ptr()), "conv_out_fwd")
    return y


def conv_out_dgrad(dF: torch.Tensor, w: torch.Tensor, dx: torch.Tensor, col: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dx[p][ci] = sum_{t,k} dF[p - d(t)][k] w[t][ci][k]: im2col(dF) (shared with the weight gradient)
    times the (27 x Cin) re-arranged kernel on the tensor cores."""
    n, h, w_, cin = dx.shape
    if col is None:
        col = im2col3(dF, -1, False)
    wt = w.reshape(9, cin, 3).permute(0, 2, 1).reshape(27, cin).contiguous()      # [(t,k)][ci], 1.7 K elements
    gemm(GEMM_KMN, col, cast_f32_bf16(_pad4(wt)), dx, n * h * w_, cin, 27, 32, cin, dx.stride(2))
    return dx


def _pad4(t: torch.Tensor) -> torch.Tensor:
    return t if t.numel() % 4 == 0 else torch.nn.functional.pad(t.reshape(-1), (0, 4 - t.numel() % 4)).reshape(-1)


def conv_out_dgrad_direct(dF: torch.Tensor, w: torch.Tensor, dx: torch.Tensor) -> torch.Tensor:
    check(load().fdx_conv_out_dgrad(ptr(dF), ptr(w), act(dx, "dx"), stream_ptr()), "conv_out_dgrad")
    return dx


def conv_out_wgrad(x, dF, dw, dbias, col: Optional[torch.Tensor] = None):
    """dW[t][ci][k] = x^T @ im2col(dF) on the tensor cores; accumulates into dw / dbias."""
    n, h, w, cin = x.shape
    P = n * h * w
    if col is None:
        col = im2col3(dF, -1, False)
    tmp = torch.zeros((cin, 32), dtype=torch.float32, device=x.device)
    gemm(GEMM_MNMN, x, col, tmp, cin, 32, P, x.stride(2), 32, 32, atomic=True, reduce_batch=True)
    dw.add_(tmp[:, :27].view(cin, 9, 3).permute(1, 0, 2).reshape(3, 3, cin, 3))
    if dbias is not None:
        cs = colsum(col.view(n, h, w, 32), per_image=False)
        dbias.add_(cs[12:15])        # centre tap (t = 4) columns = sum over pixels of dF


def conv_out_wgrad_direct(x, dF, dw, dbias):
    """Workspace-free CUDA-core variant (fdx_conv_out_wgrad)."""
    check(load().fdx_conv_out_wgrad(act(x, "x"), ptr(dF), ptr(dw), ptr(dbias), stream_ptr()), "conv_out_wgrad")


# --------------------------------------------------------------------------- GEGLU
def geglu_fwd(u: torch.Tensor) -> torch.Tensor:
    """u [rows, 2*inner] bf16 -> hidden_linear * gelu_tanh(hidden_gelu) [rows, inner]."""
    rows, two = u.shape
    assert u.dtype == torch.bfloat16 and u.is_contiguous() and two % 16 == 0
    g = torch.empty((rows, two // 2), dtype=torch.bfloat16, device=u.device)
    check(load().fdx_geglu_fwd(ptr(u), rows, two // 2, ptr(g), stream_ptr()), "geglu_fwd")
    return g


def geglu_bwd(u: torch.Tensor, dg: torch.Tensor) -> torch.Tensor:
    rows, two = u.shape
    assert dg.shape == (rows, two // 2) and dg.is_contiguous() and dg.dtype == torch.bfloat16
    du = torch.empty_like(u)
    check(load().fdx_geglu_bwd(ptr(u), ptr(dg), rows, two // 2, ptr(du), stream_ptr()), "geglu_bwd")
    return du


def colsum_rows(x2d: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[c] = sum over rows of x2d[:, c] (bias gradients of dense layers); columns in slabs of <= 2048."""
    rows, n = x2d.shape
    assert x2d.stride(1) == 1 and out.numel() == n
    for c0 in range(0, n, 2048):
        c1 = min(n, c0 + 2048)
        colsum(x2d[:, c0:c1].unsqueeze(0).unsqueeze(0), False, out=out[c0:c1])
    return out


# --------------------------------------------------------------------------- fused attention
def _attn_desc(q, k, v, o, lse, heads: int, dh: int, scale: float):
    """q / o: [B, L, heads*dh], k / v: [B, Lk, heads*dh] (bf16, last dim contiguous)."""
    B, L, HD = q.shape
    Lk = k.shape[1]
    assert HD == heads * dh and k.shape[2] == HD and v.shape == k.shape and o.shape == q.shape
    for t in (q, k, v, o):
        assert t.dtype == torch.bfloat16 and t.stride(2) == 1
    a = _lib.fdx_attn_desc()
    a.B, a.heads, a.L, a.Lk, a.dh, a.scale = B, heads, L, Lk, dh, scale
    a.q, a.q_ld, a.q_bs = ptr(q), q.stride(1), q.stride(0)
    a.k, a.k_ld, a.k_bs = ptr(k), k.stride(1), k.stride(0)
    a.v, a.v_ld, a.v_bs = ptr(v), v.stride(1), v.stride(0)
    a.o, a.o_ld, a.o_bs = ptr(o), o.stride(1), o.stride(0)
    a.lse = ptr(lse)
    return a


def attention_fwd(q, k, v, heads: int, dh: int, scale: float, out=None):
    """o = softmax(q k^T * scale) v per (image, head) - fdx_attention_fwd.  -> (o bf16 [B, L, heads*dh],
    lse f32 [B, heads, L]).  No (B, h, L, Lk) tensor exists in HBM."""
    B, L, HD = q.shape
    o = out if out is not None else torch.empty((B, L, HD), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, heads, L), dtype=torch.float32, device=q.device)
    a = _attn_desc(q, k, v, o, lse, heads, dh, scale)
    check(load().fdx_attention_fwd(a, stream_ptr()), "attention_fwd")
    return o, lse


def attention_bwd(q, k, v, o, lse, d_o, heads: int, dh: int, scale: float):
    """-> (dq [B, L, HD], dk, dv [B, Lk, HD]) bf16 - fdx_attention_bwd (S / P recomputed on chip)."""
    assert d_o.shape == q.shape and d_o.dtype == torch.bfloat16 and d_o.stride(2) == 1
    dq = torch.empty_like(q, memory_format=torch.contiguous_format)
    dk = torch.empty(tuple(k.shape), dtype=torch.bfloat16, device=k.device)
    dv = torch.empty(tuple(v.shape), dtype=torch.bfloat16, device=v.device)
    ws = torch.empty_like(lse)
    a = _attn_desc(q, k, v, o, lse, heads, dh, scale)
    a.d_o, a.do_ld, a.do_bs = ptr(d_o), d_o.stride(1), d_o.stride(0)
    a.dvec_ws = ptr(ws)
    a.dq, a.dq_ld, a.dq_bs = ptr(dq), dq.stride(1), dq.stride(0)
    a.dk, a.dk_ld, a.dk_bs = ptr(dk), dk.stride(1), dk.stride(0)
    a.dv, a.dv_ld, a.dv_bs = ptr(dv), dv.stride(1), dv.stride(0)
    check(load().fdx_attention_bwd(a, stream_ptr()), "attention_bwd")
    return dq, dk, dv


def attention_fwd_masked(q, k, v, heads: int, dh: int, scale: float, causal: bool,
                         key_mask: Optional[torch.Tensor] = None, out=None) -> torch.Tensor:
    """fdx_attention_fwd_masked: key j is allowed for query i iff (not causal or j <= i) and key_mask[b][j];
    key_mask int32 [B, Lk] or None.  A row with no allowed key is zeros.  -> o bf16 [B, L, heads*dh]."""
    B, L, HD = q.shape
    if key_mask is not None:
        assert key_mask.dtype == torch.int32 and key_mask.is_contiguous() and key_mask.shape == (B, k.shape[1])
    o = out if out is not None else torch.empty((B, L, HD), dtype=torch.bfloat16, device=q.device)
    a = _attn_desc(q, k, v, o, None, heads, dh, scale)
    check(load().fdx_attention_fwd_masked(a, int(causal), ptr(key_mask), stream_ptr()),
          "attention_fwd_masked")
    return o


# --------------------------------------------------------------------------- CLIP text tower
def token_embed(ids: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor, out=None) -> torch.Tensor:
    """bf16(tok[ids] + pos[t]) -> [B, T, D]; ids int32 [B, T]; an id outside [0, vocab) gives a NaN row."""
    B, T = ids.shape
    vocab, D = tok.shape
    assert ids.dtype == torch.int32 and ids.is_contiguous() and tok.dtype == pos.dtype == torch.float32
    assert tok.is_contiguous() and pos.is_contiguous() and pos.shape[1] == D and pos.shape[0] >= T
    if out is None:
        out = torch.empty((B, T, D), dtype=torch.bfloat16, device=ids.device)
    assert out.is_contiguous() and out.shape == (B, T, D)
    check(load().fdx_token_embed(ptr(ids), B, T, ptr(tok), vocab, ptr(pos), D, ptr(out), stream_ptr()),
          "token_embed")
    return out


def layernorm_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, out=None) -> torch.Tensor:
    """nn.LayerNorm over the last axis of a contiguous bf16 tensor; gamma / beta f32."""
    C = x.shape[-1]
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and gamma.dtype == beta.dtype == torch.float32
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    assert out.is_contiguous() and out.shape == x.shape
    check(load().fdx_layernorm_fwd(ptr(x), x.numel() // C, C, ptr(gamma), ptr(beta), eps, ptr(out), stream_ptr()),
          "layernorm_fwd")
    return out


def bias_act(x: torch.Tensor, bias: Optional[torch.Tensor], act_kind: int, out=None) -> torch.Tensor:
    """act(x + bias) over the last axis (_lib.ACT_QUICK_GELU / ACT_GELU / ACT_GELU_TANH); out may be x."""
    C = x.shape[-1]
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and (bias is None or bias.dtype == torch.float32)
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    assert out.is_contiguous() and out.shape == x.shape
    check(load().fdx_bias_act(ptr(x), x.numel() // C, C, ptr(bias), act_kind, ptr(out), stream_ptr()), "bias_act")
    return out


def bias_act_bwd(x: torch.Tensor, bias: Optional[torch.Tensor], act_kind: int, dy: torch.Tensor, out=None) -> torch.Tensor:
    """dx = dy * act'(x + bias) (act_kind = _lib.ACT_GELU_TANH)."""
    C = x.shape[-1]
    assert x.dtype == dy.dtype == torch.bfloat16 and x.is_contiguous() and dy.is_contiguous() and dy.shape == x.shape
    if out is None:
        out = torch.empty(tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_bias_act_bwd(ptr(x), x.numel() // C, C, ptr(bias), act_kind, ptr(dy), ptr(out), stream_ptr()),
          "bias_act_bwd")
    return out


# --------------------------------------------------------------------------- SimpleDiT streaming kernels
def _dit_chunks(B: int, L: int, C: int, device) -> int:
    """Token chunks per sample of the two-stage column sums: enough blocks for eight per SM, chunks of >= 32 rows."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    blocks = -(-C // 64) * B
    return max(1, min(-(-L // 32), -(-8 * sms // blocks)))


def _tokens(t: torch.Tensor, name: str):
    assert t.dtype == torch.bfloat16 and t.dim() == 2 and t.is_contiguous(), (name, t.dtype, t.shape, t.stride())
    return t.shape


def dit_adaln_fwd(x: torch.Tensor, L: int, ada: Optional[torch.Tensor] = None, scale_off: int = 0,
                  shift_off: int = 0, gamma=None, beta=None, eps: float = 1e-5, stats: bool = True, out=None):
    """adaLN LayerNorm of the token rows x [B*L, C] -> (y bf16, mean f32 [rows] or None, rstd or None)."""
    rows, C = _tokens(x, "x")
    y = out if out is not None else torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device) if stats else None
    rstd = torch.empty_like(mean) if stats else None
    a, ld = (ada, ada.stride(0)) if ada is not None else (None, 0)
    check(load().fdx_dit_adaln_fwd(ptr(x), rows, L, C, ptr(a), ld, scale_off, shift_off, ptr(gamma), ptr(beta), eps,
                                   ptr(y), ptr(mean), ptr(rstd), stream_ptr()), "dit_adaln_fwd")
    return y, mean, rstd


def dit_adaln_bwd(x, dy, L: int, mean, rstd, d0: torch.Tensor, d1: torch.Tensor, ada=None, scale_off: int = 0,
                  gamma=None, addend=None, out=None, reduce_samples: bool = False, accumulate: bool = False):
    """Backward of dit_adaln_fwd -> dx bf16 [rows, C] (+ addend).  d0 / d1: f32 [B, >= C] row views (the d(scale) /
    d(shift) chunks of d_ada) or, reduce_samples, f32 [C] (d(gamma) / d(beta))."""
    rows, C = _tokens(x, "x")
    _tokens(dy, "dy")
    B = rows // L
    dx = out if out is not None else torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    nch = _dit_chunks(B, L, C, x.device)
    ws = torch.empty(B * nch * 2 * C, dtype=torch.float32, device=x.device)
    a, ld = (ada, ada.stride(0)) if ada is not None else (None, 0)
    ld0 = d0.stride(0) if d0.dim() == 2 else 0
    ld1 = d1.stride(0) if d1.dim() == 2 else 0
    check(load().fdx_dit_adaln_bwd(ptr(x), ptr(dy), rows, L, C, ptr(a), ld, scale_off, ptr(gamma), ptr(mean),
                                   ptr(rstd), ptr(addend), ptr(dx), ptr(ws), nch, ptr(d0), ld0, ptr(d1), ld1,
                                   int(reduce_samples), int(accumulate), stream_ptr()), "dit_adaln_bwd")
    return dx


def dit_gate_fwd(x: torch.Tensor, y: torch.Tensor, L: int, gate: torch.Tensor, out=None) -> torch.Tensor:
    """x + gate[b] * y over token rows [B*L, C]; gate an f32 [B, C] row view (a chunk of the ada rows)."""
    rows, C = _tokens(x, "x")
    _tokens(y, "y")
    assert gate.dtype == torch.float32 and gate.stride(1) == 1
    out = out if out is not None else torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_dit_gate_fwd(ptr(x), ptr(y), rows, L, C, ptr(gate), gate.stride(0), ptr(out), stream_ptr()),
          "dit_gate_fwd")
    return out


def dit_gate_bwd(dout: torch.Tensor, y: torch.Tensor, L: int, gate: torch.Tensor, dgate: torch.Tensor) -> torch.Tensor:
    """-> dy = gate[b] * dout; writes dgate[b] = sum over the sample's tokens of dout * y (f32 [B, C] row view)."""
    rows, C = _tokens(dout, "dout")
    _tokens(y, "y")
    B = rows // L
    dy = torch.empty((rows, C), dtype=torch.bfloat16, device=dout.device)
    nch = _dit_chunks(B, L, C, dout.device)
    ws = torch.empty(B * nch * 2 * C, dtype=torch.float32, device=dout.device)
    check(load().fdx_dit_gate_bwd(ptr(dout), ptr(y), rows, L, C, ptr(gate), gate.stride(0), ptr(dy), ptr(ws), nch,
                                  ptr(dgate), dgate.stride(0), stream_ptr()), "dit_gate_bwd")
    return dy


def dit_token_mean(x: torch.Tensor) -> torch.Tensor:
    """f32 [B, C] mean over the tokens of x bf16 [B, T, C]."""
    B, T, C = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous()
    nch = _dit_chunks(B, T, C, x.device)
    ws = torch.empty(B * nch * 2 * C, dtype=torch.float32, device=x.device)
    out = torch.empty((B, C), dtype=torch.float32, device=x.device)
    check(load().fdx_dit_token_mean(ptr(x), B, T, C, ptr(ws), nch, ptr(out), stream_ptr()), "dit_token_mean")
    return out


def dit_rope(t: torch.Tensor, L: int, heads: int, d: int, dp: int, nmat: int = 1, mat_off: int = 0,
             inverse: bool = False) -> torch.Tensor:
    """RoPE in place on nmat head matrices (mat_off columns apart) of the bf16 rows of t [rows, >= ...]."""
    assert t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1
    check(load().fdx_dit_rope(ptr(t), t.shape[0], L, t.stride(0), heads, d, dp, nmat, mat_off, int(inverse),
                              stream_ptr()), "dit_rope")
    return t


def dit_patchify(x: torch.Tensor, p: int, ld: int) -> torch.Tensor:
    """(B, H, W, C) f32 / bf16 -> bf16 [B*(H/p)*(W/p), ld] patch rows (zeros past p*p*C)."""
    B, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype in (torch.float32, torch.bfloat16)
    out = torch.empty((B * (H // p) * (W // p), ld), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_dit_patchify(ptr(x), int(x.dtype == torch.float32), B, H, W, C, p, ld, ptr(out),
                                  stream_ptr()), "dit_patchify")
    return out


def dit_unpatchify(y: torch.Tensor, B: int, H: int, W: int, C: int, p: int) -> torch.Tensor:
    """f32 rows [B*L, ld] -> f32 (B, H, W, C)."""
    assert y.dtype == torch.float32 and y.dim() == 2 and y.stride(1) == 1
    out = torch.empty((B, H, W, C), dtype=torch.float32, device=y.device)
    check(load().fdx_dit_unpatchify(ptr(y), y.stride(0), B, H, W, C, p, ptr(out), stream_ptr()), "dit_unpatchify")
    return out


def dit_fourier(t: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    """bf16 [B, 2*len(freqs)] = [sin(2 pi t freqs), cos(2 pi t freqs)]."""
    t = _f32c(t)
    assert freqs.dtype == torch.float32 and freqs.is_contiguous()
    out = torch.empty((t.numel(), 2 * freqs.numel()), dtype=torch.bfloat16, device=t.device)
    check(load().fdx_dit_fourier(ptr(t), t.numel(), ptr(freqs), freqs.numel(), ptr(out), stream_ptr()),
          "dit_fourier")
    return out


# --------------------------------------------------------------------------- SimpleMMDiT streaming kernels
def _ada_rows(ada: torch.Tensor, C: int, name: str):
    assert ada.dtype == torch.float32 and ada.dim() == 2 and ada.stride(1) == 1 and ada.shape[1] >= 6 * C, name
    return ada.stride(0)


def mmdit_adaln_fwd(x: torch.Tensor, L: int, ada: torch.Tensor, eps: float = 1e-5, stats: bool = True):
    """One LayerNorm of the token rows x [B*L, C], modulated twice by the ada rows f32 [B, 6C] -> (y_attn bf16,
    y_mlp bf16 (clipped mlp chunks), mean f32 [rows] or None, rstd or None)."""
    rows, C = _tokens(x, "x")
    ya = torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    ym = torch.empty_like(ya)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device) if stats else None
    rstd = torch.empty_like(mean) if stats else None
    check(load().fdx_mmdit_adaln_fwd(ptr(x), rows, L, C, ptr(ada), _ada_rows(ada, C, "ada"), eps, ptr(ya), ptr(ym),
                                     ptr(mean), ptr(rstd), stream_ptr()), "mmdit_adaln_fwd")
    return ya, ym, mean, rstd


def mmdit_adaln_bwd(x, dya, dym, L: int, ada: torch.Tensor, mean, rstd, dada: torch.Tensor, addend=None, out=None):
    """Backward of mmdit_adaln_fwd -> dx bf16 [rows, C] (+ addend); writes the scale / shift chunks of both
    modulations into dada f32 [B, 6C]."""
    rows, C = _tokens(x, "x")
    _tokens(dya, "dy_attn")
    _tokens(dym, "dy_mlp")
    B = rows // L
    dx = out if out is not None else torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    nch = _dit_chunks(B, L, C, x.device)
    ws = torch.empty(B * nch * 4 * C, dtype=torch.float32, device=x.device)
    check(load().fdx_mmdit_adaln_bwd(ptr(x), ptr(dya), ptr(dym), rows, L, C, ptr(ada), _ada_rows(ada, C, "ada"),
                                     ptr(mean), ptr(rstd), ptr(addend), ptr(dx), ptr(ws), nch, ptr(dada),
                                     _ada_rows(dada, C, "dada"), stream_ptr()), "mmdit_adaln_bwd")
    return dx


def mmdit_gate_fwd(x: torch.Tensor, ya: torch.Tensor, ym: torch.Tensor, L: int, ada: torch.Tensor,
                   out=None) -> torch.Tensor:
    """x + gate_attn[b] * ya + gate_mlp[b] * ym over token rows [B*L, C] (out may be x)."""
    rows, C = _tokens(x, "x")
    _tokens(ya, "y_attn")
    _tokens(ym, "y_mlp")
    out = out if out is not None else torch.empty((rows, C), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_mmdit_gate_fwd(ptr(x), ptr(ya), ptr(ym), rows, L, C, ptr(ada), _ada_rows(ada, C, "ada"),
                                    ptr(out), stream_ptr()), "mmdit_gate_fwd")
    return out


def mmdit_gate_bwd(dout: torch.Tensor, ya: torch.Tensor, ym: torch.Tensor, L: int, ada: torch.Tensor,
                   dada: torch.Tensor):
    """-> (dy_attn = gate_attn[b] * dout, dy_mlp = gate_mlp[b] * dout); writes the gate chunks of dada f32 [B, 6C]
    (the sample's sums of dout * ya and dout * ym)."""
    rows, C = _tokens(dout, "dout")
    _tokens(ya, "y_attn")
    _tokens(ym, "y_mlp")
    B = rows // L
    dya = torch.empty((rows, C), dtype=torch.bfloat16, device=dout.device)
    dym = torch.empty_like(dya)
    nch = _dit_chunks(B, L, C, dout.device)
    ws = torch.empty(B * nch * 2 * C, dtype=torch.float32, device=dout.device)
    check(load().fdx_mmdit_gate_bwd(ptr(dout), ptr(ya), ptr(ym), rows, L, C, ptr(ada), _ada_rows(ada, C, "ada"),
                                    ptr(dya), ptr(dym), ptr(ws), nch, ptr(dada), _ada_rows(dada, C, "dada"),
                                    stream_ptr()), "mmdit_gate_bwd")
    return dya, dym


LN_GATHER, LN_CONCAT, LN_SCATTER = 0, 1, 2       # fdx_layernorm_rows modes


def layernorm_rows_fwd(mode: int, src0: torch.Tensor, src1: Optional[torch.Tensor], rows: int, C: int,
                       gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5, grid=(0, 0)):
    """Affine LayerNorm over logical rows of C columns assembled by `mode` (fdx_layernorm_rows_fwd):
    LN_GATHER - the 2x2 merge of src0's fine rows over the coarse grid `grid` = (HPc, WPc) -> y bf16 [rows, C];
    LN_CONCAT - [src0, src1] -> y bf16 [rows, C]; LN_SCATTER - src0 [rows, C] -> y bf16 fine rows [4 rows, C / 4].
    -> (y, mean f32 [rows], rstd)."""
    for t in (src0, src1):
        assert t is None or (t.dtype == torch.bfloat16 and t.is_contiguous())
    assert gamma.dtype == beta.dtype == torch.float32 and gamma.numel() == C
    C0 = src0.shape[-1] if mode == LN_CONCAT else 0
    shape = (4 * rows, C // 4) if mode == LN_SCATTER else (rows, C)
    y = torch.empty(shape, dtype=torch.bfloat16, device=src0.device)
    mean = torch.empty(rows, dtype=torch.float32, device=src0.device)
    rstd = torch.empty_like(mean)
    check(load().fdx_layernorm_rows_fwd(mode, ptr(src0), ptr(src1), rows, C, C0, grid[0], grid[1], ptr(gamma),
                                        ptr(beta), eps, ptr(y), ptr(mean), ptr(rstd), stream_ptr()),
          "layernorm_rows_fwd")
    return y, mean, rstd


def layernorm_rows_bwd(mode: int, src0, src1, dy: torch.Tensor, rows: int, C: int, gamma, mean, rstd,
                       dgamma: torch.Tensor, dbeta: torch.Tensor, grid=(0, 0), dx0=None, dx1=None,
                       accumulate0: bool = False, accumulate1: bool = False):
    """Backward of layernorm_rows_fwd: dx into dx0 (src0's layout) and, LN_CONCAT, dx1 (src1's), each overwritten or
    added to; dgamma / dbeta f32 [C] += the sums over all rows.  Missing destinations are allocated. -> (dx0, dx1)."""
    assert dy.dtype == torch.bfloat16 and dy.is_contiguous()
    if dx0 is None:
        assert not accumulate0
        dx0 = torch.empty_like(src0)
    if mode == LN_CONCAT and dx1 is None:
        assert not accumulate1
        dx1 = torch.empty_like(src1)
    for t, like in ((dx0, src0), (dx1, src1)):
        assert t is None or (t.dtype == torch.bfloat16 and t.is_contiguous() and t.shape == like.shape)
    C0 = src0.shape[-1] if mode == LN_CONCAT else 0
    sms = torch.cuda.get_device_properties(dy.device).multi_processor_count
    nch = max(1, min(rows, 2 * sms))
    ws = torch.empty(nch * 2 * C, dtype=torch.float32, device=dy.device)
    check(load().fdx_layernorm_rows_bwd(mode, ptr(src0), ptr(src1), ptr(dy), rows, C, C0, grid[0], grid[1],
                                        ptr(gamma), ptr(mean), ptr(rstd), ptr(dx0), int(accumulate0), ptr(dx1),
                                        int(accumulate1), ptr(ws), nch, ptr(dgamma), ptr(dbeta), stream_ptr()),
          "layernorm_rows_bwd")
    return dx0, dx1


# --------------------------------------------------------------------------- S5 state-space layer
def ssm_chunk(B: int, L: int, S: int, device) -> int:
    """Tokens per scan chunk: enough (sample, chunk, state) threads to fill every SM twice, chunks of >= 8 tokens."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    nchunk = max(1, min(-(-L // 8), -(-2048 * sms // (B * S))))
    return -(-L // nchunk)


def ssm_discretize(P: dict, N: int, F: int, wb: torch.Tensor, col0: int, wc: torch.Tensor, adt: torch.Tensor):
    """One direction's discretisation from its f32 leaves P (log_A_real, A_imag, log_dt, B_re, B_im, C_re, C_im):
    writes Bbar^T into columns [col0, col0 + 2N) of wb bf16 [F, ldb], wc bf16 [2N, F] and adt[col0:col0 + 2N]."""
    assert wb.dtype == wc.dtype == torch.bfloat16 and wb.is_contiguous() and wc.is_contiguous()
    assert tuple(wc.shape) == (2 * N, F) and wb.shape[0] == F and adt.dtype == torch.float32
    check(load().fdx_ssm_discretize(ptr(P["log_A_real"]), ptr(P["A_imag"]), ptr(P["log_dt"]), ptr(P["B_re"]),
                                    ptr(P["B_im"]), ptr(P["C_re"]), ptr(P["C_im"]), N, F, ptr(wb), wb.shape[1], col0,
                                    ptr(wc), ptr(adt), stream_ptr()), "ssm_discretize")


def ssm_discretize_bwd(P: dict, G: dict, N: int, F: int, dwb: torch.Tensor, col0: int, dwc: torch.Tensor,
                       dabar: torch.Tensor, dgbar: torch.Tensor):
    """Accumulates one direction's parameter gradients into G (the same leaf names as P) from dwb f32 [>= col0 + 2N, F],
    dwc f32 [2N, F] and the adjoint scan's partial sums dabar / dgbar f32 [parts, ld]."""
    assert dwb.dtype == dwc.dtype == dabar.dtype == dgbar.dtype == torch.float32 and dgbar.shape == dabar.shape
    assert dwb.is_contiguous() and dwc.is_contiguous() and dabar.is_contiguous() and dgbar.is_contiguous()
    assert dwb.shape[1] == F
    check(load().fdx_ssm_discretize_bwd(ptr(P["log_A_real"]), ptr(P["A_imag"]), ptr(P["log_dt"]), ptr(P["B_re"]),
                                        ptr(P["B_im"]), N, F, ptr(dwb), col0, ptr(dwc), ptr(dabar), ptr(dgbar),
                                        dabar.shape[0],
                                        dabar.shape[1], ptr(G["log_A_real"]), ptr(G["A_imag"]), ptr(G["log_dt"]),
                                        ptr(G["B_re"]), ptr(G["B_im"]), ptr(G["C_re"]), ptr(G["C_im"]), stream_ptr()),
          "ssm_discretize_bwd")


def ssm_scan(bu: torch.Tensor, adt: torch.Tensor, B: int, N: int, ndir: int, chunk: int, out=None,
             states: bool = True):
    """bu f32 [B*L, 2*ndir*N] -> (states f32 (into `out`, which may be bu), their bf16 copy).  states=False stores
    only the bf16 copy (what the inference forward reads; the adjoint needs the f32 states) -> (None, bf16 copy)."""
    rows, S2 = bu.shape
    assert bu.dtype == torch.float32 and bu.is_contiguous() and S2 == 2 * ndir * N and rows % B == 0
    assert states or out is None, "ssm_scan: out= names the f32 states, which states=False does not store"
    L = rows // B
    x = None
    if states:
        x = torch.empty_like(bu) if out is None else out
        assert x.shape == bu.shape and x.dtype == torch.float32 and x.is_contiguous()
    x16 = torch.empty((rows, S2), dtype=torch.bfloat16, device=bu.device)
    ws = torch.empty(B * -(-L // chunk) * S2, dtype=torch.float32, device=bu.device)
    check(load().fdx_ssm_scan(ptr(bu), ptr(x), ptr(x16), ptr(adt), B, L, N, ndir, chunk, ptr(ws), stream_ptr()),
          "ssm_scan")
    return x, x16


def ssm_scan_bwd(dx: torch.Tensor, x: torch.Tensor, bu: torch.Tensor, adt: torch.Tensor, B: int, N: int, ndir: int,
                 chunk: int):
    """-> (lambda bf16 [B*L, 2*ndir*N], partial sums f32 [B*nchunk, 2*ndir*N] of lambda conj(x_prev) = d(Abar) and of
    lambda conj(bu))."""
    rows, S2 = dx.shape
    assert dx.dtype == x.dtype == bu.dtype == torch.float32 and x.shape == dx.shape == bu.shape
    assert dx.is_contiguous() and x.is_contiguous() and bu.is_contiguous()
    L = rows // B
    nch = -(-L // chunk)
    lam = torch.empty((rows, S2), dtype=torch.bfloat16, device=dx.device)
    ws = torch.empty(B * nch * S2, dtype=torch.float32, device=dx.device)
    dab = torch.empty((B * nch, S2), dtype=torch.float32, device=dx.device)
    dgb = torch.empty_like(dab)
    check(load().fdx_ssm_scan_bwd(ptr(dx), ptr(x), ptr(bu), ptr(adt), B, L, N, ndir, chunk, ptr(ws), ptr(lam),
                                  ptr(dab), ptr(dgb), stream_ptr()), "ssm_scan_bwd")
    return lam, dab, dgb


def permute_rows(src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """dst[b*L + i] = src[b*L + idx[i]] over the rows of a contiguous 2-D tensor (L = len(idx), int32 on the device)."""
    assert src.dim() == 2 and src.is_contiguous() and idx.dtype == torch.int32 and idx.is_contiguous()
    dst = torch.empty_like(src)
    check(load().fdx_permute_rows(ptr(src), ptr(dst), src.shape[0], idx.numel(), src.shape[1] * src.element_size(),
                                  ptr(idx), stream_ptr()), "permute_rows")
    return dst


# --------------------------------------------------------------------------- CLIP metrics
def clip_image_prep(x: torch.Tensor, tables: torch.Tensor, ksize_y: int, ksize_x: int, lut: torch.Tensor, crop: int,
                    patch: int, ld: int, u8_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """f32 samples [B, H, W, 3] in [-1, 1] -> bf16 patch matrix [B * (crop / patch)^2, ld] (fdx_clip_image_prep);
    u8_out: uint8 [B, crop, crop, 3] receives the resized, cropped image."""
    B, H, W, C = x.shape
    assert C == 3 and x.dtype == torch.float32 and x.is_contiguous()
    assert tables.dtype == torch.int32 and tables.is_contiguous() and lut.dtype == torch.float32 and lut.numel() == 768
    if u8_out is not None:
        assert u8_out.dtype == torch.uint8 and u8_out.is_contiguous() and u8_out.shape == (B, crop, crop, 3)
    G = crop // patch
    out = torch.empty((B * G * G, ld), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_clip_image_prep(ptr(x), B, H, W, ptr(tables), ksize_y, ksize_x, ptr(lut), crop, patch, ld,
                                     ptr(out), ptr(u8_out), stream_ptr()), "clip_image_prep")
    return out


def clip_vision_embed(patch_f32: torch.Tensor, B: int, cls: torch.Tensor, pos: torch.Tensor, gamma: torch.Tensor,
                      beta: torch.Tensor, eps: float) -> torch.Tensor:
    """bf16 [B, G2 + 1, D] = LN([cls; patch embeddings] + pos) from the patch GEMM's f32 [B * G2, D]."""
    rows, D = patch_f32.shape
    G2 = rows // B
    assert patch_f32.dtype == torch.float32 and patch_f32.is_contiguous() and rows == B * G2
    assert tuple(pos.shape) == (G2 + 1, D) and cls.numel() == D
    out = torch.empty((B, G2 + 1, D), dtype=torch.bfloat16, device=patch_f32.device)
    check(load().fdx_clip_vision_embed(ptr(patch_f32), B, G2, D, ptr(cls), ptr(pos), ptr(gamma), ptr(beta), eps,
                                       ptr(out), stream_ptr()), "clip_vision_embed")
    return out


def clip_pool(x: torch.Tensor, ids: Optional[torch.Tensor] = None, gamma: Optional[torch.Tensor] = None,
              beta: Optional[torch.Tensor] = None, eps: float = 1e-5) -> torch.Tensor:
    """bf16 [B, D]: row 0 of each sequence of x [B, T, D] (ids None), or the row at argmax(ids[b]) (int32 [B, T]);
    LayerNorm(gamma, beta) applied when given."""
    B, T, D = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous()
    if ids is not None:
        assert ids.dtype == torch.int32 and ids.is_contiguous() and tuple(ids.shape) == (B, T)
    out = torch.empty((B, D), dtype=torch.bfloat16, device=x.device)
    check(load().fdx_clip_pool(ptr(x), B, T, D, ptr(ids), ptr(gamma), ptr(beta), eps, ptr(out), stream_ptr()),
          "clip_pool")
    return out


def clip_similarity(img: torch.Tensor, txt: torch.Tensor):
    """-> (cos f32 [B], f32 [2] = (mean(1 - cos), mean(100 max(cos, 0)))) of the f32 embeddings [B, P]."""
    B, P = img.shape
    assert img.dtype == txt.dtype == torch.float32 and img.is_contiguous() and txt.is_contiguous()
    assert tuple(txt.shape) == (B, P)
    cos = torch.empty(B, dtype=torch.float32, device=img.device)
    out2 = torch.empty(2, dtype=torch.float32, device=img.device)
    check(load().fdx_clip_similarity(ptr(img), ptr(txt), B, P, ptr(cos), ptr(out2), stream_ptr()), "clip_similarity")
    return cos, out2


# --------------------------------------------------------------------------- temb / softmax
def time_embed_fwd(t, freqs, W1, b1, W2, b2):
    B, D = t.shape[0], W1.shape[0]
    dev = t.device
    four = torch.empty((B, D), dtype=torch.float32, device=dev)
    h1 = torch.empty_like(four)
    h2 = torch.empty_like(four)
    emb = torch.empty_like(four)
    emb16 = torch.empty((B, D), dtype=torch.bfloat16, device=dev)
    check(load().fdx_time_embed_fwd(ptr(_f32c(t)), ptr(freqs), ptr(W1), ptr(b1), ptr(W2), ptr(b2), B, D, ptr(four),
                                    ptr(h1), ptr(h2), ptr(emb), ptr(emb16), stream_ptr()), "time_embed_fwd")
    return emb, emb16, (four, h1, h2)


def time_embed_bwd(demb, saved, W2, dW1, db1, dW2, db2):
    four, h1, h2 = saved
    B, D = demb.shape
    ws1 = torch.empty_like(demb)
    ws2 = torch.empty_like(demb)
    check(load().fdx_time_embed_bwd(ptr(demb), ptr(four), ptr(h1), ptr(h2), ptr(W2), B, D, ptr(ws1), ptr(ws2),
                                    ptr(dW1), ptr(db1), ptr(dW2), ptr(db2), stream_ptr()), "time_embed_bwd")


def softmax_fwd(S: torch.Tensor, valid: Optional[int] = None) -> torch.Tensor:
    """Row softmax over the first `valid` of the last dim's columns (rest are padding -> 0)."""
    Lp = S.shape[-1]
    L = Lp if valid is None else valid
    P = torch.empty(tuple(S.shape), dtype=torch.bfloat16, device=S.device)
    check(load().fdx_softmax_fwd(ptr(S), S.numel() // Lp, L, Lp, ptr(P), stream_ptr()), "softmax_fwd")
    return P


def softmax_bwd(P: torch.Tensor, dP: torch.Tensor, scale: float, valid: Optional[int] = None) -> torch.Tensor:
    Lp = P.shape[-1]
    L = Lp if valid is None else valid
    dS = torch.empty(tuple(P.shape), dtype=torch.bfloat16, device=P.device)
    check(load().fdx_softmax_bwd(ptr(P), ptr(dP), P.numel() // Lp, L, Lp, scale, ptr(dS), stream_ptr()),
          "softmax_bwd")
    return dS


# --------------------------------------------------------------------------- UViT
def uvit_assemble_fwd(patch: torch.Tensor, pos: torch.Tensor, time_tok: torch.Tensor, text: Optional[torch.Tensor],
                      B: int, N: int, T: int) -> torch.Tensor:
    """The bf16 stream [B * (N + 1 + T), F]: per sample, bf16(patch + pos) rows, the time token, the text rows."""
    F = patch.shape[1]
    assert patch.dtype == torch.bfloat16 and patch.is_contiguous() and patch.shape[0] == B * N
    assert pos.dtype == torch.float32 and pos.is_contiguous() and pos.shape[-1] == F and pos.numel() >= N * F
    assert time_tok.dtype == torch.bfloat16 and time_tok.is_contiguous() and tuple(time_tok.shape) == (B, F)
    if T:
        assert text.dtype == torch.bfloat16 and text.is_contiguous() and tuple(text.shape) == (B * T, F)
    out = torch.empty((B * (N + 1 + T), F), dtype=torch.bfloat16, device=patch.device)
    check(load().fdx_uvit_assemble_fwd(ptr(patch), ptr(pos), ptr(time_tok), ptr(text if T else None), B, N, T, F,
                                       ptr(out), stream_ptr()), "uvit_assemble_fwd")
    return out


def uvit_pos_splits(B: int, N: int, F: int) -> int:
    """Sample splits of the position gradient's first stage: enough (N * F / 8)-thread slabs to fill the GPU, at most
    B.  A function of the shape only, so the summation order is too."""
    return max(1, min(B, (1 << 20) // max(1, N * F // 8)))


def uvit_assemble_bwd(dx: torch.Tensor, B: int, N: int, T: int, dpos: torch.Tensor, want_time: bool = True,
                      want_text: bool = True):
    """-> (dpatch bf16 [B * N, F], dtime f32 [B, F] or None, dtext bf16 [B * T, F] or None); dpos f32 [N, F]
    (a row-contiguous view) += the sum over samples of the patch rows' gradient."""
    F = dx.shape[1]
    assert dx.dtype == torch.bfloat16 and dx.is_contiguous() and dx.shape[0] == B * (N + 1 + T)
    assert dpos.dtype == torch.float32 and dpos.is_contiguous() and tuple(dpos.shape) == (N, F)
    dev = dx.device
    dpatch = torch.empty((B * N, F), dtype=torch.bfloat16, device=dev)
    dtime = torch.empty((B, F), dtype=torch.float32, device=dev) if want_time else None
    dtext = torch.empty((B * T, F), dtype=torch.bfloat16, device=dev) if (want_text and T) else None
    nsplit = uvit_pos_splits(B, N, F)
    ws = torch.empty((nsplit, N, F), dtype=torch.float32, device=dev)
    check(load().fdx_uvit_assemble_bwd(ptr(dx), B, N, T, F, ptr(dpatch), ptr(dtime), ptr(dtext), ptr(ws), nsplit,
                                       ptr(dpos), stream_ptr()), "uvit_assemble_bwd")
    return dpatch, dtime, dtext


def uvit_head_norm_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, act_code: int):
    """act(LayerNorm(x) gamma + beta) per pixel of x bf16 [..., 64] (act 1 = swish, 2 = mish) -> bf16, same shape."""
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.shape[-1] == 64
    y = torch.empty_like(x)
    check(load().fdx_uvit_head_norm_fwd(ptr(x), x.numel() // 64, ptr(gamma), ptr(beta), eps, act_code, ptr(y),
                                        stream_ptr()), "uvit_head_norm_fwd")
    return y


def uvit_head_norm_chunks(pixels: int) -> int:
    """Pixel chunks of the head LayerNorm backward's first stage: 256 pixels or more each, at most 528 (four per SM of
    a 132-SM H100).  A function of the size only, so the summation order is too."""
    return max(1, min(528, -(-pixels // 256)))


def uvit_head_norm_bwd(x: torch.Tensor, dy: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
                       act_code: int, dgamma: torch.Tensor, dbeta: torch.Tensor) -> torch.Tensor:
    """-> dx bf16; dgamma / dbeta f32 [64] += the sums over pixels (fixed order)."""
    assert x.dtype == dy.dtype == torch.bfloat16 and x.is_contiguous() and dy.is_contiguous() and x.shape == dy.shape
    pixels = x.numel() // 64
    nchunk = uvit_head_norm_chunks(pixels)
    ws = torch.empty((nchunk, 2, 64), dtype=torch.float32, device=x.device)
    dx = torch.empty_like(x)
    check(load().fdx_uvit_head_norm_bwd(ptr(x), ptr(dy), pixels, ptr(gamma), ptr(beta), eps, act_code, ptr(dx),
                                        ptr(ws), nchunk, ptr(dgamma), ptr(dbeta), stream_ptr()), "uvit_head_norm_bwd")
    return dx


def im2col3_c6(src0: torch.Tensor, src1: torch.Tensor) -> torch.Tensor:
    """final_conv1's bf16 operand [n*h*w, 64] over concat([src0, src1], -1) (two dense (n, h, w, 3) tensors, f32 or
    bf16): src0's 27 taps in columns 0..26, src1's in 32..58, zeros elsewhere."""
    n, h, w, c = src0.shape
    assert c == 3 and tuple(src1.shape) == (n, h, w, 3) and src0.is_contiguous() and src1.is_contiguous()
    assert src0.dtype in (torch.float32, torch.bfloat16) and src1.dtype in (torch.float32, torch.bfloat16)
    col = torch.empty((n * h * w, 64), dtype=torch.bfloat16, device=src0.device)
    check(load().fdx_im2col3x3_c6(ptr(src0), int(src0.dtype == torch.float32), ptr(src1),
                                  int(src1.dtype == torch.float32), n, h, w, ptr(col), stream_ptr()), "im2col3x3_c6")
    return col
