"""Float64 references for the mish activation (jax.nn.mish, the reference's `--activation mish`), kept beside the
swish ones they build on:

  * `mish` and `mish_oracle()`: the CPU oracle UNet of oracle/unet_ref.py with mish in place of swish.  The oracle
    applies its activation through the module global `swish` (after norm1 / norm2 of every ResidualBlock and after
    conv_out_norm, and nowhere else, as in the reference), so the context manager rebinds that name for its
    duration; oracle/train_ref.py reaches the same function through unet_ref.unet_forward.
  * element-wise references with derived per-element bounds for the GroupNorm + mish kernels, on top of
    tests/elementwise_ref.py (its tolerance model and GroupNorm closed forms).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as Fnn

from elementwise_ref import EX2, FTZ, U32, U_BF16, GnFwd, _g, conv3x3_dgrad_ref, gn_backward_ref
from oracle import unet_ref


def mish(x):
    """jax.nn.mish: x * tanh(softplus(x)), the third activation of the reference's ACTIVATION_MAP
    (flaxdiff/utils.py:33-38)."""
    return x * torch.tanh(Fnn.softplus(x))


@contextlib.contextmanager
def mish_oracle():
    """Within the block, oracle/unet_ref.py (and oracle/train_ref.py through it) computes a mish UNet."""
    saved = unet_ref.swish
    unet_ref.swish = mish
    try:
        yield
    finally:
        unet_ref.swish = saved


# ----------------------------------------------------------------------------------------------- GroupNorm + mish
# mish(z) = z tanh(softplus z), evaluated by the kernels (mish_f / mish_grad, fdx_common.cuh) from w = __expf(min(z, 20)):
# t = n / (n + 2) with n = w (w + 2), mish'(z) = r (n + 4 z w (w + 1) r) with r = 1 / (n + 2).  Error sources:
#   * __expf = ex2.approx(z log2 e): EX2 relative plus the rounding of the product, |z| u.  A relative error e in w
#     acts like moving z by e in the w-dependent terms, so it moves t by at most |sigma (1 - t^2)| e and mish' by at
#     most (|mish''| + |sigma (1 - t^2)|) e;
#   * ~12 f32 roundings, __fdividef (2 ulp) included, each relative on |t| + |z sigma (1 - t^2)|;
#   * the error of z itself (GnFwd.dz), through mish' (forward) and mish'' (backward);
#   * below z ~ -87 w flushes to zero (FTZ), where the exact values are below 2^-126 (|z| + 1).
# The clamp at z = 20 changes t by less than 2 e^-40 (far below u).
def _mish_parts(z):
    sp = Fnn.softplus(z, threshold=30.0)
    t = torch.tanh(sp)
    s = torch.sigmoid(z)
    q = s * (1 - t * t)                      # sigma(z) (1 - t^2) = d t / d z
    d1 = t + z * q                           # mish'
    # mish'' = 2 q + z q' with q' = sigma (1 - sigma) (1 - t^2) - 2 sigma t q  (t' = q, sigma' = sigma (1 - sigma))
    d2 = 2 * q + z * (s * (1 - s) * (1 - t * t) - 2 * s * t * q)
    return t, q, d1, d2


def mish_ref(z):
    """-> (mish(z), mish'(z)) in float64."""
    t, _, d1, _ = _mish_parts(z)
    return z * t, d1


def _mish_eval_err(z, t, q):
    """Bound on the kernels' own evaluation error of tanh(softplus z) given exact z (relative-to-w part and
    roundings), as an absolute error on t."""
    zc = z.clamp(max=20.0)
    e_w = EX2 + zc.abs() * U32
    return q.abs() * e_w + 12 * U32 * (t.abs() + (z * q).abs()) + 4 * FTZ


def gn_mish_forward_ref(x, gamma_, beta_, G, eps, depth=None):
    """fdx_groupnorm_apply(act = 2) -> (y, delta) as (N, H, W, C); `depth` as in GnFwd."""
    f = GnFwd(x, gamma_, beta_, G, eps, False, depth)
    z = f.z
    t, q, d1, _ = _mish_parts(z)
    y = z * t
    delta = d1.abs() * f.dz + z.abs() * _mish_eval_err(z, t, q) + 2 * U32 * y.abs() + 4 * FTZ * (z.abs() + 1)
    return y.reshape(f.shape), delta.reshape(f.shape)


def gn_mish_backward_ref(x, dy, gamma_, beta_, G, eps, dy_delta=None):
    """GroupNorm + mish backward: the activation-free backward (gn_backward_ref, silu=False) of dz = dy mish'(z),
    with the error of that dz as its input error.  mish'(z) is off by |mish''| dz_err (the error of z) plus its
    own evaluation error (the w terms move like z does, scaled by |mish''| + |sigma (1 - t^2)|), then 3 roundings."""
    f = GnFwd(x, gamma_, beta_, G, eps, False)
    z = f.z
    t, q, d1, d2 = _mish_parts(z)
    dyg = _g(dy, G)
    zc = z.clamp(max=20.0)
    e_grad = (d2.abs() * f.dz + (d2.abs() + q.abs()) * (EX2 + zc.abs() * U32) + 12 * U32 * (t.abs() + (z * q).abs())
              + 4 * FTZ * (z.abs() + 1))
    dz = dyg * d1
    e_dz = dyg.abs() * e_grad + 3 * U32 * dz.abs()
    if dy_delta is not None:
        e_dz = e_dz + d1.abs() * _g(dy_delta, G)
    shp = x.shape
    return gn_backward_ref(x, dz.reshape(shp), gamma_, beta_, G, eps, False, dy_delta=e_dz.reshape(shp))


def conv_gn_mish_backward_ref(x, dy, w_hwio, gamma_, beta_, G, eps):
    """d/dx of conv3x3(mish(groupnorm(x))) given dy: as conv_gn_backward_ref, |mish'| <= 1.0885 < 1.1."""
    da, e_da = conv3x3_dgrad_ref(dy, w_hwio)
    return gn_mish_backward_ref(x, da, gamma_, beta_, G, eps, dy_delta=e_da + U_BF16 * 1.1 * (da.abs() + e_da))
