"""ctypes binding of libfdx.so (the sm_90a kernel library; C-ABI in include/fdx.h).

PyTorch is only the container: tensors provide device memory (`data_ptr`) and the
current CUDA stream.  There is no CPU or eager fallback: if the shared library is
missing the import of any op raises, and every op requires CUDA tensors.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libfdx.so")


class FdxError(RuntimeError):
    pass


class fdx_act(ctypes.Structure):
    _fields_ = [
        ("ptr", ctypes.c_void_p),
        ("n", ctypes.c_int),
        ("h", ctypes.c_int),
        ("w", ctypes.c_int),
        ("c", ctypes.c_int),
        ("pix_stride", ctypes.c_longlong),
    ]


class fdx_colstats(ctypes.Structure):
    _fields_ = [("ws", ctypes.c_void_p), ("slots", ctypes.c_int), ("ld", ctypes.c_int)]


class fdx_gemm_desc(ctypes.Structure):
    _fields_ = [
        ("mode", ctypes.c_int),
        ("M", ctypes.c_int), ("N", ctypes.c_int), ("K", ctypes.c_int),
        ("batch1", ctypes.c_int), ("batch2", ctypes.c_int),
        ("A", ctypes.c_void_p), ("a_ld", ctypes.c_longlong), ("a_s1", ctypes.c_longlong), ("a_s2", ctypes.c_longlong),
        ("B", ctypes.c_void_p), ("b_ld", ctypes.c_longlong), ("b_s1", ctypes.c_longlong), ("b_s2", ctypes.c_longlong),
        ("D", ctypes.c_void_p), ("d_ld", ctypes.c_longlong), ("d_s1", ctypes.c_longlong), ("d_s2", ctypes.c_longlong),
        ("d_f32", ctypes.c_int), ("d_atomic", ctypes.c_int), ("reduce_batch", ctypes.c_int),
        ("alpha", ctypes.c_float),
        ("bias", ctypes.c_void_p),
        ("res", ctypes.c_void_p), ("r_ld", ctypes.c_longlong), ("r_s1", ctypes.c_longlong), ("r_s2", ctypes.c_longlong),
    ]


class fdx_opt_desc(ctypes.Structure):
    _fields_ = [
        ("kind", ctypes.c_int),
        ("p", ctypes.c_void_p), ("g", ctypes.c_void_p), ("m", ctypes.c_void_p), ("v", ctypes.c_void_p),
        ("ema", ctypes.c_void_p), ("shadow_bf16", ctypes.c_void_p), ("n", ctypes.c_longlong),
        ("lr", ctypes.c_float), ("b1", ctypes.c_float), ("b2", ctypes.c_float), ("eps", ctypes.c_float),
        ("weight_decay", ctypes.c_float), ("step", ctypes.c_int), ("ema_decay", ctypes.c_float),
        ("grad_scale", ctypes.c_float), ("gstats", ctypes.c_void_p), ("clip_norm", ctypes.c_float),
        ("dyn_lr_bc", ctypes.c_void_p), ("dynscale", ctypes.c_void_p),
        ("seg_offsets", ctypes.c_void_p), ("nseg", ctypes.c_int), ("seg_norms", ctypes.c_void_p),
        ("u_ws", ctypes.c_void_p),
    ]


class fdx_attn_desc(ctypes.Structure):
    _fields_ = [
        ("B", ctypes.c_int), ("heads", ctypes.c_int), ("L", ctypes.c_int), ("Lk", ctypes.c_int), ("dh", ctypes.c_int),
        ("scale", ctypes.c_float),
        ("q", ctypes.c_void_p), ("q_ld", ctypes.c_longlong), ("q_bs", ctypes.c_longlong),
        ("k", ctypes.c_void_p), ("k_ld", ctypes.c_longlong), ("k_bs", ctypes.c_longlong),
        ("v", ctypes.c_void_p), ("v_ld", ctypes.c_longlong), ("v_bs", ctypes.c_longlong),
        ("o", ctypes.c_void_p), ("o_ld", ctypes.c_longlong), ("o_bs", ctypes.c_longlong),
        ("lse", ctypes.c_void_p),
        ("d_o", ctypes.c_void_p), ("do_ld", ctypes.c_longlong), ("do_bs", ctypes.c_longlong),
        ("dvec_ws", ctypes.c_void_p),
        ("dq", ctypes.c_void_p), ("dq_ld", ctypes.c_longlong), ("dq_bs", ctypes.c_longlong),
        ("dk", ctypes.c_void_p), ("dk_ld", ctypes.c_longlong), ("dk_bs", ctypes.c_longlong),
        ("dv", ctypes.c_void_p), ("dv_ld", ctypes.c_longlong), ("dv_bs", ctypes.c_longlong),
    ]


GEMM_KK, GEMM_KMN, GEMM_MNMN = 0, 1, 2
OPT_ADAM, OPT_LAMB = 0, 1
ACT_QUICK_GELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2          # fdx_bias_act


def _declare(lib) -> None:
    """Argument types of the entry points whose integer arguments are wider than C int or are pointers passed
    as Python ints (ctypes would otherwise truncate them)."""
    vp, i, ll, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
    lib.fdx_attention_fwd_masked.argtypes = [ctypes.POINTER(fdx_attn_desc), i, vp, vp]
    lib.fdx_token_embed.argtypes = [vp, i, i, vp, i, vp, i, vp, vp]
    lib.fdx_layernorm_fwd.argtypes = [vp, ll, i, vp, vp, f, vp, vp]
    lib.fdx_bias_act.argtypes = [vp, ll, i, vp, i, vp, vp]
    lib.fdx_clip_image_prep.argtypes = [vp, i, i, i, vp, i, i, vp, i, i, i, vp, vp, vp]
    lib.fdx_clip_vision_embed.argtypes = [vp, i, i, i, vp, vp, vp, vp, f, vp, vp]
    lib.fdx_clip_pool.argtypes = [vp, i, i, i, vp, vp, vp, f, vp, vp]
    lib.fdx_clip_similarity.argtypes = [vp, vp, i, i, vp, vp, vp]
    lib.fdx_dit_adaln_fwd.argtypes = [vp, ll, i, i, vp, ll, i, i, vp, vp, f, vp, vp, vp, vp]
    lib.fdx_dit_adaln_bwd.argtypes = [vp, vp, ll, i, i, vp, ll, i, vp, vp, vp, vp, vp, vp, i, vp, ll, vp, ll, i, i, vp]
    lib.fdx_dit_gate_fwd.argtypes = [vp, vp, ll, i, i, vp, ll, vp, vp]
    lib.fdx_dit_gate_bwd.argtypes = [vp, vp, ll, i, i, vp, ll, vp, vp, i, vp, ll, vp]
    lib.fdx_dit_token_mean.argtypes = [vp, i, i, i, vp, i, vp, vp]
    lib.fdx_dit_rope.argtypes = [vp, ll, i, ll, i, i, i, i, ll, i, vp]
    lib.fdx_bias_act_bwd.argtypes = [vp, ll, i, vp, i, vp, vp, vp]
    lib.fdx_dit_patchify.argtypes = [vp, i, i, i, i, i, i, i, vp, vp]
    lib.fdx_dit_unpatchify.argtypes = [vp, i, i, i, i, i, i, vp, vp]
    lib.fdx_dit_fourier.argtypes = [vp, i, vp, i, vp, vp]
    lib.fdx_ssm_discretize.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, vp, i, i, vp, vp, vp]
    lib.fdx_ssm_discretize_bwd.argtypes = [vp, vp, vp, vp, vp, i, i, vp, i, vp, vp, vp, i, i, vp, vp, vp, vp, vp, vp,
                                           vp, vp]
    lib.fdx_ssm_scan.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, vp]
    lib.fdx_ssm_scan_bwd.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp]
    lib.fdx_permute_rows.argtypes = [vp, vp, ll, i, ll, vp, vp]


_lib: Optional[ctypes.CDLL] = None


def lib_path() -> str:
    return _LIB_PATH


def load() -> ctypes.CDLL:
    """Load libfdx.so; raises FdxError (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise FdxError(
            f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C flaxdiff_b200/csrc`. flaxdiff_b200 has no CPU fallback.")
    lib = ctypes.CDLL(_LIB_PATH)
    lib.fdx_last_error.restype = ctypes.c_char_p
    _declare(lib)
    if os.environ.get("FDX_TRACE"):
        lib = _TracingLib(lib)
    _lib = lib
    return lib


class _TracingLib:
    """Debug aid (FDX_TRACE=1): log every C-ABI call to stderr and synchronise after it, so a hung
    or faulting kernel is attributed to the entry point that launched it."""

    def __init__(self, lib):
        self._lib = lib
        self._n = 0

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("fdx_") or name in ("fdx_last_error", "fdx_launch_count", "fdx_version"):
            return fn

        def traced(*args):
            import sys
            import time
            self._n += 1
            t0 = time.time()
            sys.stderr.write(f"[fdx-trace {self._n}] {name} ...")
            sys.stderr.flush()
            r = fn(*args)
            if not torch.cuda.is_current_stream_capturing():
                torch.cuda.synchronize()
            sys.stderr.write(f" rc={r} {1e3 * (time.time() - t0):.2f} ms\n")
            sys.stderr.flush()
            return r
        return traced


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = load().fdx_last_error().decode("utf-8", "replace")
        raise FdxError(f"libfdx {what} failed with status {status}: {msg}")


def stream_ptr() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _require_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise FdxError(f"{name}: expected a CUDA tensor (flaxdiff_b200 has no CPU path)")


def act(t: torch.Tensor, name: str = "act") -> fdx_act:
    """Describe an NHWC bf16 tensor (possibly a channel-slice view of a wider buffer)."""
    _require_cuda(t, name)
    if t.dim() != 4:
        raise FdxError(f"{name}: expected NHWC rank-4 tensor, got {tuple(t.shape)}")
    n, h, w, c = t.shape
    sn, sh, sw, sc = t.stride()
    if sc != 1 or sh != sw * w or sn != sh * h:
        raise FdxError(f"{name}: tensor must be pixel-contiguous NHWC (strides {t.stride()})")
    return fdx_act(ctypes.c_void_p(t.data_ptr()), n, h, w, c, sw)


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    if t is None:
        return ctypes.c_void_p(0)
    _require_cuda(t, "tensor")
    return ctypes.c_void_p(t.data_ptr())
