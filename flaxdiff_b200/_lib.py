"""ctypes binding of libfdx.so (the sm_90a kernel library; C-ABI in include/fdx.h).

PyTorch is only the container: tensors provide device memory (`data_ptr`) and the
current CUDA stream.  There is no CPU or eager fallback: if the shared library is
missing the import of any op raises, and every op requires CUDA tensors.

load() gives every entry point the restype and argtypes of SIGNATURES, so callers pass Python ints, floats, None
and descriptor structs as they are, and ctypes converts each argument to its C type (a wrong descriptor is a
TypeError, a long long is never cut to an int).
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


def _signatures() -> dict:
    """name -> (restype, argtypes) of every entry point of include/fdx.h, in the header's order.  C types map as
    int -> c_int, long long -> c_longlong, float -> c_float, uint32_t -> c_uint32, const <descriptor>* ->
    POINTER(<descriptor>), any other pointer -> c_void_p; returns int -> c_int, unsigned long long -> c_ulonglong,
    const char* -> c_char_p.  tests/test_capi_cpu.py checks the table against the header."""
    vp, i, ll, f, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_uint32
    s, u64 = ctypes.c_char_p, ctypes.c_ulonglong
    pact, pcs, pgemm, popt, pattn = (ctypes.POINTER(t) for t in
                                     (fdx_act, fdx_colstats, fdx_gemm_desc, fdx_opt_desc, fdx_attn_desc))
    return {
        # ---- library
        "fdx_last_error": (s, []),
        "fdx_version": (i, []),
        "fdx_device_sm_count": (i, []),
        "fdx_launch_count": (u64, []),
        "fdx_last_kernel_kind": (i, []),
        "fdx_kernel_kind_name": (s, [i]),
        # ---- tensor-core contractions
        "fdx_conv3x3_fwd": (i, [pact, vp, vp, vp, pact, pact, i, vp]),
        "fdx_conv3x3_fwd_stats": (i, [pact, vp, vp, vp, pact, pact, i, pcs, vp]),
        "fdx_groupnorm_stats_from_cols": (i, [vp, i, i, i, i, i, i, vp, vp]),
        "fdx_conv3x3_dgrad": (i, [pact, vp, pact, i, i, vp]),
        "fdx_conv3x3_wgrad": (i, [pact, pact, vp, i, vp]),
        "fdx_conv1x1_fwd": (i, [pact, vp, vp, pact, pact, vp]),
        "fdx_conv1x1_dgrad": (i, [pact, vp, pact, i, vp]),
        "fdx_gemm": (i, [pgemm, vp]),
        "fdx_gemm_cat": (i, [pgemm, vp, ll, i, vp]),
        "fdx_upconv3x3_pack": (i, [vp, i, i, vp, vp]),
        "fdx_upconv3x3_fwd": (i, [pact, vp, vp, pact, vp]),
        "fdx_upconv3x3_fwd_stats": (i, [pact, vp, vp, pact, pcs, vp]),
        "fdx_upconv3x3_dgrad": (i, [pact, vp, pact, i, vp]),
        "fdx_upconv3x3_wgrad": (i, [pact, pact, vp, vp, vp]),
        # ---- normalisation
        "fdx_groupnorm_stats": (i, [pact, i, vp, vp]),
        "fdx_groupnorm_apply": (i, [pact, i, vp, vp, vp, f, i, pact, vp]),
        "fdx_groupnorm_apply_cols": (i, [pact, i, vp, i, i, i, vp, vp, f, i, pact, vp, vp]),
        "fdx_groupnorm_bwd": (i, [pact, pact, i, vp, vp, vp, f, i, vp, vp, vp, pact, i, vp, vp, vp]),
        "fdx_groupnorm_bwd_add": (i, [pact, pact, i, vp, vp, vp, f, i, vp, vp, vp, pact, pact, vp, vp, vp]),
        "fdx_groupnorm_coeffs": (i, [vp, vp, vp, i, i, i, i, f, vp, vp]),
        "fdx_conv3x3_dgrad_gn": (i, [pact, vp, pact, pact, vp, vp, i, vp]),
        "fdx_conv3x3_dgrad_gn_act": (i, [pact, vp, pact, pact, vp, vp, i, i, vp]),
        "fdx_groupnorm_bwd_dz": (i, [pact, pact, i, vp, vp, f, vp, i, vp, vp, vp, pact, i, vp, vp, vp]),
        "fdx_groupnorm_bwd_dz_add": (i, [pact, pact, i, vp, vp, f, vp, i, vp, vp, vp, pact, pact, vp, vp, vp]),
        "fdx_rmsnorm_fwd": (i, [pact, vp, f, pact, vp]),
        "fdx_rmsnorm_bwd": (i, [pact, pact, vp, f, pact, i, vp, vp]),
        # ---- diffusion step streaming kernels
        "fdx_diffuse_forward": (i, [vp, i, vp, vp, vp, vp, i, ll, i, i, vp, vp, vp, vp]),
        "fdx_loss_fwd_bwd": (i, [vp, vp, vp, vp, vp, vp, i, ll, vp, vp, vp]),
        "fdx_affine_combine": (i, [i, vp, vp, vp, vp, i, ll, vp, vp, vp, i, f, f, vp]),
        # ---- jax.random's threefry streams
        "fdx_random_bits": (i, [u32, u32, vp, ll, vp, vp]),
        "fdx_random_uniform": (i, [u32, u32, vp, ll, f, f, vp, vp]),
        "fdx_random_normal": (i, [u32, u32, vp, ll, vp, vp]),
        "fdx_random_randint": (i, [u32, u32, vp, ll, i, i, vp, vp]),
        # ---- optimiser / EMA / loss scaling
        "fdx_optimizer_step": (i, [popt, vp]),
        "fdx_adamw_ema_step": (i, [vp, vp, vp, vp, vp, vp, ll, f, f, f, f, f, i, f, f, vp, f, vp, vp]),
        "fdx_ema_update": (i, [vp, vp, ll, f, vp]),
        "fdx_grad_stats": (i, [vp, ll, vp, vp, vp]),
        "fdx_sumsq": (i, [vp, ll, vp, vp]),
        "fdx_dynscale_update": (i, [vp, vp, f, f, i, f, vp]),
        # ---- data-parallel exchange, casts, nearest upsampling, column sums
        "fdx_comm_unique_id": (i, [vp]),
        "fdx_comm_init": (i, [vp, i, i, vp]),
        "fdx_comm_allreduce_avg": (i, [vp, vp, ll, vp]),
        "fdx_comm_world": (i, [vp, vp, vp]),
        "fdx_comm_nccl_version": (i, []),
        "fdx_comm_destroy": (i, [vp]),
        "fdx_cast_f32_bf16": (i, [vp, vp, ll, vp]),
        "fdx_upsample2x": (i, [pact, pact, vp]),
        "fdx_upsample2x_bwd": (i, [pact, pact, i, vp]),
        "fdx_act_add": (i, [pact, pact, pact, vp]),
        "fdx_colsum": (i, [pact, vp, i, vp]),
        # ---- 3-channel convolutions
        "fdx_conv_in_fwd": (i, [vp, i, i, i, vp, vp, pact, vp]),
        "fdx_conv_in_wgrad": (i, [vp, pact, vp, vp, vp]),
        "fdx_im2col3x3_c3": (i, [vp, i, i, i, i, i, i, vp, vp]),
        "fdx_col2im3x3_c3": (i, [vp, vp, i, i, i, vp, vp]),
        "fdx_conv_out_fwd": (i, [pact, vp, vp, vp, vp]),
        "fdx_conv_out_dgrad": (i, [vp, vp, pact, vp]),
        "fdx_conv_out_wgrad": (i, [pact, vp, vp, vp, vp]),
        # ---- timestep embedding, softmax, GEGLU
        "fdx_time_embed_fwd": (i, [vp, vp, vp, vp, vp, vp, i, i, vp, vp, vp, vp, vp, vp]),
        "fdx_time_embed_bwd": (i, [vp, vp, vp, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp]),
        "fdx_softmax_fwd": (i, [vp, ll, i, i, vp, vp]),
        "fdx_softmax_bwd": (i, [vp, vp, ll, i, i, f, vp, vp]),
        "fdx_geglu_fwd": (i, [vp, ll, i, vp, vp]),
        "fdx_geglu_bwd": (i, [vp, vp, ll, i, vp, vp]),
        # ---- fused attention
        "fdx_attention_fwd": (i, [pattn, vp]),
        "fdx_attention_bwd": (i, [pattn, vp]),
        "fdx_attention_fwd_masked": (i, [pattn, i, vp, vp]),
        # ---- CLIP text tower
        "fdx_token_embed": (i, [vp, i, i, vp, i, vp, i, vp, vp]),
        "fdx_layernorm_fwd": (i, [vp, ll, i, vp, vp, f, vp, vp]),
        "fdx_bias_act": (i, [vp, ll, i, vp, i, vp, vp]),
        # ---- CLIP validation metrics
        "fdx_clip_image_prep": (i, [vp, i, i, i, vp, i, i, vp, i, i, i, vp, vp, vp]),
        "fdx_clip_vision_embed": (i, [vp, i, i, i, vp, vp, vp, vp, f, vp, vp]),
        "fdx_clip_pool": (i, [vp, i, i, i, vp, vp, vp, f, vp, vp]),
        "fdx_clip_similarity": (i, [vp, vp, i, i, vp, vp, vp]),
        # ---- SimpleDiT
        "fdx_dit_adaln_fwd": (i, [vp, ll, i, i, vp, ll, i, i, vp, vp, f, vp, vp, vp, vp]),
        "fdx_dit_adaln_bwd": (i, [vp, vp, ll, i, i, vp, ll, i, vp, vp, vp, vp, vp, vp, i, vp, ll, vp, ll, i, i, vp]),
        "fdx_dit_gate_fwd": (i, [vp, vp, ll, i, i, vp, ll, vp, vp]),
        "fdx_dit_gate_bwd": (i, [vp, vp, ll, i, i, vp, ll, vp, vp, i, vp, ll, vp]),
        "fdx_dit_token_mean": (i, [vp, i, i, i, vp, i, vp, vp]),
        "fdx_dit_rope": (i, [vp, ll, i, ll, i, i, i, i, ll, i, vp]),
        "fdx_bias_act_bwd": (i, [vp, ll, i, vp, i, vp, vp, vp]),
        "fdx_dit_patchify": (i, [vp, i, i, i, i, i, i, i, vp, vp]),
        "fdx_dit_unpatchify": (i, [vp, i, i, i, i, i, i, vp, vp]),
        "fdx_dit_fourier": (i, [vp, i, vp, i, vp, vp]),
        # ---- S5 state-space layer
        "fdx_ssm_discretize": (i, [vp, vp, vp, vp, vp, vp, vp, i, i, vp, i, i, vp, vp, vp]),
        "fdx_ssm_discretize_bwd": (i, [vp, vp, vp, vp, vp, i, i, vp, i, vp, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp,
                                       vp]),
        "fdx_ssm_scan": (i, [vp, vp, vp, vp, i, i, i, i, i, vp, vp]),
        "fdx_ssm_scan_bwd": (i, [vp, vp, vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp]),
        "fdx_permute_rows": (i, [vp, vp, ll, i, ll, vp, vp]),
        # ---- SimpleMMDiT
        "fdx_mmdit_adaln_fwd": (i, [vp, ll, i, i, vp, ll, f, vp, vp, vp, vp, vp]),
        "fdx_mmdit_adaln_bwd": (i, [vp, vp, vp, ll, i, i, vp, ll, vp, vp, vp, vp, vp, i, vp, ll, vp]),
        "fdx_mmdit_gate_fwd": (i, [vp, vp, vp, ll, i, i, vp, ll, vp, vp]),
        "fdx_mmdit_gate_bwd": (i, [vp, vp, vp, ll, i, i, vp, ll, vp, vp, vp, i, vp, ll, vp]),
        # ---- HierarchicalMMDiT
        "fdx_layernorm_rows_fwd": (i, [i, vp, vp, ll, i, i, i, i, vp, vp, f, vp, vp, vp, vp]),
        "fdx_layernorm_rows_bwd": (i, [i, vp, vp, vp, ll, i, i, i, i, vp, vp, vp, vp, i, vp, i, vp, i, vp, vp, vp]),
        # ---- UViT
        "fdx_uvit_assemble_fwd": (i, [vp, vp, vp, vp, i, i, i, i, vp, vp]),
        "fdx_uvit_assemble_bwd": (i, [vp, i, i, i, i, vp, vp, vp, vp, i, vp, vp]),
        "fdx_uvit_head_norm_fwd": (i, [vp, ll, vp, vp, f, i, vp, vp]),
        "fdx_uvit_head_norm_bwd": (i, [vp, vp, ll, vp, vp, f, i, vp, vp, i, vp, vp, vp]),
        "fdx_im2col3x3_c6": (i, [vp, i, vp, i, i, i, i, vp, vp]),
    }


SIGNATURES = _signatures()

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
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
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
