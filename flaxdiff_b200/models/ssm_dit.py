"""`HybridSSMAttentionDiT` - the reference's hybrid SSM-attention denoiser (flaxdiff/models/ssm_dit.py:545-779) on the
engine, with the same program interface as `SimpleDiT` and `Unet` (init / apply / forward / backward / layout), so
GeneralDiffusionTrainer, the samplers and the checkpoint writer take it unchanged.

    model = HybridSSMAttentionDiT(patch_size=2, emb_features=768, num_layers=12, num_heads=12,
                                  ssm_attention_ratio="3:1", use_hilbert=True)
    params = model.init(key)                              # {'params': tree}, flax names
    y = model.apply(params, x, temb, textcontext)         # (B, H, W, 3) f32

The attention blocks are SimpleDiT's DiTBlock program (shared code); the SSM blocks (SSMDiTBlock, ssm_dit.py:504-538)
keep its adaLN / gated-residual / MLP skeleton around an S5 layer: the discretisation and the sequence-parallel scans
are fdx_ssm.cu's, the dense products (Bu = u Bbar^T, y = Re(C x), out_proj and their gradients) run on fdx_gemm, and
D * u is the gated-residual kernel with the gate D broadcast over the samples.  Under the Hilbert / zigzag patch orders
the patch rows are permuted on the device (fdx_permute_rows), `hilbert_projection` replaces `patch_embed`, the sin-cos
table follows the order and RoPE is off.  use_2d_fusion is refused.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

from .. import ops
from .._lib import GEMM_KK, FdxError
from .simple_dit import BF16, F32, SimpleDiT, _lecun_normal
from .simple_unet import _dense_dgrad, _dense_wgrad

S5_LEAVES = ("log_A_real", "A_imag", "B_re", "B_im", "C_re", "C_im", "D", "log_dt")


# ---------------------------------------------------------------------------------------------- patch orders
def hilbert_d2xy(n: int, d: int):
    """Position d along the Hilbert curve of an n x n grid (n a power of two) -> (x = column, y = row)."""
    x = y = 0
    s = 1
    while s < n:
        rx = (d >> 1) & 1
        ry = (d ^ rx) & 1
        if ry == 0:
            if rx == 1:
                x, y = s - 1 - x, s - 1 - y
            x, y = y, x
        x += s * rx
        y += s * ry
        d >>= 2
        s <<= 1
    return x, y


def hilbert_indices(HP: int, WP: int) -> np.ndarray:
    """Row-major patch index of each position along the Hilbert curve of the next power-of-two square, keeping only
    the cells inside the HP x WP grid (hilbert.py:87-130)."""
    n = 1 << max(0, math.ceil(math.log2(max(HP, WP, 1))))
    out = []
    for d in range(n * n):
        x, y = hilbert_d2xy(n, d)
        if x < WP and y < HP:
            out.append(y * WP + x)
            if len(out) == HP * WP:
                break
    return np.asarray(out, dtype=np.int64)


def zigzag_indices(HP: int, WP: int) -> np.ndarray:
    """Serpentine order: even rows left to right, odd rows right to left (hilbert.py:248-269)."""
    rows = [np.arange(r * WP, (r + 1) * WP) for r in range(HP)]
    return np.concatenate([r if i % 2 == 0 else r[::-1] for i, r in enumerate(rows)]).astype(np.int64)


def build_block_pattern(num_layers: int, block_pattern: Optional[Sequence[str]], ratio: str) -> List[str]:
    """_build_block_pattern (ssm_dit.py:588-601): block_pattern wins; "all-ssm" / "all-attn"; "a:b" repeats
    a 'ssm' and b 'attn' entries, truncated to num_layers.  Any entry but 'ssm' is an attention block."""
    if block_pattern is not None:
        return list(block_pattern)
    if ratio == "all-ssm":
        return ["ssm"] * num_layers
    if ratio == "all-attn":
        return ["attn"] * num_layers
    parts = str(ratio).split(":")
    try:
        a, b = (int(v) for v in parts)
    except ValueError:
        a = b = -1
    if len(parts) != 2 or a < 0 or b < 0 or a + b == 0:
        raise FdxError(f"HybridSSMAttentionDiT: ssm_attention_ratio={ratio!r} is not 'all-ssm', 'all-attn' or "
                       "'a:b' with non-negative integers, not both zero")
    unit = ["ssm"] * a + ["attn"] * b
    return (unit * (num_layers // len(unit) + 1))[:num_layers]


class HybridSSMAttentionDiT(SimpleDiT):
    def __init__(self, output_channels: int = 3, patch_size: int = 16, emb_features: int = 768, num_layers: int = 12,
                 num_heads: int = 12, mlp_ratio: int = 4, ssm_state_dim: int = 64, dropout_rate: float = 0.0,
                 dtype=None, precision=None, use_flash_attention: bool = False, force_fp32_for_softmax: bool = True,
                 norm_epsilon: float = 1e-5, learn_sigma: bool = False, use_hilbert: bool = False,
                 use_zigzag: bool = False, norm_groups: int = 0, activation=None,
                 block_pattern: Optional[Sequence[str]] = None, ssm_attention_ratio: str = "3:1",
                 bidirectional_ssm: bool = True, use_2d_fusion: bool = False, context_dim: Optional[int] = None,
                 use_remat: bool = False):
        if use_hilbert and use_zigzag:
            raise FdxError("HybridSSMAttentionDiT: use_hilbert and use_zigzag are mutually exclusive")
        if use_2d_fusion:
            raise FdxError("HybridSSMAttentionDiT: use_2d_fusion=True (SpatialFusionConv) is not supported")
        N = ssm_state_dim
        if not isinstance(N, int) or N <= 0 or N % 16:
            raise FdxError(f"HybridSSMAttentionDiT: ssm_state_dim={N} must be a positive multiple of 16 (the state "
                           "products run on the GEMM engine with K = 2 * ssm_state_dim, a multiple of 32)")
        super().__init__(output_channels=output_channels, patch_size=patch_size, emb_features=emb_features,
                         num_layers=num_layers, num_heads=num_heads, mlp_ratio=mlp_ratio, dropout_rate=dropout_rate,
                         dtype=dtype, precision=precision, use_flash_attention=use_flash_attention,
                         force_fp32_for_softmax=force_fp32_for_softmax, norm_epsilon=norm_epsilon,
                         learn_sigma=learn_sigma, norm_groups=norm_groups, activation=activation,
                         context_dim=context_dim, use_remat=use_remat)
        self.use_hilbert = use_hilbert
        self.use_zigzag = use_zigzag
        self.ssm_state_dim = N
        self.block_pattern = None if block_pattern is None else list(block_pattern)
        self.ssm_attention_ratio = ssm_attention_ratio
        self.bidirectional_ssm = bidirectional_ssm
        self.use_2d_fusion = use_2d_fusion
        self.pattern = build_block_pattern(num_layers, self.block_pattern, ssm_attention_ratio)

    # ------------------------------------------------------------------ structure
    def config(self) -> dict:
        """The constructor arguments (a config round trip: HybridSSMAttentionDiT(**model.config()))."""
        cfg = super().config()
        cfg.update({k: getattr(self, k) for k in ("ssm_state_dim", "block_pattern", "ssm_attention_ratio",
                                                   "bidirectional_ssm", "use_2d_fusion")})
        return cfg

    def _scan_order(self) -> bool:
        return self.use_hilbert or self.use_zigzag

    def _embed_name(self) -> str:
        return "hilbert_projection" if self._scan_order() else super()._embed_name()

    def _embed_specs(self):
        if not self._scan_order():
            return super()._embed_specs()
        p, F = self.patch_size, self.emb_features
        return [("hilbert_projection/kernel", (p * p * 3, F)), ("hilbert_projection/bias", (F,))]

    def _scan_indices(self, HP: int, WP: int):
        if self.use_hilbert:
            return hilbert_indices(HP, WP)
        if self.use_zigzag:
            return zigzag_indices(HP, WP)
        return None

    def _blocks(self):
        return [(f"ssm_block_{i}", self._ssm_block_fwd, self._ssm_block_bwd) if kind == "ssm" else
                (f"dit_block_{i}", self._block_fwd, self._block_bwd) for i, kind in enumerate(self.pattern)]

    def _s5_names(self, n: str) -> List[str]:
        """The S5 layers of SSM block n: s5_forward / s5_backward under a BidirectionalS5Layer, else the S5Layer."""
        return [f"{n}/ssm/s5_forward", f"{n}/ssm/s5_backward"] if self.bidirectional_ssm else [f"{n}/ssm"]

    def _block_specs(self, n):
        if not n.startswith("ssm_block_"):
            return super()._block_specs(n)
        F, N, E = self.emb_features, self.ssm_state_dim, self.emb_features * self.mlp_ratio
        shapes = {"log_A_real": (N,), "A_imag": (N,), "B_re": (N, F), "B_im": (N, F), "C_re": (F, N),
                  "C_im": (F, N), "D": (F,), "log_dt": (N,)}
        specs = [(f"{n}/ada_params_module/ada_proj/kernel", (F, 6 * F)),
                 (f"{n}/ada_params_module/ada_proj/bias", (6 * F,))]
        for s5 in self._s5_names(n):
            specs += [(f"{s5}/{leaf}", shapes[leaf]) for leaf in S5_LEAVES]
        if self.bidirectional_ssm:
            specs += [(f"{n}/ssm/out_proj/kernel", (2 * F, F)), (f"{n}/ssm/out_proj/bias", (F,))]
        specs += [(f"{n}/mlp/layers_0/kernel", (F, E)), (f"{n}/mlp/layers_0/bias", (E,)),
                  (f"{n}/mlp/layers_2/kernel", (E, F)), (f"{n}/mlp/layers_2/bias", (F,))]
        return specs

    def _init_leaf(self, name: str, t: torch.Tensor, gen: torch.Generator) -> None:
        """S5 leaves as S5Layer initialises them (ssm_dit.py:37-153): HiPPO log_A_real = log(n + 1/2) and
        A_imag = pi n, log_dt ~ U[log 0.001, log 0.1], D ~ N(0, 1), B / C lecun-normal with flax's fan-in (the
        second-to-last axis); out_proj is a Dense kernel.  Everything else as SimpleDiT."""
        leaf = name.rsplit("/", 1)[1]
        if "/ssm/" not in name or leaf in ("kernel", "bias"):
            return super()._init_leaf(name, t, gen)
        if leaf == "log_A_real":
            t.copy_(torch.log(torch.arange(t.numel(), dtype=F32) + 0.5))
        elif leaf == "A_imag":
            t.copy_(math.pi * torch.arange(t.numel(), dtype=F32))
        elif leaf == "log_dt":
            t.uniform_(math.log(0.001), math.log(0.1), generator=gen)
        elif leaf == "D":
            t.normal_(0.0, 1.0, generator=gen)
        else:
            _lecun_normal(t, t.shape[-2], gen)

    # ------------------------------------------------------------------ SSM block
    def _s5_leaves(self, named, base):
        return {leaf: named[f"{base}/{leaf}"] for leaf in S5_LEAVES}

    def _ssm_block_fwd(self, n, x, cond16, W32, W16, B, L, save: bool = True):
        """SSMDiTBlock: x1 = x + gate_attn * S5(adaLN(x)); x2 = x1 + gate_mlp * MLP(adaLN(x1)).  ada chunks as the
        DiTBlock's.  -> (x2, record; None unless save).  Without save the scan stores no f32 states, Bu is released
        after the scan, the bf16 states after the C products and the per-direction rows after out_proj."""
        F, N, eps = self.emb_features, self.ssm_state_dim, self.norm_epsilon
        dev = x.device
        s5 = self._s5_names(n)
        nd = len(s5)
        S2 = 2 * nd * N
        ada = self._ada_fwd(n, cond16, W32, W16)
        u, m1, r1 = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps)
        wb = torch.empty((F, S2), dtype=BF16, device=dev)
        adt = torch.empty(S2, dtype=F32, device=dev)
        wcs = []
        for d, base in enumerate(s5):
            wc = torch.empty((2 * N, F), dtype=BF16, device=dev)
            ops.ssm_discretize(self._s5_leaves(W32, base), N, F, wb, 2 * d * N, wc, adt)
            wcs.append(wc)
        bu = ops.linear_fwd(u, wb, out_dtype=F32)                   # Bu of every direction
        chunk = ops.ssm_chunk(B, L, nd * N, dev)
        xs, x16 = ops.ssm_scan(bu, adt, B, N, nd, chunk, states=save)
        if not save:
            del bu
        ys = []
        for d, base in enumerate(s5):
            yd = ops.linear_fwd(x16[:, 2 * d * N:2 * (d + 1) * N], wcs[d])
            ops.dit_gate_fwd(yd, u, L, W32[f"{base}/D"].expand(B, F), out=yd)    # + D * u
            ys.append(yd)
        del u
        if not save:
            del x16, yd
        if nd == 2:
            # out_proj over [y_fwd, y_bwd]: the two K halves as two products, the second adding onto the first
            wo = W16[f"{n}/ssm/out_proj/kernel"]
            y = ops.linear_fwd(ys[0], wo[:F], bias=W32[f"{n}/ssm/out_proj/bias"])
            ops.linear_fwd(ys[1], wo[F:], out=y, res=y)
        else:
            y = ys[0]
        if not save:
            del ys
        x1 = ops.dit_gate_fwd(x, y, L, ada[:, 5 * F:])
        if not save:
            del y
        x2, mlp = self._mlp_fwd(n, x1, ada, W32, W16, L, save)
        if not save:
            return x2, None
        return x2, (n, x, ada, m1, r1, bu, xs, x16, ys, y, x1, mlp, (wb, wcs, adt, chunk))

    def _ssm_block_bwd(self, rec, dx2, cond16, dcond, W32, W16, Gd, B, L):
        n, x, ada, m1, r1, bu, xs, x16, ys, y, x1, mlp, (wb, wcs, adt, chunk) = rec
        F, N, eps = self.emb_features, self.ssm_state_dim, self.norm_epsilon
        dev = x.device
        M = x.shape[0]
        s5 = self._s5_names(n)
        nd = len(s5)
        S2 = 2 * nd * N
        dada = torch.empty((B, 6 * F), dtype=F32, device=dev)
        dx1 = self._mlp_bwd(n, dx2, x1, ada, mlp, dada, W16, Gd, L)
        dy = ops.dit_gate_bwd(dx1, y, L, ada[:, 5 * F:], dada[:, 5 * F:])
        u, _, _ = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps, stats=False)
        if nd == 2:
            go = Gd[f"{n}/ssm/out_proj/kernel"]
            _dense_wgrad(go[:F], ys[0], dy)
            _dense_wgrad(go[F:], ys[1], dy)
            ops.colsum_rows(dy, Gd[f"{n}/ssm/out_proj/bias"])
            wo = W16[f"{n}/ssm/out_proj/kernel"]
            dys = [_dense_dgrad(dy, wo[:F]), _dense_dgrad(dy, wo[F:])]
        else:
            dys = [dy]
        del dy
        # y_d = Re(C x_d) + D * u: dD, the D * dy_d term of du, dC and dx_d = dy_d [C_re, -C_im] (f32)
        dX = torch.empty((M, S2), dtype=F32, device=dev)
        dgate = torch.empty((B, F), dtype=F32, device=dev)
        dwcs, du_d = [], None
        for d, base in enumerate(s5):
            Dd = W32[f"{base}/D"].expand(B, F)
            du_dy = ops.dit_gate_bwd(dys[d], u, L, Dd, dgate)
            Gd[f"{base}/D"].add_(dgate.sum(0))
            if d == 0:
                du_d = du_dy
            ops.gemm(GEMM_KK, dys[d], wcs[d], dX[:, 2 * d * N:], M, 2 * N, F, F, F, S2)
            dwc = torch.zeros((2 * N, F), dtype=F32, device=dev)
            _dense_wgrad(dwc, x16[:, 2 * d * N:2 * (d + 1) * N], dys[d])
            dwcs.append(dwc)
        lam, dab, dgb = ops.ssm_scan_bwd(dX, xs, bu, adt, B, N, nd, chunk)
        del dX
        dwb = torch.zeros((S2, F), dtype=F32, device=dev)
        _dense_wgrad(dwb, lam, u)
        for d, base in enumerate(s5):
            ops.ssm_discretize_bwd(self._s5_leaves(W32, base), self._s5_leaves(Gd, base), N, F, dwb, 2 * d * N,
                                   dwcs[d], dab, dgb)
        # du = Re(Bbar^H lambda) over every direction + sum_d D_d * dy_d
        dn1 = _dense_dgrad(lam, wb, res=du_d)
        del lam, u
        if nd == 2:
            ops.dit_gate_fwd(dn1, dys[1], L, W32[f"{s5[1]}/D"].expand(B, F), out=dn1)
        dx0 = ops.dit_adaln_bwd(x, dn1, L, m1, r1, dada[:, 3 * F:4 * F], dada[:, 4 * F:5 * F], ada=ada,
                                scale_off=3 * F, addend=dx1)
        self._ada_bwd(n, dada, cond16, dcond, Gd, W16)
        return dx0
