"""`SimpleUDiT` - the reference's U-shaped DiT (flaxdiff/models/simple_vit.py:255-446) on the engine, with the same
program interface as `SimpleDiT` and `Unet` (init / apply / forward / backward / layout / config), so
GeneralDiffusionTrainer, the samplers and the checkpoint writer take it unchanged.

    model = SimpleUDiT(patch_size=2, emb_features=768, num_layers=12, num_heads=12)
    params = model.init(key, textcontext=None)            # {'params': tree}, flax names
    y = model.apply(params, x, temb, textcontext)         # (B, H, W, 3) f32; textcontext [B, S, D], [B, D] or None

What differs from SimpleDiT, and how it runs:
  * SimpleDiT's DiTBlock arranged as a U: down_block_{i} for i < num_layers / 2, mid_block, then per up layer i
    up_dense_{i} (a Dense with a [2F, F] kernel over concat([x, skip], -1)) and up_block_{i}.  The skips are popped, so
    up layer i pairs with down_block_{half-1-i}.  num_layers = 12 is 13 DiT blocks.
  * up_dense runs on fdx_gemm_cat: the GEMM reads its A operand from x for k < F and from the skip for k >= F, so the
    [B*L, 2F] concatenation is never written (forward) or kept (backward).  Its backward is two products against the
    kernel's row halves for d(x) and d(skip), and two weight-gradient products into the gradient's row halves.  d(skip)
    is formed when the backward reaches the down block: one product whose bf16 side input is the gradient arriving
    from the next block, so the two are added in its f32 epilogue.
  * final_proj is float32 (nn.Dense(dtype=float32)): the bf16 final_norm output times the f32 kernel.  It runs as
    fdx_gemm_cat([xf | xf], [W_hi; W_lo]) with W_hi = bf16(W), W_lo = bf16(W - W_hi): every product of two bf16 values
    is exact in the f32 accumulator, so the kernel enters with about 2^-16 relative error instead of bf16's 2^-9.  Its
    backward is SimpleDiT's bf16 product with W_hi.
  * No sin-cos position table: RoPE is on in both patch orders (under use_hilbert, positions are indices along the
    Hilbert sequence).  Under use_hilbert, `hilbert_projection` replaces `patch_embed` (which then has no parameters),
    the patch rows are permuted on the device and the output rows go back through the inverse order.
  * Text: `text_proj` (not text_context_proj), mean-pooled over tokens only when the text is 3-D.  Pooling first is
    exact by linearity, bias included.

Refused with FdxError: odd num_layers, and what SimpleDiT refuses (use_flash_attention=True, a dtype other than bf16,
emb_features not a multiple of num_heads or of 64 or above 1536, odd head widths and heads wider than 256, images not
divisible by the patch size).  dropout_rate, norm_groups, activation and force_fp32_for_softmax are accepted and
ignored, as in the reference.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops
from .._lib import GEMM_KMN, FdxError
from .simple_dit import BF16, F32, SimpleDiT, _round_up
from .simple_unet import _dense_dgrad, _dense_wgrad
from .ssm_dit import hilbert_indices


class SimpleUDiT(SimpleDiT):
    _text_proj = "text_proj"

    def __init__(self, output_channels: int = 3, patch_size: int = 16, emb_features: int = 768, num_layers: int = 12,
                 num_heads: int = 12, mlp_ratio: int = 4, dropout_rate: float = 0.0, dtype=None, precision=None,
                 use_flash_attention: bool = False, force_fp32_for_softmax: bool = True, norm_epsilon: float = 1e-5,
                 learn_sigma: bool = False, use_hilbert: bool = False, norm_groups: int = 0, activation=None,
                 context_dim: Optional[int] = None):
        if num_layers % 2:
            raise FdxError(f"{type(self).__name__}: num_layers={num_layers} must be even (a U of num_layers / 2 down "
                           "and up blocks around a middle block)")
        super().__init__(output_channels=output_channels, patch_size=patch_size, emb_features=emb_features,
                         num_layers=num_layers, num_heads=num_heads, mlp_ratio=mlp_ratio, dropout_rate=dropout_rate,
                         dtype=dtype, precision=precision, use_flash_attention=use_flash_attention,
                         force_fp32_for_softmax=force_fp32_for_softmax, norm_epsilon=norm_epsilon,
                         learn_sigma=learn_sigma, norm_groups=norm_groups, activation=activation,
                         context_dim=context_dim)
        self.use_hilbert = use_hilbert

    # ------------------------------------------------------------------ structure
    def config(self) -> dict:
        """The constructor arguments (a config round trip: SimpleUDiT(**model.config()))."""
        keys = ("output_channels", "patch_size", "emb_features", "num_layers", "num_heads", "mlp_ratio",
                "dropout_rate", "dtype", "precision", "use_flash_attention", "force_fp32_for_softmax", "norm_epsilon",
                "learn_sigma", "use_hilbert", "norm_groups", "activation", "context_dim")
        return {k: getattr(self, k) for k in keys}

    def _blocks(self):
        """The DiT blocks in forward order; up_dense_{i} precedes up_block_{i} in the layout (_block_specs)."""
        h = self.num_layers // 2
        names = [f"down_block_{i}" for i in range(h)] + ["mid_block"] + [f"up_block_{i}" for i in range(h)]
        return [(n, self._block_fwd, self._block_bwd) for n in names]

    def _block_specs(self, n):
        specs = super()._block_specs(n)
        if n.startswith("up_block_"):
            i, F = n[len("up_block_"):], self.emb_features
            specs = [(f"up_dense_{i}/kernel", (2 * F, F)), (f"up_dense_{i}/bias", (F,))] + specs
        return specs

    def _embed_name(self) -> str:
        return "hilbert_projection" if self.use_hilbert else super()._embed_name()

    def _embed_specs(self):
        if not self.use_hilbert:
            return super()._embed_specs()
        p, F = self.patch_size, self.emb_features
        return [("hilbert_projection/kernel", (p * p * 3, F)), ("hilbert_projection/bias", (F,))]

    def _scan_indices(self, HP: int, WP: int):
        return hilbert_indices(HP, WP) if self.use_hilbert else None

    def _pos_table(self, device, HP: int, WP: int):
        return None

    def _rope(self) -> bool:
        return True

    @staticmethod
    def _pool_text(tc16: torch.Tensor) -> torch.Tensor:
        return ops.cast_f32_bf16(ops.dit_token_mean(tc16)) if tc16.dim() == 3 else tc16

    # ------------------------------------------------------------------ forward program
    def forward(self, fp, x: torch.Tensor, temb: torch.Tensor, textcontext=None, save: bool = True):
        if textcontext is not None and textcontext.dim() not in (2, 3):
            raise FdxError(f"{type(self).__name__}: textcontext must be [B, S, D] or [B, D], got "
                           f"{tuple(textcontext.shape)}")
        return super().forward(fp, x, temb, textcontext, save)

    def _trunk_fwd(self, tok, cond16, W32, W16, B: int, L: int):
        """down blocks -> mid block -> (up_dense over [x, popped skip], up block) -> (tokens, tape)."""
        h = self.num_layers // 2
        recs, skips, ups = {}, [], []
        for i in range(h):
            tok, recs[f"down_block_{i}"] = self._block_fwd(f"down_block_{i}", tok, cond16, W32, W16, B, L)
            skips.append(tok)
        tok, recs["mid_block"] = self._block_fwd("mid_block", tok, cond16, W32, W16, B, L)
        for i in range(h):
            u = f"up_dense_{i}"
            ups.append(tok)
            tok = ops.linear_cat_fwd(tok, skips[h - 1 - i], W16[u + "/kernel"], bias=W32[u + "/bias"])
            tok, recs[f"up_block_{i}"] = self._block_fwd(f"up_block_{i}", tok, cond16, W32, W16, B, L)
        return tok, (recs, skips, ups)

    def _final_fwd(self, tok, W32, W16, B, H, W, L, order):
        """final_norm -> the float32 final_proj as [xf | xf] x [W_hi; W_lo] (the first p*p*out columns, zero-padded to
        the GEMM's multiple of 32) -> unpatchify -> (output f32 (B, H, W, out), SimpleDiT's tape with W_hi)."""
        p, F = self.patch_size, tok.shape[1]
        xf, mf, rf = ops.dit_adaln_fwd(tok, L, gamma=W32["final_norm/scale"], beta=W32["final_norm/bias"],
                                       eps=self.norm_epsilon)
        P_ = p * p * self.output_channels
        Np = _round_up(P_, 32)
        w_hi = W16["final_proj/kernel"][:, :P_]
        w_lo = ops.cast_f32_bf16((W32["final_proj/kernel"][:, :P_] - w_hi.float()).contiguous())
        wsplit = torch.zeros((2 * F, Np), dtype=BF16, device=tok.device)
        wsplit[:F, :P_] = w_hi
        wsplit[F:, :P_] = w_lo
        bfp = torch.nn.functional.pad(W32["final_proj/bias"][:P_], (0, Np - P_)).contiguous()
        M = xf.shape[0]
        yf = torch.empty((M, Np), dtype=F32, device=tok.device)
        ops.gemm_cat(GEMM_KMN, xf, xf, wsplit, yf, M, Np, 2 * F, F, F, F, Np, Np, bias=bfp)
        if order is not None:
            yf = ops.permute_rows(yf, order[1])
        return ops.dit_unpatchify(yf, B, H, W, self.output_channels, p), (tok, mf, rf, xf, wsplit[:F])

    # ------------------------------------------------------------------ backward program
    def _trunk_bwd(self, tape, dx, cond16, dcond, W32, W16, Gd, B: int, L: int, ready):
        """Backward of _trunk_fwd.  The gradient of down_block_{j}'s output is the next block's input gradient plus
        the skip half of the up_dense that popped it, added in the epilogue of that half's product."""
        recs, skips, ups = tape
        h, F = self.num_layers // 2, self.emb_features
        dys = [None] * h                    # dys[j]: the output gradient of the up_dense whose skip is down_block_j
        for i in reversed(range(h)):
            n, u = f"up_block_{i}", f"up_dense_{i}"
            dx = self._block_bwd(recs[n], dx, cond16, dcond, W32, W16, Gd, B, L)
            ready(self._ada_leaf(n))
            j = h - 1 - i
            g = Gd[u + "/kernel"]
            _dense_wgrad(g[:F], ups[i], dx)
            _dense_wgrad(g[F:], skips[j], dx)
            ops.colsum_rows(dx, Gd[u + "/bias"])
            dys[j] = dx
            dx = _dense_dgrad(dx, W16[u + "/kernel"][:F])
            ready(u + "/kernel")
        dx = self._block_bwd(recs["mid_block"], dx, cond16, dcond, W32, W16, Gd, B, L)
        ready(self._ada_leaf("mid_block"))
        for j in reversed(range(h)):
            n = f"down_block_{j}"
            dx = _dense_dgrad(dys[j], W16[f"up_dense_{h - 1 - j}/kernel"][F:], res=dx)
            dys[j] = None
            dx = self._block_bwd(recs[n], dx, cond16, dcond, W32, W16, Gd, B, L)
            ready(self._ada_leaf(n))
        return dx
