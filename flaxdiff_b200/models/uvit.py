"""`UViT` - the reference's U-shaped ViT (flaxdiff/models/simple_vit.py:18-250) on the engine, with the same program
interface as `SimpleDiT`, `SimpleUDiT` and `Unet` (init / apply / forward / backward / layout / config / param_specs),
so GeneralDiffusionTrainer, the samplers and the checkpoint writer take it unchanged.

    model = UViT(patch_size=2, emb_features=768, num_layers=12, num_heads=12)
    params = model.init(key, textcontext=None)            # {'params': tree}, flax names
    y = model.apply(params, x, temb, textcontext)         # (B, H, W, out) f32; textcontext [B, T, D] or None

What differs from SimpleUDiT, and how it runs:
  * No adaLN.  The time embedding (FourierEmbedding -> TimeProjection: Dense, gelu, Dense, gelu in f32, the UNet's
    fdx_time_embed kernels) and text_proj's rows (3-D text only, not pooled) are TOKENS: the sequence is
    [patches + pos_encoding | time | text], L = N + 1 + T, assembled by fdx_uvit_assemble_fwd.  pos_encoding is a
    learned f32 table (1, (512 / p)^2, F); its gradient is the batch sum of the patch rows' gradient, formed in a fixed
    order by fdx_uvit_assemble_bwd.
  * Every block is the UNet's TransformerBlock program (Unet._tblock_fwd / _tblock_bwd) on token rows viewed as
    [B, L, 1, F], with only_pure_attention=False, norm_epsilon from the constructor and use_projection /
    use_self_and_cross / norm_inputs / explicitly_add_residual as given.  With the defaults a block is the cross-only
    path with context = x: h = x + Attention2(norm2(x), x); h = h + ff(norm3(h)); out = x + h.
  * The U: down_block_{i} outputs are pushed as skips, mid_block, then per up layer i up_dense_{i} over [x, popped
    skip] on fdx_gemm_cat (the concatenation is never written) and up_block_{i}; SimpleUDiT's backward program.
  * final_norm (LayerNorm with scale and bias) and final_proj (bf16 Dense) read the first N rows of each sample.
    Under use_hilbert, `hilbert_projection` replaces `patch_embed`; sequence position s holds row-major patch
    idx[idx[s]] (hilbert_patchify already orders the patches, and __call__ gathers by idx again), and the output goes
    back through inv_idx once.  Both gathers are one fdx_permute_rows each, the first over the raw patch rows.
  * add_residualblock_output=True adds the convolutional head: final_conv1 (3x3, 6 -> 64, bf16, over
    concat([x, x_image]) read through fdx_im2col3x3_c6, so the concat is never written), final_norm_conv + activation
    (fdx_uvit_head_norm, swish or mish), final_conv2 (3x3, 64 -> out, float32: the kernel enters as bf16(W) plus
    bf16(W - bf16(W)) through fdx_gemm_cat, then fdx_col2im3x3_c3).
  * The residual stream is stored in bf16, as in every model here; the reference carries it in f32 from the position
    add on.  Each add runs in f32 inside a GEMM epilogue or a streaming kernel and is rounded once (DESIGN.md, UViT).

Refused with FdxError: use_flash_attention=True, a dtype other than bf16, odd num_layers, emb_features not a multiple
of num_heads or of 64 or above 1024, head widths above 256, images not divisible by the patch size or with more
patches than pos_encoding has rows, inputs with other than 3 channels, 2-D text, and the head with output_channels != 3.
dropout_rate, norm_groups, force_fp32_for_softmax, use_remat and precision are accepted and ignored.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops
from .._lib import GEMM_KMN, GEMM_MNMN, FdxError
from .simple_dit import BF16, F32, SimpleDiT, _round_up
from .simple_unet import Node, Unet, _dense_dgrad, _dense_wgrad
from .ssm_dit import hilbert_indices


def _act_code(activation) -> int:
    """swish / silu -> 1, mish -> 2 (the two activations fdx_uvit_head_norm implements)."""
    name = activation if isinstance(activation, str) else getattr(activation, "__name__", repr(activation))
    if name in ("swish", "silu"):
        return ops.ACT_SILU
    if name == "mish":
        return ops.ACT_MISH
    raise FdxError(f"UViT: activation {name!r} is not supported (the output head implements swish / silu and mish)")


class UViT(SimpleDiT):
    _text_proj = "text_proj"
    # TransformerBlock's program, shared with the UNet (it reads only these methods of its instance)
    _tblock_fwd = Unet._tblock_fwd
    _tblock_bwd = Unet._tblock_bwd
    _mha_fwd = Unet._mha_fwd
    _mha_bwd = Unet._mha_bwd
    _pad_heads = staticmethod(Unet._pad_heads)
    _add2d = staticmethod(Unet._add2d)

    def __init__(self, output_channels: int = 3, patch_size: int = 16, emb_features: int = 768, num_layers: int = 12,
                 num_heads: int = 12, dropout_rate: float = 0.1, use_projection: bool = False,
                 use_flash_attention: bool = False, use_self_and_cross: bool = False,
                 force_fp32_for_softmax: bool = True, activation="swish", norm_groups: int = 8, dtype=None,
                 precision=None, add_residualblock_output: bool = False, norm_inputs: bool = False,
                 explicitly_add_residual: bool = True, norm_epsilon: float = 1e-5, use_hilbert: bool = False,
                 use_remat: bool = False, context_dim: Optional[int] = None):
        name = type(self).__name__
        self.output_channels = output_channels
        self.patch_size = patch_size
        self.emb_features = emb_features
        self.num_layers = num_layers
        self.num_heads = num_heads
        self.dropout_rate = dropout_rate        # accepted and ignored, with norm_groups, force_fp32_for_softmax,
        self.norm_groups = norm_groups          # use_remat and precision, as SimpleUDiT does with its equivalents
        self.force_fp32_for_softmax = force_fp32_for_softmax
        self.use_remat = use_remat
        self.precision = precision
        self.dtype = dtype
        self.use_flash_attention = use_flash_attention
        self.use_projection = use_projection
        self.use_self_and_cross = use_self_and_cross
        self.activation = activation
        self.add_residualblock_output = add_residualblock_output
        self.norm_inputs = norm_inputs
        self.explicitly_add_residual = explicitly_add_residual
        self.norm_epsilon = norm_epsilon
        self.use_hilbert = use_hilbert
        self.use_zigzag = False
        self.learn_sigma = False
        self.mlp_ratio = 4
        self.context_dim = context_dim          # text_proj exists only when init saw a context (as Unet.context_dim)
        if use_flash_attention:
            raise FdxError(f"{name}: use_flash_attention=True has no counterpart here; the fused attention kernel is "
                           "always used")
        if dtype is not None and dtype != torch.bfloat16:
            raise FdxError(f"{name}: dtype={dtype} is not supported: the engine computes in bf16 with f32 "
                           "accumulation (pass dtype=None or torch.bfloat16)")
        if num_layers % 2:
            raise FdxError(f"{name}: num_layers={num_layers} must be even (a U of num_layers / 2 down and up blocks "
                           "around a middle block)")
        F, h = emb_features, num_heads
        if h <= 0 or F % h:
            raise FdxError(f"{name}: emb_features={F} is not a multiple of num_heads={h}")
        if F // h > 256:
            raise FdxError(f"{name}: head width {F // h} > 256 is not supported by the fused attention")
        if F % 64 or F > 1024:
            raise FdxError(f"{name}: emb_features={F} must be a multiple of 64, at most 1024")
        if add_residualblock_output:
            self._act = _act_code(activation)
            if output_channels != 3:
                raise FdxError(f"{name}: add_residualblock_output needs output_channels=3 (the head's convolutions "
                               f"run on 3-channel images), got {output_channels}")
        self._layouts = {}
        self._consts = {}

    # ------------------------------------------------------------------ structure
    def config(self) -> dict:
        """The constructor arguments (a config round trip: UViT(**model.config()))."""
        keys = ("output_channels", "patch_size", "emb_features", "num_layers", "num_heads", "dropout_rate",
                "use_projection", "use_flash_attention", "use_self_and_cross", "force_fp32_for_softmax", "activation",
                "norm_groups", "dtype", "precision", "add_residualblock_output", "norm_inputs",
                "explicitly_add_residual", "norm_epsilon", "use_hilbert", "use_remat", "context_dim")
        return {k: getattr(self, k) for k in keys}

    def max_patches(self) -> int:
        return (512 // self.patch_size) ** 2

    def _acfg(self) -> dict:
        return {"heads": self.num_heads, "only_pure_attention": False, "use_projection": self.use_projection,
                "use_self_and_cross": self.use_self_and_cross, "norm_inputs": self.norm_inputs,
                "explicitly_add_residual": self.explicitly_add_residual, "eps": self.norm_epsilon}

    def _block_names(self):
        h = self.num_layers // 2
        return [f"down_block_{i}" for i in range(h)] + ["mid_block"] + [f"up_block_{i}" for i in range(h)]

    def _blocks(self):
        return [(n, None, None) for n in self._block_names()]

    def _block_specs(self, n):
        """TransformerBlock `n` (attention.py:305-380) with only_pure_attention=False; up_dense_{i} precedes
        up_block_{i}."""
        F, h = self.emb_features, self.num_heads
        d = F // h
        specs = []
        if n.startswith("up_block_"):
            i = n[len("up_block_"):]
            specs += [(f"up_dense_{i}/kernel", (2 * F, F)), (f"up_dense_{i}/bias", (F,))]
        if self.norm_inputs:
            specs += [(f"{n}/RMSNorm_0/scale", (F,))]
        if self.use_projection:
            specs += [(f"{n}/project_in/kernel", (F, F))]
        pre = f"{n}/Attention"
        mhas = ["Attention1", "Attention2"] if self.use_self_and_cross else ["Attention2"]
        for a in mhas:
            specs += [(f"{pre}/{a}/to_q/kernel", (F, h, d)), (f"{pre}/{a}/to_k/kernel", (F, h, d)),
                      (f"{pre}/{a}/to_v/kernel", (F, h, d)), (f"{pre}/{a}/to_out_0/kernel", (h, d, F))]
        specs += [(f"{pre}/ff/net_0/proj/kernel", (F, 8 * F)), (f"{pre}/ff/net_0/proj/bias", (8 * F,)),
                  (f"{pre}/ff/net_2/kernel", (4 * F, F)), (f"{pre}/ff/net_2/bias", (F,))]
        if self.use_self_and_cross:
            specs += [(f"{pre}/norm1/scale", (F,))]
        specs += [(f"{pre}/norm2/scale", (F,)), (f"{pre}/norm3/scale", (F,))]
        if self.use_projection:
            specs += [(f"{n}/project_out/kernel", (F, F))]
        return specs

    def _ada_leaf(self, n: str) -> str:
        """Block n's first own parameter in the layout (up_dense_{i} is announced with it)."""
        return self._block_specs(n)[2 if n.startswith("up_block_") else 0][0]

    def param_specs(self):
        F, p, out = self.emb_features, self.patch_size, self.output_channels
        specs = self._embed_specs() + [("pos_encoding", (1, self.max_patches(), F)),
                                       ("time_embed/layers_1/DenseGeneral_0/kernel", (F, F)),
                                       ("time_embed/layers_1/DenseGeneral_0/bias", (F,)),
                                       ("time_embed/layers_1/DenseGeneral_1/kernel", (F, F)),
                                       ("time_embed/layers_1/DenseGeneral_1/bias", (F,))]
        if self.context_dim:
            specs += [("text_proj/kernel", (self.context_dim, F)), ("text_proj/bias", (F,))]
        for n in self._block_names():
            specs += self._block_specs(n)
        specs += [("final_norm/scale", (F,)), ("final_norm/bias", (F,)),
                  ("final_proj/kernel", (F, p * p * out)), ("final_proj/bias", (p * p * out,))]
        if self.add_residualblock_output:
            specs += [("final_conv1/conv/kernel", (3, 3, 3 + out, 64)), ("final_conv1/conv/bias", (64,)),
                      ("final_norm_conv/scale", (64,)), ("final_norm_conv/bias", (64,)),
                      ("final_conv2/conv/kernel", (3, 3, 64, out)), ("final_conv2/conv/bias", (out,))]
        return specs

    def _embed_name(self) -> str:
        return "hilbert_projection" if self.use_hilbert else super()._embed_name()

    def _embed_specs(self):
        if not self.use_hilbert:
            return super()._embed_specs()
        p, F = self.patch_size, self.emb_features
        return [("hilbert_projection/kernel", (p * p * 3, F)), ("hilbert_projection/bias", (F,))]

    def _scan_indices(self, HP: int, WP: int):
        """The Hilbert order as row-major indices, or None (raster)."""
        return hilbert_indices(HP, WP) if self.use_hilbert else None

    def _order(self, HP: int, WP: int, device):
        """(input gather idx[idx], output gather inv_idx, its inverse idx) as int32 device tensors, or None."""
        idx = self._scan_indices(HP, WP)
        if idx is None:
            return None
        key = ("uvit_order", str(device), HP, WP)
        if key not in self._consts:
            import numpy as np
            inv = np.empty_like(idx)
            inv[idx] = np.arange(len(idx))
            self._consts[key] = tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)
                                      for a in (idx[idx], inv, idx))
        return self._consts[key]

    def _pos_table(self, device, HP: int, WP: int):
        return None             # the learned table is added by the sequence assembly

    def _init_leaf(self, name: str, t: torch.Tensor, gen: torch.Generator) -> None:
        """pos_encoding: normal(0.02); the rest as flax's defaults (lecun-normal kernels, zero biases, unit scales,
        zero final_proj kernel)."""
        if name == "pos_encoding":
            t.normal_(0.0, 0.02, generator=gen)
        else:
            super()._init_leaf(name, t, gen)

    # ------------------------------------------------------------------ forward program
    def forward(self, fp, x: torch.Tensor, temb: torch.Tensor, textcontext=None, save: bool = True):
        """x (B, H, W, 3) bf16 or f32 -> (F f32 (B, H, W, output_channels), tape or None)."""
        name = type(self).__name__
        B, H, W, C = x.shape
        p, F = self.patch_size, self.emb_features
        if C != 3:
            raise FdxError(f"{name}: the input must have 3 channels, got {C}")
        if H % p or W % p:
            raise FdxError(f"{name}: image {H}x{W} is not divisible by the patch size {p}")
        HP, WP = H // p, W // p
        N = HP * WP
        if N > self.max_patches():
            raise FdxError(f"{name}: {N} patches exceed pos_encoding's {self.max_patches()} rows ((512 / p)^2)")
        if textcontext is not None and textcontext.dim() != 3:
            raise FdxError(f"{name}: textcontext must be [B, T, D] (the text tokens join the sequence), got "
                           f"{tuple(textcontext.shape)}")
        if textcontext is not None and int(textcontext.shape[-1]) != (self.context_dim or -1):
            raise FdxError(f"{name}: textcontext width {tuple(textcontext.shape)} does not match the parameters "
                           f"(context_dim={self.context_dim}); build / init the model with it")
        if textcontext is None and self.context_dim is not None:
            raise FdxError(f"{name}: parameters were built with text_proj but textcontext is None")
        W32, W16 = fp.named, fp.shadow()
        dev = x.device
        T = int(textcontext.shape[1]) if textcontext is not None else 0
        L = N + 1 + T
        sv = {"B": B, "H": H, "W": W, "N": N, "T": T, "L": L, "x": x}

        # time token: FourierEmbedding -> TimeProjection in f32, then bf16 --------------------------------------------
        te = "time_embed/layers_1/DenseGeneral_"
        t = temb.reshape(-1).to(F32)
        if t.numel() == 1 and B > 1:
            t = t.expand(B)
        _, emb16, sv["temb"] = ops.time_embed_fwd(t.contiguous(), self._fourier_freqs(dev), W32[te + "0/kernel"],
                                                  W32[te + "0/bias"], W32[te + "1/kernel"], W32[te + "1/bias"])
        # text tokens: text_proj over every token ---------------------------------------------------------------------
        txt = None
        if T:
            tc16 = self._text_rows(textcontext, B).view(B * T, -1)
            txt = ops.linear_fwd(tc16, W16["text_proj/kernel"], bias=W32["text_proj/bias"])
            sv["text_rows"] = tc16
        # patches (in the sequence order) + pos_encoding, then the sequence -------------------------------------------
        order = self._order(HP, WP, dev)
        ptok, sv["patch_rows"] = self._embed_fwd(x, W32, W16, HP, WP, order)
        tok = ops.uvit_assemble_fwd(ptok, W32["pos_encoding"].view(-1, F), emb16, txt, B, N, T)
        del ptok, txt
        sv["order"] = order

        tok, sv["blocks"] = self._trunk_fwd(tok, W32, W16, B, L)
        out, sv["final"] = self._final_fwd(tok, W32, W16, B, H, W, N, L, order)
        if self.add_residualblock_output:
            out, sv["head"] = self._head_fwd(x, out, W32, W16)
        return (out, sv) if save else (out, None)

    def _block_fwd(self, n, tok, W32, W16, B, L):
        F = self.emb_features
        out = torch.empty_like(tok)
        rec = self._tblock_fwd(n, Node(tok.view(B, L, 1, F)), Node(out.view(B, L, 1, F)), self._acfg(), W32, W16)
        return out, rec

    def _trunk_fwd(self, tok, W32, W16, B: int, L: int):
        """down blocks -> mid block -> (up_dense over [x, popped skip], up block) -> (tokens, tape)."""
        h = self.num_layers // 2
        recs, skips, ups = {}, [], []
        for i in range(h):
            tok, recs[f"down_block_{i}"] = self._block_fwd(f"down_block_{i}", tok, W32, W16, B, L)
            skips.append(tok)
        tok, recs["mid_block"] = self._block_fwd("mid_block", tok, W32, W16, B, L)
        for i in range(h):
            u = f"up_dense_{i}"
            ups.append(tok)
            tok = ops.linear_cat_fwd(tok, skips[h - 1 - i], W16[u + "/kernel"], bias=W32[u + "/bias"])
            tok, recs[f"up_block_{i}"] = self._block_fwd(f"up_block_{i}", tok, W32, W16, B, L)
        return tok, (recs, skips, ups)

    def _final_fwd(self, tok, W32, W16, B, H, W, N, L, order):
        """final_norm (every row; only the first N of each sample are read) -> final_proj over those rows (one batched
        GEMM with the sample stride L * F, f32 out, columns zero-padded to 32) -> unpatchify."""
        p, F, out = self.patch_size, self.emb_features, self.output_channels
        xf, mf, rf = ops.dit_adaln_fwd(tok, L, gamma=W32["final_norm/scale"], beta=W32["final_norm/bias"],
                                       eps=self.norm_epsilon)
        P_ = p * p * out
        Np = _round_up(P_, 32)
        wfp = torch.nn.functional.pad(W16["final_proj/kernel"], (0, Np - P_)).contiguous()
        bfp = torch.nn.functional.pad(W32["final_proj/bias"], (0, Np - P_)).contiguous()
        yf = torch.empty((B * N, Np), dtype=F32, device=tok.device)
        ops.gemm(GEMM_KMN, xf, wfp, yf, N, Np, F, F, Np, Np, batch1=B, a_s=(L * F, 0), d_s=(N * Np, 0), bias=bfp)
        if order is not None:
            yf = ops.permute_rows(yf, order[1])
        return ops.dit_unpatchify(yf, B, H, W, out, p), (tok, mf, rf, xf, wfp)

    def _head_fwd(self, x, ximg, W32, W16):
        """final_conv1 over concat([bf16(x), x_image]) -> final_norm_conv + activation -> the float32 final_conv2."""
        B, H, W, _ = x.shape
        col = ops.im2col3_c6(x, ximg)
        w1 = W16["final_conv1/conv/kernel"].reshape(9, 6, 64)
        wc1 = torch.zeros((64, 64), dtype=BF16, device=x.device)
        wc1[:27] = w1[:, :3].reshape(27, 64)
        wc1[32:59] = w1[:, 3:].reshape(27, 64)
        z1 = ops.linear_fwd(col, wc1, bias=W32["final_conv1/conv/bias"])
        a = ops.uvit_head_norm_fwd(z1, W32["final_norm_conv/scale"], W32["final_norm_conv/bias"], self.norm_epsilon,
                                   self._act)
        # final_conv2 in f32: [a | a] x [W_hi; W_lo] (exact bf16 products, f32 sums), then the taps' scatter + bias
        wr = W32["final_conv2/conv/kernel"].reshape(9, 64, 3).permute(1, 0, 2).reshape(64, 27)
        w_hi = ops.cast_f32_bf16(wr.contiguous())
        w_lo = ops.cast_f32_bf16((wr - w_hi.float()).contiguous())
        wsplit = torch.zeros((128, 32), dtype=BF16, device=x.device)
        wsplit[:64, :27] = w_hi
        wsplit[64:, :27] = w_lo
        P = B * H * W
        c2 = torch.empty((P, 32), dtype=F32, device=x.device)
        ops.gemm_cat(GEMM_KMN, a, a, wsplit, c2, P, 32, 128, 64, 64, 64, 32, 32)
        y = ops.col2im3(c2, W32["final_conv2/conv/bias"], B, H, W)
        return y, (col, z1, a)

    # ------------------------------------------------------------------ backward program
    def backward(self, fp, saved: dict, dF: torch.Tensor, grads, on_ready=None):
        """Accumulates d(loss)/d(params) into `grads` (f32, zeroed by the caller) given dF = dL/dF (B, H, W, out) f32.
        `on_ready(lo, streams)`: every gradient at flat offset >= lo is final once the queued work has run."""
        W32, W16, Gd = fp.named, fp.shadow(), grads.named
        B, N, T, L = saved["B"], saved["N"], saved["T"], saved["L"]
        lay = fp.layout
        stream = [torch.cuda.current_stream()]

        def ready(leaf: str) -> None:
            if on_ready is not None:
                on_ready(lay.table[leaf][0], stream)

        dF = dF.contiguous()
        if self.add_residualblock_output:
            dF = self._head_bwd(saved["head"], saved["x"], dF, W32, Gd)
        dx = self._final_bwd(saved["final"], dF, saved["order"], W32, Gd, N, L)
        ready("final_norm/scale")
        dx = self._trunk_bwd(saved["blocks"], dx, W32, W16, Gd, B, L, ready)

        F = self.emb_features
        dpos = Gd["pos_encoding"].view(-1, F)[:N]
        dpatch, dtime, dtext = ops.uvit_assemble_bwd(dx, B, N, T, dpos)
        del dx
        self._embed_bwd(saved["patch_rows"], dpatch, Gd)
        if T:
            _dense_wgrad(Gd["text_proj/kernel"], saved["text_rows"], dtext)
            ops.colsum_rows(dtext, Gd["text_proj/bias"])
        te = "time_embed/layers_1/DenseGeneral_"
        ops.time_embed_bwd(dtime, saved["temb"], W32[te + "1/kernel"], Gd[te + "0/kernel"], Gd[te + "0/bias"],
                           Gd[te + "1/kernel"], Gd[te + "1/bias"])
        if on_ready is not None:
            on_ready(0, stream)

    def _head_bwd(self, tape, x, dF, W32, Gd):
        """Backward of _head_fwd -> d(x_image) f32 (B, H, W, 3); the x half of the concat needs no gradient."""
        col, z1, a = tape
        B, H, W, _ = dF.shape
        P = B * H * W
        w2 = W32["final_conv2/conv/kernel"]
        dcol = ops.im2col3(dF, -1, False)                       # shared by final_conv2's two gradients
        da = torch.empty((B, H, W, 64), dtype=BF16, device=dF.device)
        ops.conv_out_dgrad(dF, w2, da, col=dcol)
        ops.conv_out_wgrad(a.view(B, H, W, 64), dF, Gd["final_conv2/conv/kernel"], Gd["final_conv2/conv/bias"],
                           col=dcol)
        del dcol
        dz1 = ops.uvit_head_norm_bwd(z1, da.view(P, 64), W32["final_norm_conv/scale"], W32["final_norm_conv/bias"],
                                     self.norm_epsilon, self._act, Gd["final_norm_conv/scale"],
                                     Gd["final_norm_conv/bias"])
        del da
        gw = torch.zeros((64, 64), dtype=F32, device=dF.device)
        ops.gemm(GEMM_MNMN, col, dz1, gw, 64, 64, P, 64, 64, 64, atomic=True, reduce_batch=True)
        g1 = Gd["final_conv1/conv/kernel"].view(9, 6, 64)
        g1[:, :3].add_(gw[:27].view(9, 3, 64))
        g1[:, 3:].add_(gw[32:59].view(9, 3, 64))
        ops.colsum_rows(dz1, Gd["final_conv1/conv/bias"])
        # d x_image[q][c] = sum_t sum_co dz1[q - d(t)][co] w1[t][3 + c][co]: a 64 -> 3 convolution of dz1 with the
        # image half of the kernel, taps mirrored
        w1 = W32["final_conv1/conv/kernel"].reshape(9, 6, 64)
        wflip = w1.flip(0)[:, 3:].permute(0, 2, 1).reshape(3, 3, 64, 3).contiguous()
        return ops.conv_out_fwd(dz1.view(B, H, W, 64), wflip, None)

    def _final_bwd(self, tape, dF, order, W32, Gd, N, L):
        """Backward of _final_fwd -> d(tokens) bf16 [B * L, F] (zero past the first N rows of each sample before the
        LayerNorm backward)."""
        tok, mf, rf, xf, wfp = tape
        p, F, out = self.patch_size, self.emb_features, self.output_channels
        P_ = p * p * out
        Np = wfp.shape[1]
        B = dF.shape[0]
        dY = ops.dit_patchify(dF, p, Np)
        if order is not None:
            dY = ops.permute_rows(dY, order[2])
        dYf = torch.zeros((B, L, Np), dtype=BF16, device=dF.device)
        dYf[:, :N] = dY.view(B, N, Np)
        dYf = dYf.view(B * L, Np)
        gw = torch.zeros((F, Np), dtype=F32, device=dF.device)
        ops.gemm(GEMM_MNMN, xf, dYf, gw, F, Np, xf.shape[0], F, Np, Np, atomic=True, reduce_batch=True)
        Gd["final_proj/kernel"].add_(gw[:, :P_])
        gb = torch.zeros(Np, dtype=F32, device=dF.device)
        ops.colsum_rows(dYf, gb)
        Gd["final_proj/bias"].add_(gb[:P_])
        dxf = _dense_dgrad(dYf, wfp)
        return ops.dit_adaln_bwd(tok, dxf, L, mf, rf, Gd["final_norm/scale"], Gd["final_norm/bias"],
                                 gamma=W32["final_norm/scale"], reduce_samples=True, accumulate=True)

    def _block_bwd(self, rec, dout, W32, W16, Gd, B, L):
        """Backward of one TransformerBlock -> d(input) bf16 [B * L, F]."""
        F = self.emb_features
        got = {}

        def want(node):
            got["dx"] = torch.empty((B, L, 1, F), dtype=BF16, device=dout.device)
            return got["dx"], False
        r = self._tblock_bwd(rec, W32, W16, Gd, want, lambda node: dout.view(B, L, 1, F))
        return r if r is not None else got["dx"].view(B * L, F)

    def _trunk_bwd(self, tape, dx, W32, W16, Gd, B: int, L: int, ready):
        """Backward of _trunk_fwd (SimpleUDiT's program): the gradient of down_block_{j}'s output is the next block's
        input gradient plus the skip half of the up_dense that popped it, added in the epilogue of that half's
        product."""
        recs, skips, ups = tape
        h, F = self.num_layers // 2, self.emb_features
        dys = [None] * h
        for i in reversed(range(h)):
            n, u = f"up_block_{i}", f"up_dense_{i}"
            dx = self._block_bwd(recs[n], dx, W32, W16, Gd, B, L)
            j = h - 1 - i
            g = Gd[u + "/kernel"]
            _dense_wgrad(g[:F], ups[i], dx)
            _dense_wgrad(g[F:], skips[j], dx)
            ops.colsum_rows(dx, Gd[u + "/bias"])
            dys[j] = dx
            dx = _dense_dgrad(dx, W16[u + "/kernel"][:F])
            ready(u + "/kernel")
        dx = self._block_bwd(recs["mid_block"], dx, W32, W16, Gd, B, L)
        ready(self._ada_leaf("mid_block"))
        for j in reversed(range(h)):
            n = f"down_block_{j}"
            dx = _dense_dgrad(dys[j], W16[f"up_dense_{h - 1 - j}/kernel"][F:], res=dx)
            dys[j] = None
            dx = self._block_bwd(recs[n], dx, W32, W16, Gd, B, L)
            ready(self._ada_leaf(n))
        return dx
