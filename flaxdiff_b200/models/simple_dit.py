"""`SimpleDiT` - the reference's transformer denoiser (flaxdiff/models/simple_dit.py:23-306) rebuilt as an explicit
forward / backward program over libfdx kernels, with the same program interface as `Unet` (init / apply / forward /
backward / layout), so GeneralDiffusionTrainer, the samplers and the checkpoint writer take it unchanged.

    model = SimpleDiT(output_channels=3, patch_size=2, emb_features=768, num_layers=12, num_heads=12)
    params = model.init(key, textcontext=None)            # {'params': tree}, flax names
    y = model.apply(params, x, temb, textcontext)         # (B, H, W, 3) f32

Execution design: tokens are bf16 [B*L, F] row matrices.  Dense layers run on the tensor-core GEMM (QKV as one GEMM
over the concatenated, head-padded kernels), attention on the fused kernels; the streaming passes between them are
fdx_dit.cu's: adaLN LayerNorm, the gated residual, RoPE in place on the QKV output, bias + tanh-gelu, patchify /
unpatchify.  The backward is an explicit tape; every per-sample column sum is deterministic.  Raster patch order
only: the Hilbert / zigzag scans are refused at construction.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .. import ops, utils
from .._lib import ACT_GELU_TANH, GEMM_KK, GEMM_MNMN, FdxError
from .params import FlatParams, ParamLayout, from_tree
from .simple_unet import Unet, _attn_width, _dense_dgrad, _dense_wgrad

BF16 = torch.bfloat16
F32 = torch.float32


def _round_up(n: int, m: int) -> int:
    return -(-n // m) * m


def sincos_2d_table(F: int, HP: int, WP: int):
    """build_2d_sincos_pos_embed (hilbert.py:12-45) as a host constant [HP*WP, F]: quarters row-sin, row-cos, col-sin,
    col-cos, omega = 10000^(-i/quarter)."""
    import numpy as np
    quarter = F // 4
    omega = 1.0 / (10000.0 ** (np.arange(quarter, dtype=np.float32) / np.float32(quarter)))
    rows = np.arange(HP, dtype=np.float32)[:, None] * omega[None]
    cols = np.arange(WP, dtype=np.float32)[:, None] * omega[None]
    pos = np.zeros((HP, WP, F), dtype=np.float32)
    pos[..., 0:quarter] = np.sin(rows)[:, None, :]
    pos[..., quarter:2 * quarter] = np.cos(rows)[:, None, :]
    pos[..., 2 * quarter:3 * quarter] = np.sin(cols)[None, :, :]
    pos[..., 3 * quarter:] = np.cos(cols)[None, :, :]
    return pos.reshape(HP * WP, F)


class SimpleDiT:
    def __init__(self, output_channels: int = 3, patch_size: int = 16, emb_features: int = 768, num_layers: int = 12,
                 num_heads: int = 12, mlp_ratio: int = 4, dropout_rate: float = 0.0, dtype=None, precision=None,
                 use_flash_attention: bool = False, force_fp32_for_softmax: bool = True, norm_epsilon: float = 1e-5,
                 learn_sigma: bool = False, use_hilbert: bool = False, use_zigzag: bool = False, norm_groups: int = 0,
                 activation=None, context_dim: Optional[int] = None):
        self.output_channels = output_channels
        self.patch_size = patch_size
        self.emb_features = emb_features
        self.num_layers = num_layers
        self.num_heads = num_heads
        self.mlp_ratio = mlp_ratio
        self.dropout_rate = dropout_rate        # accepted and unused, as in the reference
        self.dtype = dtype
        self.precision = precision
        self.use_flash_attention = use_flash_attention
        self.force_fp32_for_softmax = force_fp32_for_softmax
        self.norm_epsilon = norm_epsilon
        self.learn_sigma = learn_sigma
        self.use_hilbert = use_hilbert
        self.use_zigzag = use_zigzag
        self.norm_groups = norm_groups          # accepted and ignored, as the reference ignores them
        self.activation = activation
        # width of `textcontext`: text_context_proj exists only when init saw a context (as Unet.context_dim)
        self.context_dim = context_dim
        if use_hilbert or use_zigzag:
            raise FdxError("SimpleDiT: the Hilbert / zigzag patch orders are not supported (raster order only)")
        if use_flash_attention:
            raise FdxError("SimpleDiT: use_flash_attention=True has no counterpart here; the fused attention kernel "
                           "is always used")
        if dtype is not None and dtype != torch.bfloat16:
            raise FdxError(f"SimpleDiT: dtype={dtype} is not supported: the engine computes in bf16 with f32 "
                           "accumulation (pass dtype=None or torch.bfloat16)")
        F, h = emb_features, num_heads
        if h <= 0 or F % h != 0:
            raise FdxError(f"SimpleDiT: emb_features={F} is not a multiple of num_heads={h}")
        d = F // h
        if d % 2:
            raise FdxError(f"SimpleDiT: head width {d} is odd (RoPE rotates channel pairs)")
        if d > 256:
            raise FdxError(f"SimpleDiT: head width {d} > 256 is not supported by the fused attention")
        if F % 64 or F > 1536:
            raise FdxError(f"SimpleDiT: emb_features={F} must be a multiple of 64, at most 1536")
        self._layouts: Dict[Optional[int], ParamLayout] = {}
        self._consts: Dict[tuple, torch.Tensor] = {}

    # ------------------------------------------------------------------ structure
    def param_specs(self):
        F, h, p, E = self.emb_features, self.num_heads, self.patch_size, self.emb_features * self.mlp_ratio
        d = F // h
        nout = p * p * self.output_channels * (2 if self.learn_sigma else 1)
        specs = [("patch_embed/Conv_0/kernel", (p, p, 3, F)), ("patch_embed/Conv_0/bias", (F,)),
                 ("time_embed/layers_1/DenseGeneral_0/kernel", (F, E)), ("time_embed/layers_1/DenseGeneral_0/bias", (E,)),
                 ("time_embed/layers_1/DenseGeneral_1/kernel", (E, E)), ("time_embed/layers_1/DenseGeneral_1/bias", (E,)),
                 ("time_embed/layers_2/kernel", (E, F)), ("time_embed/layers_2/bias", (F,))]
        if self.context_dim:
            specs += [("text_context_proj/kernel", (self.context_dim, F)), ("text_context_proj/bias", (F,))]
        for i in range(self.num_layers):
            n = f"dit_block_{i}"
            specs += [(f"{n}/ada_params_module/ada_proj/kernel", (F, 6 * F)),
                      (f"{n}/ada_params_module/ada_proj/bias", (6 * F,))]
            for m in ("to_q", "to_k", "to_v"):
                specs += [(f"{n}/attention/{m}/kernel", (F, h, d)), (f"{n}/attention/{m}/bias", (h, d))]
            specs += [(f"{n}/attention/to_out_0/kernel", (h, d, F)), (f"{n}/attention/to_out_0/bias", (F,)),
                      (f"{n}/mlp/layers_0/kernel", (F, E)), (f"{n}/mlp/layers_0/bias", (E,)),
                      (f"{n}/mlp/layers_2/kernel", (E, F)), (f"{n}/mlp/layers_2/bias", (F,))]
        specs += [("final_norm/scale", (F,)), ("final_norm/bias", (F,)),
                  ("final_proj/kernel", (F, nout)), ("final_proj/bias", (nout,))]
        return specs

    def layout(self) -> ParamLayout:
        if self.context_dim not in self._layouts:
            self._layouts[self.context_dim] = ParamLayout(self.param_specs())
        return self._layouts[self.context_dim]

    def config(self) -> dict:
        """The constructor arguments (a config round trip: SimpleDiT(**model.config()))."""
        keys = ("output_channels", "patch_size", "emb_features", "num_layers", "num_heads", "mlp_ratio",
                "dropout_rate", "dtype", "precision", "use_flash_attention", "force_fp32_for_softmax", "norm_epsilon",
                "learn_sigma", "use_hilbert", "use_zigzag", "norm_groups", "activation", "context_dim")
        return {k: getattr(self, k) for k in keys}

    # ------------------------------------------------------------------ init
    def init(self, key, x=None, temb=None, textcontext=None, device=None) -> FlatParams:
        """flax `model.init`: lecun-normal kernels (fan-in = every axis but the last for Dense / DenseGeneral over one
        axis, (heads, d) for to_out_0), zero biases, unit final_norm scale; ada_proj and final_proj kernels zero
        (their kernel_init)."""
        if device is None:
            device = x.device if isinstance(x, torch.Tensor) else torch.device("cuda")
        if isinstance(textcontext, torch.Tensor):
            self.context_dim = int(textcontext.shape[-1])
        fp = FlatParams(self.layout(), torch.zeros(self.layout().total, dtype=F32, device=device))
        if isinstance(key, int):
            key = utils.PRNGKey(key)
        gen = torch.Generator(device=device)
        gen.manual_seed(utils.key_to_seed(tuple(key)))
        for name, t in fp.named.items():
            leaf = name.rsplit('/', 1)[1]
            if leaf == "scale":
                t.fill_(1.0)
            elif leaf == "kernel" and not name.startswith("final_proj") and "ada_proj" not in name:
                if name.endswith("to_out_0/kernel"):
                    fan_in = t.shape[0] * t.shape[1]
                elif t.dim() == 4:
                    fan_in = t.shape[0] * t.shape[1] * t.shape[2]
                else:
                    fan_in = t.shape[0]
                std = math.sqrt(1.0 / fan_in) / 0.87962566103423978
                torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)
        return fp

    def _const(self, kind: str, device, *shape) -> torch.Tensor:
        key = (kind, str(device)) + shape
        if key not in self._consts:
            if kind == "freqs":   # FourierEmbedding.freqs: normal(PRNGKey(42), (F//2,)) * 16 (common.py:101-102)
                f = utils.normal(utils.PRNGKey(42), self.emb_features // 2) * 16.0
                self._consts[key] = torch.from_numpy(f.astype("float32")).to(device)
            else:                 # the 2-D sin-cos position table, bf16 [L, F]
                self._consts[key] = torch.from_numpy(sincos_2d_table(self.emb_features, *shape)).to(device, BF16)
        return self._consts[key]

    def _fourier_freqs(self, device) -> torch.Tensor:
        return self._const("freqs", device)

    def _as_flat(self, params, device) -> FlatParams:
        if isinstance(params, FlatParams):
            return params
        return from_tree(self.layout(), params, device)

    def apply(self, params, x: torch.Tensor, temb: torch.Tensor, textcontext=None) -> torch.Tensor:
        """`model.apply(params, x, temb, textcontext)`."""
        if not x.is_cuda:
            raise FdxError("SimpleDiT.apply: CUDA tensors required (no CPU path in flaxdiff_b200)")
        fp = self._as_flat(params, x.device)
        out, _ = self.forward(fp, x.contiguous(), temb, textcontext, save=False)
        return out

    # ------------------------------------------------------------------ forward program
    def forward(self, fp: FlatParams, x: torch.Tensor, temb: torch.Tensor, textcontext=None, save: bool = True):
        """x (B, H, W, 3) bf16 or f32 -> (F f32 (B, H, W, output_channels), tape or None)."""
        B, H, W, C = x.shape
        p, F, heads = self.patch_size, self.emb_features, self.num_heads
        if H % p or W % p:
            raise FdxError(f"SimpleDiT: image {H}x{W} is not divisible by the patch size {p}")
        if textcontext is not None and int(textcontext.shape[-1]) != (self.context_dim or -1):
            raise FdxError(f"SimpleDiT: textcontext width {tuple(textcontext.shape)} does not match the parameters "
                           f"(context_dim={self.context_dim}); build / init the model with it")
        if textcontext is None and self.context_dim is not None:
            raise FdxError("SimpleDiT: parameters were built with text_context_proj but textcontext is None")
        W32, W16 = fp.named, fp.shadow()
        dev = x.device
        HP, WP = H // p, W // p
        L, M = HP * WP, B * HP * WP
        eps = self.norm_epsilon
        sv = {"B": B, "H": H, "W": W, "L": L}

        # conditioning: time_embed(t) [+ mean over tokens of text_context_proj(textcontext)] ------------------------
        temb = temb.reshape(-1).to(F32)
        if temb.numel() == 1 and B > 1:
            temb = temb.expand(B)
        te = "time_embed/layers_"
        four = ops.dit_fourier(temb, self._fourier_freqs(dev))
        u1 = ops.linear_fwd(four, W16[te + "1/DenseGeneral_0/kernel"], bias=W32[te + "1/DenseGeneral_0/bias"])
        h1 = ops.bias_act(u1, None, ACT_GELU_TANH)
        u2 = ops.linear_fwd(h1, W16[te + "1/DenseGeneral_1/kernel"], bias=W32[te + "1/DenseGeneral_1/bias"])
        h2 = ops.bias_act(u2, None, ACT_GELU_TANH)
        ctxm16 = None
        if textcontext is None:
            cond = ops.linear_fwd(h2, W16[te + "2/kernel"], bias=W32[te + "2/bias"], out_dtype=F32)
        else:
            tc = textcontext
            if tc.shape[0] == 1 and B > 1:
                tc = tc.expand(B, -1, -1)
            tc = tc.contiguous()
            tc16 = tc if tc.dtype == BF16 else ops.cast_f32_bf16(tc.to(F32).contiguous())
            # mean_t(ctx W + b) = mean_t(ctx) W + b: the token mean first, then one [B, Dc] x [Dc, F] product added
            # onto the time embedding's last dense layer (both biases in that layer's epilogue)
            ctxm16 = ops.cast_f32_bf16(ops.dit_token_mean(tc16))
            cond = ops.linear_fwd(h2, W16[te + "2/kernel"], bias=W32[te + "2/bias"] + W32["text_context_proj/bias"],
                                  out_dtype=F32)
            ops.gemm(ops.GEMM_KMN, ctxm16, W16["text_context_proj/kernel"], cond, B, F, ctxm16.shape[1],
                     ctxm16.shape[1], F, F, atomic=True)
        cond16 = ops.cast_f32_bf16(cond)
        sv["temb"] = (four, u1, h1, u2, h2, ctxm16, cond16)

        # patch embedding + the 2-D sin-cos table (the GEMM's residual, shared by every image) ---------------------
        K = p * p * C
        Kp = _round_up(K, 32)
        rows = ops.dit_patchify(x, p, Kp)
        wpe = torch.nn.functional.pad(W16["patch_embed/Conv_0/kernel"].reshape(K, F), (0, 0, 0, Kp - K))
        tok = torch.empty((M, F), dtype=BF16, device=dev)
        ops.gemm(ops.GEMM_KMN, rows, wpe, tok, L, F, Kp, Kp, F, F, batch1=B, a_s=(L * Kp, 0), d_s=(L * F, 0),
                 bias=W32["patch_embed/Conv_0/bias"], res=self._const("pos", dev, HP, WP), r_ld=F, r_s=(0, 0))
        sv["patch_rows"] = rows

        blocks = []
        for i in range(self.num_layers):
            tok, rec = self._block_fwd(f"dit_block_{i}", tok, cond16, W32, W16, B, L)
            blocks.append(rec)
        sv["blocks"] = blocks

        # final_norm -> final_proj (the first p*p*out columns, zero-padded to the GEMM's multiple of 32) -> unpatchify
        xf, mf, rf = ops.dit_adaln_fwd(tok, L, gamma=W32["final_norm/scale"], beta=W32["final_norm/bias"], eps=eps)
        P_ = p * p * self.output_channels
        Np = _round_up(P_, 32)
        wfp = torch.nn.functional.pad(W16["final_proj/kernel"][:, :P_], (0, Np - P_)).contiguous()
        bfp = torch.nn.functional.pad(W32["final_proj/bias"][:P_], (0, Np - P_)).contiguous()
        yf = ops.linear_fwd(xf, wfp, bias=bfp, out_dtype=F32)
        out = ops.dit_unpatchify(yf, B, H, W, self.output_channels, p)
        if not save:
            return out, None
        sv.update(final=(tok, mf, rf, xf, wfp))
        return out, sv

    def _qkv_weights(self, n, W32, W16):
        """The fused QKV kernel [F, 3*heads*dp] bf16 and bias f32, heads zero-padded to the attention width dp."""
        F, heads = self.emb_features, self.num_heads
        d = F // heads
        dp = _attn_width(d)
        pad = Unet._pad_heads
        w = torch.cat([pad(W16[f"{n}/attention/{m}/kernel"], 2, d, dp).reshape(F, heads * dp)
                       for m in ("to_q", "to_k", "to_v")], 1).contiguous()
        b = torch.cat([pad(W32[f"{n}/attention/{m}/bias"], 1, d, dp).reshape(heads * dp)
                       for m in ("to_q", "to_k", "to_v")]).contiguous()
        wo = pad(W16[f"{n}/attention/to_out_0/kernel"], 1, d, dp).reshape(heads * dp, F).contiguous()
        return w, b, wo

    def _block_fwd(self, n, x, cond16, W32, W16, B, L):
        """DiTBlock (simple_dit.py:62-92): ada chunks scale_mlp 0, shift_mlp 1, gate_mlp 2, scale_attn 3, shift_attn 4,
        gate_attn 5 (F columns each)."""
        F, heads, eps = self.emb_features, self.num_heads, self.norm_epsilon
        d = F // heads
        dp = _attn_width(d)
        HD = heads * dp
        M = x.shape[0]
        ada = ops.linear_fwd(cond16, W16[f"{n}/ada_params_module/ada_proj/kernel"],
                             bias=W32[f"{n}/ada_params_module/ada_proj/bias"], out_dtype=F32)
        n1, m1, r1 = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps)
        wqkv, bqkv, wo = self._qkv_weights(n, W32, W16)
        qkv = ops.linear_fwd(n1, wqkv, bias=bqkv)
        del n1
        ops.dit_rope(qkv, L, heads, d, dp, nmat=2, mat_off=HD)
        q3 = qkv.view(B, L, 3 * HD)
        q, k, v = q3[..., :HD], q3[..., HD:2 * HD], q3[..., 2 * HD:]
        o, lse = ops.attention_fwd(q, k, v, heads, dp, d ** -0.5)
        ya = ops.linear_fwd(o.view(M, HD), wo, bias=W32[f"{n}/attention/to_out_0/bias"])
        x1 = ops.dit_gate_fwd(x, ya, L, ada[:, 5 * F:])
        n2, m2, r2 = ops.dit_adaln_fwd(x1, L, ada, 0, F, eps=eps)
        u = ops.linear_fwd(n2, W16[f"{n}/mlp/layers_0/kernel"], bias=W32[f"{n}/mlp/layers_0/bias"])
        del n2
        g = ops.bias_act(u, None, ACT_GELU_TANH)
        ym = ops.linear_fwd(g, W16[f"{n}/mlp/layers_2/kernel"], bias=W32[f"{n}/mlp/layers_2/bias"])
        del g
        x2 = ops.dit_gate_fwd(x1, ym, L, ada[:, 2 * F:3 * F])
        return x2, (n, x, ada, m1, r1, qkv, o, lse, ya, x1, m2, r2, u, ym, (wqkv, wo))

    # ------------------------------------------------------------------ backward program
    def backward(self, fp: FlatParams, saved: dict, dF: torch.Tensor, grads: FlatParams, on_ready=None):
        """Accumulates d(loss)/d(params) into `grads` (f32, zeroed by the caller) given dF = dL/dF (B, H, W, out) f32.
        `on_ready(lo, streams)`: every gradient at flat offset >= lo is final once the queued work has run (the layout
        follows the forward order; the backward walks it from the end)."""
        W32, W16, Gd = fp.named, fp.shadow(), grads.named
        B, H, W, L = saved["B"], saved["H"], saved["W"], saved["L"]
        F, p, eps = self.emb_features, self.patch_size, self.norm_epsilon
        dev = dF.device
        lay = fp.layout
        stream = [torch.cuda.current_stream()]

        # final_proj + unpatchify: the gradient rows are the patchified dF (zero columns past p*p*out)
        tok, mf, rf, xf, wfp = saved["final"]
        P_ = p * p * self.output_channels
        Np = wfp.shape[1]
        dY = ops.dit_patchify(dF.contiguous(), p, Np)
        gw = torch.zeros((F, Np), dtype=F32, device=dev)
        ops.gemm(GEMM_MNMN, xf, dY, gw, F, Np, xf.shape[0], F, Np, Np, atomic=True, reduce_batch=True)
        Gd["final_proj/kernel"][:, :P_].add_(gw[:, :P_])
        gb = torch.zeros(Np, dtype=F32, device=dev)
        ops.colsum_rows(dY, gb)
        Gd["final_proj/bias"][:P_].add_(gb[:P_])
        dxf = _dense_dgrad(dY, wfp)
        dx = ops.dit_adaln_bwd(tok, dxf, L, mf, rf, Gd["final_norm/scale"], Gd["final_norm/bias"],
                               gamma=W32["final_norm/scale"], reduce_samples=True, accumulate=True)
        if on_ready is not None:
            on_ready(lay.table["final_norm/scale"][0], stream)

        dcond = torch.zeros((B, F), dtype=F32, device=dev)
        four, u1, h1, u2, h2, ctxm16, cond16 = saved["temb"]
        for rec in reversed(saved["blocks"]):
            dx = self._block_bwd(rec, dx, cond16, dcond, W32, W16, Gd, B, L)
            if on_ready is not None:
                on_ready(lay.table[f"{rec[0]}/ada_params_module/ada_proj/kernel"][0], stream)

        # patch embedding: weight and bias gradients only (the image needs none)
        rows = saved["patch_rows"]
        K, Kp = p * p * 3, rows.shape[1]
        gpe = torch.zeros((Kp, F), dtype=F32, device=dev)
        ops.gemm(GEMM_MNMN, rows, dx, gpe, Kp, F, rows.shape[0], Kp, F, F, atomic=True, reduce_batch=True)
        Gd["patch_embed/Conv_0/kernel"].view(K, F).add_(gpe[:K])
        ops.colsum_rows(dx, Gd["patch_embed/Conv_0/bias"])

        # conditioning: Dense(F) <- TimeProjection <- Fourier, and text_context_proj
        te = "time_embed/layers_"
        dc16 = ops.cast_f32_bf16(dcond)
        _dense_wgrad(Gd[te + "2/kernel"], h2, dc16)
        ops.colsum_rows(dc16, Gd[te + "2/bias"])
        if ctxm16 is not None:
            _dense_wgrad(Gd["text_context_proj/kernel"], ctxm16, dc16)
            Gd["text_context_proj/bias"].copy_(Gd[te + "2/bias"])
        dh2 = _dense_dgrad(dc16, W16[te + "2/kernel"])
        du2 = ops.bias_act_bwd(u2, None, ACT_GELU_TANH, dh2)
        _dense_wgrad(Gd[te + "1/DenseGeneral_1/kernel"], h1, du2)
        ops.colsum_rows(du2, Gd[te + "1/DenseGeneral_1/bias"])
        dh1 = _dense_dgrad(du2, W16[te + "1/DenseGeneral_1/kernel"])
        du1 = ops.bias_act_bwd(u1, None, ACT_GELU_TANH, dh1)
        _dense_wgrad(Gd[te + "1/DenseGeneral_0/kernel"], four, du1)
        ops.colsum_rows(du1, Gd[te + "1/DenseGeneral_0/bias"])
        if on_ready is not None:
            on_ready(0, stream)

    def _block_bwd(self, rec, dx2, cond16, dcond, W32, W16, Gd, B, L):
        n, x, ada, m1, r1, qkv, o, lse, ya, x1, m2, r2, u, ym, (wqkv, wo) = rec
        F, heads, eps = self.emb_features, self.num_heads, self.norm_epsilon
        d = F // heads
        dp = _attn_width(d)
        HD = heads * dp
        M = x.shape[0]
        dada = torch.empty((B, 6 * F), dtype=F32, device=x.device)
        # MLP branch: x2 = x1 + gate_mlp * (gelu(n2 W0 + b0) W2 + b2)
        dym = ops.dit_gate_bwd(dx2, ym, L, ada[:, 2 * F:3 * F], dada[:, 2 * F:3 * F])
        g = ops.bias_act(u, None, ACT_GELU_TANH)
        _dense_wgrad(Gd[f"{n}/mlp/layers_2/kernel"], g, dym)
        ops.colsum_rows(dym, Gd[f"{n}/mlp/layers_2/bias"])
        del g
        dg = _dense_dgrad(dym, W16[f"{n}/mlp/layers_2/kernel"])
        du = ops.bias_act_bwd(u, None, ACT_GELU_TANH, dg)
        del dg
        n2, _, _ = ops.dit_adaln_fwd(x1, L, ada, 0, F, eps=eps, stats=False)
        _dense_wgrad(Gd[f"{n}/mlp/layers_0/kernel"], n2, du)
        ops.colsum_rows(du, Gd[f"{n}/mlp/layers_0/bias"])
        del n2
        dn2 = _dense_dgrad(du, W16[f"{n}/mlp/layers_0/kernel"])
        del du
        dx1 = ops.dit_adaln_bwd(x1, dn2, L, m2, r2, dada[:, 0:F], dada[:, F:2 * F], ada=ada, scale_off=0, addend=dx2)
        del dn2
        # attention branch: x1 = x + gate_attn * (attn(rope(n1 Wq + bq), rope(n1 Wk + bk), n1 Wv + bv) Wo + bo)
        dya = ops.dit_gate_bwd(dx1, ya, L, ada[:, 5 * F:], dada[:, 5 * F:])
        _dense_wgrad(Gd[f"{n}/attention/to_out_0/kernel"], o.view(M, HD), dya, 1, dp)
        ops.colsum_rows(dya, Gd[f"{n}/attention/to_out_0/bias"])
        do = _dense_dgrad(dya, wo).view(B, L, HD)
        del dya
        q3 = qkv.view(B, L, 3 * HD)
        dq, dk, dv = ops.attention_bwd(q3[..., :HD], q3[..., HD:2 * HD], q3[..., 2 * HD:], o, lse, do, heads, dp,
                                       d ** -0.5)
        del do
        dq2, dk2, dv2 = dq.view(M, HD), dk.view(M, HD), dv.view(M, HD)
        ops.dit_rope(dq2, L, heads, d, dp, inverse=True)
        ops.dit_rope(dk2, L, heads, d, dp, inverse=True)
        n1, _, _ = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps, stats=False)
        bt = torch.empty(HD, dtype=F32, device=x.device)
        dn1 = None
        for j, (m, dm) in enumerate((("to_q", dq2), ("to_k", dk2), ("to_v", dv2))):
            _dense_wgrad(Gd[f"{n}/attention/{m}/kernel"], n1, dm, 2, dp)
            ops.colsum_rows(dm, bt)
            Gd[f"{n}/attention/{m}/bias"].add_(bt.view(heads, dp)[:, :d])
            wj = wqkv[:, j * HD:(j + 1) * HD]
            # dn1 = sum_j dm_j Wj^T: [rows, HD] x [F, HD]^T (the weight slice is row-strided in the fused kernel)
            out = torch.empty((M, F), dtype=BF16, device=x.device) if dn1 is None else dn1
            ops.gemm(GEMM_KK, dm, wj, out, M, F, HD, HD, wqkv.stride(0), F, res=dn1, r_ld=F if dn1 is not None else 0)
            dn1 = out
        del n1, dq, dk, dv
        dx0 = ops.dit_adaln_bwd(x, dn1, L, m1, r1, dada[:, 3 * F:4 * F], dada[:, 4 * F:5 * F], ada=ada,
                                scale_off=3 * F, addend=dx1)
        # ada_proj: ada = cond W + b
        dada16 = ops.cast_f32_bf16(dada)
        _dense_wgrad(Gd[f"{n}/ada_params_module/ada_proj/kernel"], cond16, dada16)
        ops.colsum_rows(dada16, Gd[f"{n}/ada_params_module/ada_proj/bias"])
        ops.gemm(GEMM_KK, dada16, W16[f"{n}/ada_params_module/ada_proj/kernel"], dcond, B, F, 6 * F, 6 * F, 6 * F, F,
                 atomic=True)
        return dx0
