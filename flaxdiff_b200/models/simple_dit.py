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


def _lecun_normal(t: torch.Tensor, fan_in: int, gen: torch.Generator) -> None:
    """flax's lecun_normal: a normal truncated at two standard deviations, rescaled to variance 1 / fan_in."""
    std = math.sqrt(1.0 / fan_in) / 0.87962566103423978
    torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)


class SimpleDiT:
    # the text projection's module name (mean-pooled over tokens; SimpleUDiT names it text_proj)
    _text_proj = "text_context_proj"

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
            raise FdxError(f"{type(self).__name__}: use_flash_attention=True has no counterpart here; the fused attention kernel "
                           "is always used")
        if dtype is not None and dtype != torch.bfloat16:
            raise FdxError(f"{type(self).__name__}: dtype={dtype} is not supported: the engine computes in bf16 with f32 "
                           "accumulation (pass dtype=None or torch.bfloat16)")
        F, h = emb_features, num_heads
        if h <= 0 or F % h != 0:
            raise FdxError(f"{type(self).__name__}: emb_features={F} is not a multiple of num_heads={h}")
        d = F // h
        if d % 2:
            raise FdxError(f"{type(self).__name__}: head width {d} is odd (RoPE rotates channel pairs)")
        if d > 256:
            raise FdxError(f"{type(self).__name__}: head width {d} > 256 is not supported by the fused attention")
        if F % 64 or F > 1536:
            raise FdxError(f"{type(self).__name__}: emb_features={F} must be a multiple of 64, at most 1536")
        self._layouts: Dict[Optional[int], ParamLayout] = {}
        self._consts: Dict[tuple, torch.Tensor] = {}

    # ------------------------------------------------------------------ structure
    def param_specs(self):
        F, p, E = self.emb_features, self.patch_size, self.emb_features * self.mlp_ratio
        nout = p * p * self.output_channels * (2 if self.learn_sigma else 1)
        specs = self._embed_specs() + [
                 ("time_embed/layers_1/DenseGeneral_0/kernel", (F, E)), ("time_embed/layers_1/DenseGeneral_0/bias", (E,)),
                 ("time_embed/layers_1/DenseGeneral_1/kernel", (E, E)), ("time_embed/layers_1/DenseGeneral_1/bias", (E,)),
                 ("time_embed/layers_2/kernel", (E, F)), ("time_embed/layers_2/bias", (F,))]
        if self.context_dim:
            specs += [(f"{self._text_proj}/kernel", (self.context_dim, F)), (f"{self._text_proj}/bias", (F,))]
        for n, _, _ in self._blocks():
            specs += self._block_specs(n)
        specs += [("final_norm/scale", (F,)), ("final_norm/bias", (F,)),
                  ("final_proj/kernel", (F, nout)), ("final_proj/bias", (nout,))]
        return specs

    def _embed_name(self) -> str:
        """The patch embedding's dense layer: PatchEmbedding's p x p stride-p conv."""
        return "patch_embed/Conv_0"

    def _embed_specs(self):
        p, F = self.patch_size, self.emb_features
        return [("patch_embed/Conv_0/kernel", (p, p, 3, F)), ("patch_embed/Conv_0/bias", (F,))]

    def _block_specs(self, n):
        """DiTBlock `n`'s parameters: ada_proj, the attention's q / k / v / out DenseGenerals and the MLP."""
        F, h = self._widths(n)
        E = F * self.mlp_ratio
        d = F // h
        specs = [(f"{n}/ada_params_module/ada_proj/kernel", (F, 6 * F)),
                 (f"{n}/ada_params_module/ada_proj/bias", (6 * F,))]
        for m in ("to_q", "to_k", "to_v"):
            specs += [(f"{n}/attention/{m}/kernel", (F, h, d)), (f"{n}/attention/{m}/bias", (h, d))]
        specs += [(f"{n}/attention/to_out_0/kernel", (h, d, F)), (f"{n}/attention/to_out_0/bias", (F,)),
                  (f"{n}/mlp/layers_0/kernel", (F, E)), (f"{n}/mlp/layers_0/bias", (E,)),
                  (f"{n}/mlp/layers_2/kernel", (E, F)), (f"{n}/mlp/layers_2/bias", (F,))]
        return specs

    def _widths(self, n: str):
        """(width, heads) of block n."""
        return self.emb_features, self.num_heads

    def _blocks(self):
        """(name, forward, backward) of every block, in order."""
        return [(f"dit_block_{i}", self._block_fwd, self._block_bwd) for i in range(self.num_layers)]

    def _scan_indices(self, HP: int, WP: int):
        """The patch order as row-major indices (token i is patch idx[i]), or None for raster order."""
        return None

    def _order(self, HP: int, WP: int, device):
        """(index table, inverse) as int32 device tensors, or None for raster order."""
        idx = self._scan_indices(HP, WP)
        if idx is None:
            return None
        key = ("order", str(device), HP, WP)
        if key not in self._consts:
            import numpy as np
            inv = np.empty_like(idx)
            inv[idx] = np.arange(len(idx))
            self._consts[key] = tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)
                                      for a in (idx, inv))
        return self._consts[key]

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
            self._init_leaf(name, t, gen)
        return fp

    def _init_leaf(self, name: str, t: torch.Tensor, gen: torch.Generator) -> None:
        """Fills one zero-initialised leaf (biases stay zero)."""
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
            _lecun_normal(t, fan_in, gen)

    def _const(self, kind: str, device, *shape) -> torch.Tensor:
        key = (kind, str(device)) + shape
        if key not in self._consts:
            if kind == "freqs":   # FourierEmbedding.freqs: normal(PRNGKey(42), (F//2,)) * 16 (common.py:101-102)
                f = utils.normal(utils.PRNGKey(42), self.emb_features // 2) * 16.0
                self._consts[key] = torch.from_numpy(f.astype("float32")).to(device)
            else:                 # the 2-D sin-cos position table, bf16 [L, F], in the patch order
                tab = sincos_2d_table(self.emb_features, *shape)
                idx = self._scan_indices(*shape)
                if idx is not None:
                    tab = tab[idx]
                self._consts[key] = torch.from_numpy(tab).to(device, BF16)
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
        p = self.patch_size
        if H % p or W % p:
            raise FdxError(f"{type(self).__name__}: image {H}x{W} is not divisible by the patch size {p}")
        if textcontext is not None and int(textcontext.shape[-1]) != (self.context_dim or -1):
            raise FdxError(f"{type(self).__name__}: textcontext width {tuple(textcontext.shape)} does not match the parameters "
                           f"(context_dim={self.context_dim}); build / init the model with it")
        if textcontext is None and self.context_dim is not None:
            raise FdxError(f"{type(self).__name__}: parameters were built with {self._text_proj} but textcontext is None")
        W32, W16 = fp.named, fp.shadow()
        dev = x.device
        HP, WP = H // p, W // p
        L = HP * WP
        sv = {"B": B, "H": H, "W": W, "L": L}

        # conditioning: time_embed(t) [+ mean over tokens of text_context_proj(textcontext)] ------------------------
        cond16, sv["temb"] = self._cond_fwd(W32, W16, temb, textcontext, B, dev)
        sv["cond16"] = cond16

        # patch embedding [+ the 2-D sin-cos table, the GEMM's residual shared by every image] ----------------------
        order = self._order(HP, WP, dev)
        tok, sv["patch_rows"] = self._embed_fwd(x, W32, W16, HP, WP, order)
        sv["order"] = order

        tok, sv["blocks"] = self._trunk_fwd(tok, cond16, W32, W16, B, L)

        out, sv["final"] = self._final_fwd(tok, W32, W16, B, H, W, L, order)
        if not save:
            return out, None
        return out, sv

    def _trunk_fwd(self, tok, cond16, W32, W16, B: int, L: int):
        """The blocks between the patch embedding and final_norm -> (tokens, tape)."""
        blocks = []
        for n, fwd, _ in self._blocks():
            tok, rec = fwd(n, tok, cond16, W32, W16, B, L)
            blocks.append(rec)
        return tok, blocks

    def _embed_fwd(self, x, W32, W16, HP: int, WP: int, order):
        """Patch rows (in the patch order) x the patch embedding [+ the position table] -> (tokens bf16, patch rows)."""
        B, C = x.shape[0], x.shape[3]
        p = self.patch_size
        emb = self._embed_name()
        F = W32[emb + "/bias"].numel()
        L = HP * WP
        K = p * p * C
        Kp = _round_up(K, 32)
        rows = ops.dit_patchify(x, p, Kp)
        if order is not None:
            rows = ops.permute_rows(rows, order[0])
        wpe = torch.nn.functional.pad(W16[emb + "/kernel"].reshape(K, F), (0, 0, 0, Kp - K))
        tok = torch.empty((B * L, F), dtype=BF16, device=x.device)
        pos = self._pos_table(x.device, HP, WP)
        ops.gemm(ops.GEMM_KMN, rows, wpe, tok, L, F, Kp, Kp, F, F, batch1=B, a_s=(L * Kp, 0), d_s=(L * F, 0),
                 bias=W32[emb + "/bias"], res=pos, r_ld=F if pos is not None else 0, r_s=(0, 0))
        return tok, rows

    def _embed_bwd(self, rows, dx, Gd) -> None:
        """The patch embedding's weight and bias gradients (the image needs none)."""
        p, F = self.patch_size, dx.shape[1]
        K, Kp = p * p * 3, rows.shape[1]
        gpe = torch.zeros((Kp, F), dtype=F32, device=dx.device)
        ops.gemm(GEMM_MNMN, rows, dx, gpe, Kp, F, rows.shape[0], Kp, F, F, atomic=True, reduce_batch=True)
        emb = self._embed_name()
        Gd[emb + "/kernel"].view(K, F).add_(gpe[:K])
        ops.colsum_rows(dx, Gd[emb + "/bias"])

    def _final_fwd(self, tok, W32, W16, B, H, W, L, order):
        """final_norm -> final_proj (the first p*p*out columns, zero-padded to the GEMM's multiple of 32) ->
        unpatchify -> (output f32 (B, H, W, out), tape)."""
        p = self.patch_size
        xf, mf, rf = ops.dit_adaln_fwd(tok, L, gamma=W32["final_norm/scale"], beta=W32["final_norm/bias"],
                                       eps=self.norm_epsilon)
        P_ = p * p * self.output_channels
        Np = _round_up(P_, 32)
        wfp = torch.nn.functional.pad(W16["final_proj/kernel"][:, :P_], (0, Np - P_)).contiguous()
        bfp = torch.nn.functional.pad(W32["final_proj/bias"][:P_], (0, Np - P_)).contiguous()
        yf = ops.linear_fwd(xf, wfp, bias=bfp, out_dtype=F32)
        if order is not None:
            yf = ops.permute_rows(yf, order[1])
        return ops.dit_unpatchify(yf, B, H, W, self.output_channels, p), (tok, mf, rf, xf, wfp)

    def _final_bwd(self, tape, dF, order, W32, Gd, L):
        """Backward of _final_fwd -> d(tokens); the gradient rows are the patchified dF (zero columns past p*p*out)."""
        tok, mf, rf, xf, wfp = tape
        p, F = self.patch_size, tok.shape[1]
        P_ = p * p * self.output_channels
        Np = wfp.shape[1]
        dY = ops.dit_patchify(dF.contiguous(), p, Np)
        if order is not None:
            dY = ops.permute_rows(dY, order[0])
        gw = torch.zeros((F, Np), dtype=F32, device=dF.device)
        ops.gemm(GEMM_MNMN, xf, dY, gw, F, Np, xf.shape[0], F, Np, Np, atomic=True, reduce_batch=True)
        Gd["final_proj/kernel"][:, :P_].add_(gw[:, :P_])
        gb = torch.zeros(Np, dtype=F32, device=dF.device)
        ops.colsum_rows(dY, gb)
        Gd["final_proj/bias"][:P_].add_(gb[:P_])
        dxf = _dense_dgrad(dY, wfp)
        return ops.dit_adaln_bwd(tok, dxf, L, mf, rf, Gd["final_norm/scale"], Gd["final_norm/bias"],
                                 gamma=W32["final_norm/scale"], reduce_samples=True, accumulate=True)

    def _pos_table(self, device, HP: int, WP: int):
        """The position table added to the patch embedding (bf16 [L, F], in the patch order), or None."""
        return self._const("pos", device, HP, WP)

    def _time_mlp_fwd(self, base: str, temb: torch.Tensor, B: int, freqs, W32, W16):
        """FourierEmbedding -> TimeProjection of nn.Sequential `base` -> (h2 bf16 [B, 4F], tape)."""
        temb = temb.reshape(-1).to(F32)
        if temb.numel() == 1 and B > 1:
            temb = temb.expand(B)
        te = base + "/layers_"
        four = ops.dit_fourier(temb, freqs)
        u1 = ops.linear_fwd(four, W16[te + "1/DenseGeneral_0/kernel"], bias=W32[te + "1/DenseGeneral_0/bias"])
        h1 = ops.bias_act(u1, None, ACT_GELU_TANH)
        u2 = ops.linear_fwd(h1, W16[te + "1/DenseGeneral_1/kernel"], bias=W32[te + "1/DenseGeneral_1/bias"])
        h2 = ops.bias_act(u2, None, ACT_GELU_TANH)
        return h2, (four, u1, h1, u2)

    def _time_mlp_bwd(self, base: str, tape, dh2: torch.Tensor, W16, Gd) -> None:
        four, u1, h1, u2 = tape
        te = base + "/layers_"
        du2 = ops.bias_act_bwd(u2, None, ACT_GELU_TANH, dh2)
        _dense_wgrad(Gd[te + "1/DenseGeneral_1/kernel"], h1, du2)
        ops.colsum_rows(du2, Gd[te + "1/DenseGeneral_1/bias"])
        dh1 = _dense_dgrad(du2, W16[te + "1/DenseGeneral_1/kernel"])
        du1 = ops.bias_act_bwd(u1, None, ACT_GELU_TANH, dh1)
        _dense_wgrad(Gd[te + "1/DenseGeneral_0/kernel"], four, du1)
        ops.colsum_rows(du1, Gd[te + "1/DenseGeneral_0/bias"])

    @staticmethod
    def _text_rows(textcontext: torch.Tensor, B: int) -> torch.Tensor:
        """textcontext as contiguous bf16 with the batch broadcast to B."""
        tc = textcontext
        if tc.shape[0] == 1 and B > 1:
            tc = tc.expand(B, *tc.shape[1:])
        tc = tc.contiguous()
        return tc if tc.dtype == BF16 else ops.cast_f32_bf16(tc.to(F32).contiguous())

    def _cond_width(self) -> int:
        return self.emb_features

    @staticmethod
    def _pool_text(tc16: torch.Tensor) -> torch.Tensor:
        """The text tokens [B, S, D] mean-pooled to bf16 [B, D]."""
        return ops.cast_f32_bf16(ops.dit_token_mean(tc16))

    def _cond_fwd(self, W32, W16, temb, textcontext, B: int, dev):
        """The blocks' conditioning: bf16 [B, F] = time_embed(t) [+ mean over tokens of text_context_proj(ctx)]."""
        F = self.emb_features
        te = "time_embed/layers_"
        h2, tt = self._time_mlp_fwd("time_embed", temb, B, self._fourier_freqs(dev), W32, W16)
        ctxm16 = None
        if textcontext is None:
            cond = ops.linear_fwd(h2, W16[te + "2/kernel"], bias=W32[te + "2/bias"], out_dtype=F32)
        else:
            tc16 = self._text_rows(textcontext, B)
            # mean_t(ctx W + b) = mean_t(ctx) W + b: the token mean first, then one [B, Dc] x [Dc, F] product added
            # onto the time embedding's last dense layer (both biases in that layer's epilogue)
            ctxm16 = self._pool_text(tc16)
            cond = ops.linear_fwd(h2, W16[te + "2/kernel"], bias=W32[te + "2/bias"] + W32[self._text_proj + "/bias"],
                                  out_dtype=F32)
            ops.gemm(ops.GEMM_KMN, ctxm16, W16[self._text_proj + "/kernel"], cond, B, F, ctxm16.shape[1],
                     ctxm16.shape[1], F, F, atomic=True)
        cond16 = ops.cast_f32_bf16(cond)
        return cond16, (tt, h2, ctxm16)

    def _cond_bwd(self, tape, dcond: torch.Tensor, W16, Gd) -> None:
        """Dense(F) <- TimeProjection <- Fourier, and text_context_proj."""
        tt, h2, ctxm16 = tape
        te = "time_embed/layers_"
        dc16 = ops.cast_f32_bf16(dcond)
        _dense_wgrad(Gd[te + "2/kernel"], h2, dc16)
        ops.colsum_rows(dc16, Gd[te + "2/bias"])
        if ctxm16 is not None:
            _dense_wgrad(Gd[self._text_proj + "/kernel"], ctxm16, dc16)
            Gd[self._text_proj + "/bias"].copy_(Gd[te + "2/bias"])
        dh2 = _dense_dgrad(dc16, W16[te + "2/kernel"])
        self._time_mlp_bwd("time_embed", tt, dh2, W16, Gd)

    def _rope(self) -> bool:
        """RoPE in the attention blocks: off under the Hilbert / zigzag orders, where the reference sets cos = 1,
        sin = 0 (ssm_dit.py:750-759).  The head channels [d, dp) stay zero without it: the QKV kernel and bias are
        zero-padded there."""
        return not (self.use_hilbert or self.use_zigzag)

    def _qkv_weights(self, n, W32, W16):
        """The fused QKV kernel [F, 3*heads*dp] bf16 and bias f32, heads zero-padded to the attention width dp."""
        F, heads = self._widths(n)
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
        F, eps = self.emb_features, self.norm_epsilon
        ada = self._ada_fwd(n, cond16, W32, W16)
        n1, m1, r1 = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps)
        ya, attn = self._attn_fwd(n, n1, W32, W16, B, L)
        del n1
        x1 = ops.dit_gate_fwd(x, ya, L, ada[:, 5 * F:])
        x2, mlp = self._mlp_fwd(n, x1, ada, W32, W16, L)
        return x2, (n, x, ada, m1, r1, attn, ya, x1, mlp)

    def _attn_fwd(self, n, n1, W32, W16, B, L):
        """RoPEAttention of the normalised rows n1 [B*L, F]: one QKV GEMM over the head-padded kernels, RoPE in place,
        the fused attention and to_out_0 -> (y bf16 [B*L, F], tape)."""
        F, heads = self._widths(n)
        d = F // heads
        dp = _attn_width(d)
        HD = heads * dp
        M = n1.shape[0]
        wqkv, bqkv, wo = self._qkv_weights(n, W32, W16)
        qkv = ops.linear_fwd(n1, wqkv, bias=bqkv)
        if self._rope():
            ops.dit_rope(qkv, L, heads, d, dp, nmat=2, mat_off=HD)
        q3 = qkv.view(B, L, 3 * HD)
        q, k, v = q3[..., :HD], q3[..., HD:2 * HD], q3[..., 2 * HD:]
        o, lse = ops.attention_fwd(q, k, v, heads, dp, d ** -0.5)
        ya = ops.linear_fwd(o.view(M, HD), wo, bias=W32[f"{n}/attention/to_out_0/bias"])
        return ya, (qkv, o, lse, wqkv, wo)

    def _ada_fwd(self, n, cond16, W32, W16):
        return ops.linear_fwd(cond16, W16[f"{n}/ada_params_module/ada_proj/kernel"],
                              bias=W32[f"{n}/ada_params_module/ada_proj/bias"], out_dtype=F32)

    def _mlp_fwd(self, n, x1, ada, W32, W16, L):
        """The MLP half of a block: x2 = x1 + gate_mlp * (gelu(adaLN(x1) W0 + b0) W2 + b2)."""
        F = self.emb_features
        n2, m2, r2 = ops.dit_adaln_fwd(x1, L, ada, 0, F, eps=self.norm_epsilon)
        ym, u = self._mlp_core_fwd(n, n2, W32, W16)
        del n2
        x2 = ops.dit_gate_fwd(x1, ym, L, ada[:, 2 * F:3 * F])
        return x2, (m2, r2, u, ym)

    def _mlp_core_fwd(self, n, n2, W32, W16):
        """Dense(4F) -> tanh-gelu -> Dense(F) of the rows n2 -> (y bf16, the pre-activation u)."""
        u = ops.linear_fwd(n2, W16[f"{n}/mlp/layers_0/kernel"], bias=W32[f"{n}/mlp/layers_0/bias"])
        g = ops.bias_act(u, None, ACT_GELU_TANH)
        ym = ops.linear_fwd(g, W16[f"{n}/mlp/layers_2/kernel"], bias=W32[f"{n}/mlp/layers_2/bias"])
        return ym, u

    # ------------------------------------------------------------------ backward program
    def backward(self, fp: FlatParams, saved: dict, dF: torch.Tensor, grads: FlatParams, on_ready=None):
        """Accumulates d(loss)/d(params) into `grads` (f32, zeroed by the caller) given dF = dL/dF (B, H, W, out) f32.
        `on_ready(lo, streams)`: every gradient at flat offset >= lo is final once the queued work has run (the layout
        follows the forward order; the backward walks it from the end)."""
        W32, W16, Gd = fp.named, fp.shadow(), grads.named
        B, H, W, L = saved["B"], saved["H"], saved["W"], saved["L"]
        dev = dF.device
        lay = fp.layout
        stream = [torch.cuda.current_stream()]

        dx = self._final_bwd(saved["final"], dF, saved["order"], W32, Gd, L)
        if on_ready is not None:
            on_ready(lay.table["final_norm/scale"][0], stream)

        dcond = torch.zeros((B, self._cond_width()), dtype=F32, device=dev)
        cond16 = saved["cond16"]

        def ready(leaf: str) -> None:
            if on_ready is not None:
                on_ready(lay.table[leaf][0], stream)
        dx = self._trunk_bwd(saved["blocks"], dx, cond16, dcond, W32, W16, Gd, B, L, ready)

        self._embed_bwd(saved["patch_rows"], dx, Gd)

        self._cond_bwd(saved["temb"], dcond, W16, Gd)
        if on_ready is not None:
            on_ready(0, stream)

    def _trunk_bwd(self, tape, dx, cond16, dcond, W32, W16, Gd, B: int, L: int, ready):
        """Backward of _trunk_fwd -> d(its input tokens); ready(leaf) announces every gradient from `leaf` on final."""
        for (n, _, bwd), rec in zip(reversed(self._blocks()), reversed(tape)):
            dx = bwd(rec, dx, cond16, dcond, W32, W16, Gd, B, L)
            ready(self._ada_leaf(n))
        return dx

    def _ada_leaf(self, n: str) -> str:
        """Block n's first parameter in the layout: its gradients are final once the block's backward has run."""
        return f"{n}/ada_params_module/ada_proj/kernel"

    def _block_bwd(self, rec, dx2, cond16, dcond, W32, W16, Gd, B, L):
        n, x, ada, m1, r1, attn, ya, x1, mlp = rec
        F, eps = self.emb_features, self.norm_epsilon
        dada = torch.empty((B, 6 * F), dtype=F32, device=x.device)
        dx1 = self._mlp_bwd(n, dx2, x1, ada, mlp, dada, W16, Gd, L)
        # attention branch: x1 = x + gate_attn * (attn(rope(n1 Wq + bq), rope(n1 Wk + bk), n1 Wv + bv) Wo + bo)
        dya = ops.dit_gate_bwd(dx1, ya, L, ada[:, 5 * F:], dada[:, 5 * F:])
        dn1 = self._attn_bwd(n, attn, dya, lambda: ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F, eps=eps, stats=False)[0],
                             Gd, B, L)
        dx0 = ops.dit_adaln_bwd(x, dn1, L, m1, r1, dada[:, 3 * F:4 * F], dada[:, 4 * F:5 * F], ada=ada,
                                scale_off=3 * F, addend=dx1)
        self._ada_bwd(n, dada, cond16, dcond, Gd, W16)
        return dx0

    def _attn_bwd(self, n, tape, dya, make_n1, Gd, B, L):
        """Backward of _attn_fwd -> dn1 bf16 [B*L, F]; accumulates the attention's parameter gradients.  make_n1()
        recomputes the attention input once the attention backward has released its buffers."""
        qkv, o, lse, wqkv, wo = tape
        F, heads = self._widths(n)
        d = F // heads
        dp = _attn_width(d)
        HD = heads * dp
        M = dya.shape[0]
        _dense_wgrad(Gd[f"{n}/attention/to_out_0/kernel"], o.view(M, HD), dya, 1, dp)
        ops.colsum_rows(dya, Gd[f"{n}/attention/to_out_0/bias"])
        do = _dense_dgrad(dya, wo).view(B, L, HD)
        del dya
        q3 = qkv.view(B, L, 3 * HD)
        dq, dk, dv = ops.attention_bwd(q3[..., :HD], q3[..., HD:2 * HD], q3[..., 2 * HD:], o, lse, do, heads, dp,
                                       d ** -0.5)
        del do
        dq2, dk2, dv2 = dq.view(M, HD), dk.view(M, HD), dv.view(M, HD)
        if self._rope():
            ops.dit_rope(dq2, L, heads, d, dp, inverse=True)
            ops.dit_rope(dk2, L, heads, d, dp, inverse=True)
        n1 = make_n1()
        bt = torch.empty(HD, dtype=F32, device=n1.device)
        dn1 = None
        for j, (m, dm) in enumerate((("to_q", dq2), ("to_k", dk2), ("to_v", dv2))):
            _dense_wgrad(Gd[f"{n}/attention/{m}/kernel"], n1, dm, 2, dp)
            ops.colsum_rows(dm, bt)
            Gd[f"{n}/attention/{m}/bias"].add_(bt.view(heads, dp)[:, :d])
            wj = wqkv[:, j * HD:(j + 1) * HD]
            # dn1 = sum_j dm_j Wj^T: [rows, HD] x [F, HD]^T (the weight slice is row-strided in the fused kernel)
            out = torch.empty((M, F), dtype=BF16, device=n1.device) if dn1 is None else dn1
            ops.gemm(GEMM_KK, dm, wj, out, M, F, HD, HD, wqkv.stride(0), F, res=dn1, r_ld=F if dn1 is not None else 0)
            dn1 = out
        return dn1

    def _mlp_bwd(self, n, dx2, x1, ada, mlp, dada, W16, Gd, L):
        """Backward of _mlp_fwd: -> dx1; writes the gate_mlp / scale_mlp / shift_mlp chunks of dada."""
        m2, r2, u, ym = mlp
        F, eps = self.emb_features, self.norm_epsilon
        dym = ops.dit_gate_bwd(dx2, ym, L, ada[:, 2 * F:3 * F], dada[:, 2 * F:3 * F])
        dn2 = self._mlp_core_bwd(n, u, dym, lambda: ops.dit_adaln_fwd(x1, L, ada, 0, F, eps=eps, stats=False)[0],
                                 W16, Gd)
        return ops.dit_adaln_bwd(x1, dn2, L, m2, r2, dada[:, 0:F], dada[:, F:2 * F], ada=ada, scale_off=0, addend=dx2)

    def _mlp_core_bwd(self, n, u, dym, make_n2, W16, Gd):
        """Backward of _mlp_core_fwd -> dn2; make_n2() recomputes its input when the weight gradient needs it."""
        g = ops.bias_act(u, None, ACT_GELU_TANH)
        _dense_wgrad(Gd[f"{n}/mlp/layers_2/kernel"], g, dym)
        ops.colsum_rows(dym, Gd[f"{n}/mlp/layers_2/bias"])
        del g
        dg = _dense_dgrad(dym, W16[f"{n}/mlp/layers_2/kernel"])
        du = ops.bias_act_bwd(u, None, ACT_GELU_TANH, dg)
        del dg
        n2 = make_n2()
        _dense_wgrad(Gd[f"{n}/mlp/layers_0/kernel"], n2, du)
        ops.colsum_rows(du, Gd[f"{n}/mlp/layers_0/bias"])
        del n2
        dn2 = _dense_dgrad(du, W16[f"{n}/mlp/layers_0/kernel"])
        del du
        return dn2

    def _ada_bwd(self, n, dada, cond16, dcond, Gd, W16):
        """ada = cond W + b: the kernel and bias gradients, and dcond += dada W^T."""
        F = self.emb_features
        dada16 = ops.cast_f32_bf16(dada)
        _dense_wgrad(Gd[f"{n}/ada_params_module/ada_proj/kernel"], cond16, dada16)
        ops.colsum_rows(dada16, Gd[f"{n}/ada_params_module/ada_proj/bias"])
        ops.gemm(GEMM_KK, dada16, W16[f"{n}/ada_params_module/ada_proj/kernel"], dcond, dada.shape[0], F, 6 * F,
                 6 * F, 6 * F, F, atomic=True)
