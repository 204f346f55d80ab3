"""`SimpleMMDiT` - the reference's text-conditioned multi-modal DiT (flaxdiff/models/simple_mmdit.py:17-331) on the
engine, with the same program interface as `SimpleDiT` and `Unet` (init / apply / forward / backward / layout), so
GeneralDiffusionTrainer, the samplers and the checkpoint writer take it unchanged.

    model = SimpleMMDiT(patch_size=2, emb_features=768, num_layers=12, num_heads=12, context_dim=768)
    params = model.init(key, textcontext=ctx)             # {'params': tree}, flax names
    y = model.apply(params, x, temb, ctx)                 # (B, H, W, 3) f32; ctx [B, S, D] or [B, D]

What differs from SimpleDiT, and how it runs:
  * The block (MMDiTBlock, :94-158) is a parallel block.  ONE LayerNorm of the block input is modulated twice -
    x_attn with (scale_attn, shift_attn), x_mlp with (clip(scale_mlp), clip(shift_mlp)), clipped to [-10, 10] - and
    both branches are added onto the same residual: x + gate_attn * attn(x_attn) + gate_mlp * mlp(x_mlp).
    fdx_mmdit.cu fuses exactly that: one pass over x writes both modulated rows (fdx_mmdit_adaln_fwd), one pass adds
    both gated branches (fdx_mmdit_gate_fwd), and their backwards.  The attention and MLP GEMM programs are
    SimpleDiT's.
  * The clip's backward passes the gradient inside (-10, 10), zero outside and one half at exactly -10 or 10: that
    is the derivative of jnp.clip = min(max(v, lo), hi) under JAX's autodiff, whose lax.max / lax.min split the
    cotangent evenly between equal operands.  The one half follows from that rule; it has not been checked against a
    running JAX.
  * Conditioning (MMAdaLNZero, :17-90): each block's ada parameters are ada_t_proj(t_emb) + ada_text_proj(text_emb),
    two zero-initialised Dense(6F) layers.  text_emb = text_context_proj(textcontext) mean-pooled over tokens; as both
    are linear, the token mean runs first (fdx_dit_token_mean) and the products are [B, .] GEMMs.  A block's ada is
    one product of [t_emb, text_emb] [B, 2F] with the stacked [ada_t_proj; ada_text_proj] kernels [2F, 6F] - adjacent
    in the flat parameter buffer, so the stack is a view - plus the two biases.
  * No sin-cos position table: positions come only from RoPE, which stays on under use_hilbert (positions are then
    indices along the Hilbert sequence).  Under use_hilbert, `hilbert_projection` replaces `patch_embed` (which then
    has no parameters) and the patch rows are permuted on the device, as in HybridSSMAttentionDiT.
  * textcontext is required (the reference asserts): None raises FdxError.

`HierarchicalMMDiT` (below) is the reference's U-shaped multi-resolution variant built from the same block.

Refused with FdxError, as SimpleDiT refuses them: use_flash_attention=True, a dtype other than bf16, emb_features not a
multiple of num_heads or of 64 or above 1536, odd head widths (the reference itself fails there: its RoPE cos table is
one wider than the head) and heads wider than 256, images not divisible by the patch size.  dropout_rate, norm_groups,
activation and force_fp32_for_softmax are accepted and ignored, as in the reference.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import ops
from .._lib import GEMM_KK, FdxError
from .simple_dit import F32, SimpleDiT
from .simple_unet import _dense_dgrad, _dense_wgrad
from .ssm_dit import hilbert_indices


class SimpleMMDiT(SimpleDiT):
    def __init__(self, output_channels: int = 3, patch_size: int = 16, emb_features: int = 768, num_layers: int = 12,
                 num_heads: int = 12, mlp_ratio: int = 4, dropout_rate: float = 0.0, dtype=None, precision=None,
                 use_flash_attention: bool = False, force_fp32_for_softmax: bool = True, norm_epsilon: float = 1e-5,
                 learn_sigma: bool = False, use_hilbert: bool = False, norm_groups: int = 0, activation=None,
                 context_dim: Optional[int] = None):
        super().__init__(output_channels=output_channels, patch_size=patch_size, emb_features=emb_features,
                         num_layers=num_layers, num_heads=num_heads, mlp_ratio=mlp_ratio, dropout_rate=dropout_rate,
                         dtype=dtype, precision=precision, use_flash_attention=use_flash_attention,
                         force_fp32_for_softmax=force_fp32_for_softmax, norm_epsilon=norm_epsilon,
                         learn_sigma=learn_sigma, norm_groups=norm_groups, activation=activation,
                         context_dim=context_dim)
        self.use_hilbert = use_hilbert

    # ------------------------------------------------------------------ structure
    def config(self) -> dict:
        """The constructor arguments (a config round trip: SimpleMMDiT(**model.config()))."""
        keys = ("output_channels", "patch_size", "emb_features", "num_layers", "num_heads", "mlp_ratio",
                "dropout_rate", "dtype", "precision", "use_flash_attention", "force_fp32_for_softmax", "norm_epsilon",
                "learn_sigma", "use_hilbert", "norm_groups", "activation", "context_dim")
        return {k: getattr(self, k) for k in keys}

    def param_specs(self):
        if not self.context_dim:
            raise FdxError(f"{type(self).__name__}: text conditioning is required; pass context_dim or init with a "
                           "textcontext")
        return super().param_specs()

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

    def _blocks(self):
        return [(f"mmdit_block_{i}", self._mm_block_fwd, self._mm_block_bwd) for i in range(self.num_layers)]

    def _block_specs(self, n):
        """MMDiTBlock `n`: ada_ln_zero's two projections (the kernels first and adjacent, so that their stack
        [2F, 6F] is one view of the flat buffer), then SimpleDiT's attention and MLP."""
        F = self._widths(n)[0]
        a = f"{n}/ada_ln_zero/"
        specs = [(a + "ada_t_proj/kernel", (F, 6 * F)), (a + "ada_text_proj/kernel", (F, 6 * F)),
                 (a + "ada_t_proj/bias", (6 * F,)), (a + "ada_text_proj/bias", (6 * F,))]
        return specs + [s for s in super()._block_specs(n) if "/ada_params_module/" not in s[0]]

    def _ada_leaf(self, n: str) -> str:
        return f"{n}/ada_ln_zero/ada_t_proj/kernel"

    def _init_leaf(self, name: str, t: torch.Tensor, gen: torch.Generator) -> None:
        """ada_t_proj / ada_text_proj kernels zero (their kernel_init); everything else as SimpleDiT."""
        if "/ada_ln_zero/" not in name:
            super()._init_leaf(name, t, gen)

    def _ada_stack(self, named, n: str) -> torch.Tensor:
        """[ada_t_proj; ada_text_proj] kernels of block n as one [2F, 6F] view of `named`'s flat buffer."""
        F = self._widths(n)[0]
        kt, kx = named[f"{n}/ada_ln_zero/ada_t_proj/kernel"], named[f"{n}/ada_ln_zero/ada_text_proj/kernel"]
        assert kx.data_ptr() == kt.data_ptr() + kt.numel() * kt.element_size(), "ada kernels are not adjacent"
        return kt.as_strided((2 * F, 6 * F), (6 * F, 1))

    # ------------------------------------------------------------------ forward program
    def forward(self, fp, x: torch.Tensor, temb: torch.Tensor, textcontext=None, save: bool = True):
        self._check_text(textcontext)
        return super().forward(fp, x, temb, textcontext, save)

    def _check_text(self, textcontext) -> None:
        name = type(self).__name__
        if textcontext is None:
            raise FdxError(f"{name}: textcontext is required (text-conditioned model)")
        if textcontext.dim() not in (2, 3):
            raise FdxError(f"{name}: textcontext must be [B, S, D] or [B, D], got {tuple(textcontext.shape)}")
        if int(textcontext.shape[-1]) != (self.context_dim or -1):
            raise FdxError(f"{name}: textcontext width {tuple(textcontext.shape)} does not match the parameters "
                           f"(context_dim={self.context_dim}); build / init the model with it")

    def _cond_width(self) -> int:
        return 2 * self.emb_features

    def _cond_fwd(self, W32, W16, temb, textcontext, B: int, dev):
        """bf16 [B, 2F] = [time_embed(t), text_context_proj(mean over tokens of ctx)]."""
        F = self.emb_features
        te = "time_embed/layers_"
        h2, tt = self._time_mlp_fwd("time_embed", temb, B, self._fourier_freqs(dev), W32, W16)
        cond16 = torch.empty((B, 2 * F), dtype=torch.bfloat16, device=dev)
        ops.linear_fwd(h2, W16[te + "2/kernel"], bias=W32[te + "2/bias"], out=cond16[:, :F])
        tc16 = self._text_rows(textcontext, B)
        ctx16 = ops.cast_f32_bf16(ops.dit_token_mean(tc16)) if tc16.dim() == 3 else tc16
        ops.linear_fwd(ctx16, W16["text_context_proj/kernel"], bias=W32["text_context_proj/bias"], out=cond16[:, F:])
        return cond16, (tt, h2, ctx16)

    def _cond_bwd(self, tape, dcond: torch.Tensor, W16, Gd) -> None:
        tt, h2, ctx16 = tape
        F = self.emb_features
        te = "time_embed/layers_"
        dt16 = ops.cast_f32_bf16(dcond[:, :F].contiguous())
        dx16 = ops.cast_f32_bf16(dcond[:, F:].contiguous())
        _dense_wgrad(Gd[te + "2/kernel"], h2, dt16)
        ops.colsum_rows(dt16, Gd[te + "2/bias"])
        _dense_wgrad(Gd["text_context_proj/kernel"], ctx16, dx16)
        ops.colsum_rows(dx16, Gd["text_context_proj/bias"])
        dh2 = _dense_dgrad(dt16, W16[te + "2/kernel"])
        self._time_mlp_bwd("time_embed", tt, dh2, W16, Gd)

    def _ada_fwd(self, n, cond16, W32, W16):
        a = f"{n}/ada_ln_zero/"
        return ops.linear_fwd(cond16, self._ada_stack(W16, n), bias=W32[a + "ada_t_proj/bias"] +
                              W32[a + "ada_text_proj/bias"], out_dtype=F32)

    def _ada_bwd(self, n, dada, cond16, dcond, Gd, W16):
        """ada = [t_emb, text_emb] [Wt; Wtext] + bt + btext: the kernel and bias gradients, dcond += dada [Wt; Wtext]^T."""
        F = self._widths(n)[0]
        a = f"{n}/ada_ln_zero/"
        dada16 = ops.cast_f32_bf16(dada)
        _dense_wgrad(self._ada_stack(Gd, n), cond16, dada16)
        ops.colsum_rows(dada16, Gd[a + "ada_t_proj/bias"])
        Gd[a + "ada_text_proj/bias"].copy_(Gd[a + "ada_t_proj/bias"])
        ops.gemm(GEMM_KK, dada16, self._ada_stack(W16, n), dcond, dada.shape[0], 2 * F, 6 * F, 6 * F, 6 * F, 2 * F,
                 atomic=True)

    def _mm_block_fwd(self, n, x, cond16, W32, W16, B, L):
        """MMDiTBlock: x + gate_attn * attn(x_attn) + gate_mlp * mlp(x_mlp), x_attn / x_mlp the two modulations of one
        LayerNorm of x.  ada chunks scale_mlp 0, shift_mlp 1, gate_mlp 2, scale_attn 3, shift_attn 4, gate_attn 5."""
        ada = self._ada_fwd(n, cond16, W32, W16)
        xa, xm, m1, r1 = ops.mmdit_adaln_fwd(x, L, ada, self.norm_epsilon)
        ya, attn = self._attn_fwd(n, xa, W32, W16, B, L)
        del xa
        ym, u = self._mlp_core_fwd(n, xm, W32, W16)
        del xm
        out = ops.mmdit_gate_fwd(x, ya, ym, L, ada)
        return out, (n, x, ada, m1, r1, attn, ya, u, ym)

    def _mm_block_bwd(self, rec, dout, cond16, dcond, W32, W16, Gd, B, L):
        n, x, ada, m1, r1, attn, ya, u, ym = rec
        F = self._widths(n)[0]
        dada = torch.empty((B, 6 * F), dtype=F32, device=x.device)
        dya, dym = ops.mmdit_gate_bwd(dout, ya, ym, L, ada, dada)
        # x_attn / x_mlp are recomputed (one pass writes both) when the MLP's weight gradient first needs x_mlp,
        # after that backward's own buffers are gone; x_mlp is dropped before the attention backward runs
        mod = []

        def modulated(i):
            if not mod:
                mod.extend(ops.mmdit_adaln_fwd(x, L, ada, self.norm_epsilon, stats=False)[:2])
            return mod[i]
        dxm = self._mlp_core_bwd(n, u, dym, lambda: modulated(1), W16, Gd)
        del dym
        mod[1] = None
        dxa = self._attn_bwd(n, attn, dya, lambda: modulated(0), Gd, B, L)
        del dya, mod
        dx = ops.mmdit_adaln_bwd(x, dxa, dxm, L, ada, m1, r1, dada, addend=dout)
        self._ada_bwd(n, dada, cond16, dcond, Gd, W16)
        return dx


class HierarchicalMMDiT(SimpleMMDiT):
    """The reference's U-shaped multi-resolution MMDiT (simple_mmdit.py:336-730) on the engine, with SimpleMMDiT's
    blocks at each stage's own width and heads.

        model = HierarchicalMMDiT(base_patch_size=8, emb_features=(512, 768, 1024), num_layers=(4, 4, 14),
                                  num_heads=(8, 12, 16), context_dim=768)

    Topology: encoder stages 0 .. N-1 (num_layers[s] blocks each; the skip is taken before merging), decoder stages
    N-2 .. 0 (num_layers[s] blocks each), each with its own RoPE width F_s / heads_s.  PatchMerging is the 2x2
    rearrange 'b (h p1) (w p2) c -> b h w (p1 p2 c)', an affine LayerNorm over 4C and a Dense; PatchExpanding a Dense to
    4C, the LayerNorm and the inverse rearrange; each decoder stage fuses with LayerNorm([expanded, skip]) and a Dense.
    The rearranges, the concat and the LayerNorms are one fdx_layernorm_rows pass each (and its backward), so no
    rearranged or concatenated copy is written.  Under use_hilbert the merge and expand treat the Hilbert-ordered
    sequence as a raster grid of the stage's HP x WP, as the reference's reshape does; the inverse permutation is
    applied once, at the finest level, before unpatchify.

    Conditioning: time_embed_base = Fourier(F_last) -> TimeProjection(4 F_last) -> Dense(F_last), the Fourier
    frequencies drawn at F_last; text_context_proj_base (Dense(F_last)), then per stage t_emb_proj_stage{s} /
    text_emb_proj_stage{s}, then each block's two ada projections.  All linear, so the text tokens are averaged first.

    Parameter names: flax attaches a named module constructed in setup() to the module being set up, even when it is
    then wrapped in an nn.Sequential; so the fusion layers are the top-level fusion_norm_{s} / fusion_dense_{s}, not
    fusion_layers_{i}/....  Nobody has checked this against a flax-written file (the reference ships no MMDiT
    checkpoint); the names are pinned in tests/test_mmdit_cpu.py.

    Refused with FdxError: tuples of different lengths, and per stage what SimpleMMDiT refuses (F_s not a multiple of
    heads_s or of 64 or above 1536, odd head widths - training.py's hierarchical mapping of num_heads = 12 gives 51- and
    73-wide heads, where the reference itself fails - heads wider than 256), use_flash_attention, a dtype other than
    bf16, and images not divisible by base_patch_size * 2^(stages - 1).
    """

    # SimpleDiT.__init__ validates one width; the stage tuples are validated here instead.
    def __init__(self, output_channels: int = 3, base_patch_size: int = 8, emb_features=(512, 768, 1024),
                 num_layers=(4, 4, 14), num_heads=(8, 12, 16), mlp_ratio: int = 4, dropout_rate: float = 0.0,
                 dtype=None, precision=None, use_flash_attention: bool = False, force_fp32_for_softmax: bool = True,
                 norm_epsilon: float = 1e-5, learn_sigma: bool = False, use_hilbert: bool = False,
                 norm_groups: int = 0, activation=None, context_dim: Optional[int] = None):
        name = type(self).__name__
        Fs, Ls, Hs = tuple(emb_features), tuple(num_layers), tuple(num_heads)
        if not Fs or not len(Fs) == len(Ls) == len(Hs):
            raise FdxError(f"{name}: emb_features, num_layers and num_heads must have the same number of stages "
                           f"(got {len(Fs)}, {len(Ls)}, {len(Hs)})")
        if use_flash_attention:
            raise FdxError(f"{name}: use_flash_attention=True has no counterpart here; the fused attention kernel is "
                           "always used")
        if dtype is not None and dtype != torch.bfloat16:
            raise FdxError(f"{name}: dtype={dtype} is not supported: the engine computes in bf16 with f32 "
                           "accumulation (pass dtype=None or torch.bfloat16)")
        for s, (F, h) in enumerate(zip(Fs, Hs)):
            if h <= 0 or F % h != 0:
                raise FdxError(f"{name}: stage {s}: emb_features={F} is not a multiple of num_heads={h}")
            d = F // h
            if d % 2:
                raise FdxError(f"{name}: stage {s}: head width {d} is odd (RoPE rotates channel pairs)")
            if d > 256:
                raise FdxError(f"{name}: stage {s}: head width {d} > 256 is not supported by the fused attention")
            if F % 64 or F > 1536:
                raise FdxError(f"{name}: stage {s}: emb_features={F} must be a multiple of 64, at most 1536")
        self.output_channels = output_channels
        self.base_patch_size = self.patch_size = base_patch_size
        self.emb_features, self.num_layers, self.num_heads = Fs, Ls, Hs
        self.mlp_ratio = mlp_ratio
        self.dropout_rate = dropout_rate        # accepted and unused, as in the reference
        self.dtype = dtype
        self.precision = precision
        self.use_flash_attention = use_flash_attention
        self.force_fp32_for_softmax = force_fp32_for_softmax
        self.norm_epsilon = norm_epsilon
        self.learn_sigma = learn_sigma
        self.use_hilbert = use_hilbert
        self.use_zigzag = False
        self.norm_groups = norm_groups
        self.activation = activation
        self.context_dim = context_dim
        self._layouts = {}
        self._consts = {}
        self._stage = {n: s for s in range(len(Fs)) for n in self._stage_blocks("encoder", s) +
                       self._stage_blocks("decoder", s)}

    # ------------------------------------------------------------------ structure
    def config(self) -> dict:
        """The constructor arguments (a config round trip: HierarchicalMMDiT(**model.config()))."""
        keys = ("output_channels", "base_patch_size", "emb_features", "num_layers", "num_heads", "mlp_ratio",
                "dropout_rate", "dtype", "precision", "use_flash_attention", "force_fp32_for_softmax", "norm_epsilon",
                "learn_sigma", "use_hilbert", "norm_groups", "activation", "context_dim")
        return {k: getattr(self, k) for k in keys}

    def _stage_blocks(self, kind: str, s: int):
        return [f"{kind}_block_stage{s}_{i}" for i in range(self.num_layers[s])]

    def _widths(self, n: str):
        s = self._stage[n]
        return self.emb_features[s], self.num_heads[s]

    def _blocks(self):
        N = len(self.emb_features)
        names = [n for s in range(N) for n in self._stage_blocks("encoder", s)]
        names += [n for s in range(N - 2, -1, -1) for n in self._stage_blocks("decoder", s)]
        return [(n, self._mm_block_fwd, self._mm_block_bwd) for n in names]

    def _embed_specs(self):
        p, F = self.patch_size, self.emb_features[0]
        if self.use_hilbert:
            return [("hilbert_projection/kernel", (p * p * 3, F)), ("hilbert_projection/bias", (F,))]
        return [("patch_embed/Conv_0/kernel", (p, p, 3, F)), ("patch_embed/Conv_0/bias", (F,))]

    def param_specs(self):
        if not self.context_dim:
            raise FdxError(f"{type(self).__name__}: text conditioning is required; pass context_dim or init with a "
                           "textcontext")
        Fs, N = self.emb_features, len(self.emb_features)
        FL = Fs[-1]
        E = FL * self.mlp_ratio
        p = self.patch_size
        nout = p * p * self.output_channels * (2 if self.learn_sigma else 1)
        te = "time_embed_base/layers_"
        specs = self._embed_specs() + [
            (te + "1/DenseGeneral_0/kernel", (FL, E)), (te + "1/DenseGeneral_0/bias", (E,)),
            (te + "1/DenseGeneral_1/kernel", (E, E)), (te + "1/DenseGeneral_1/bias", (E,)),
            (te + "2/kernel", (E, FL)), (te + "2/bias", (FL,)),
            ("text_context_proj_base/kernel", (self.context_dim, FL)), ("text_context_proj_base/bias", (FL,))]
        for s in range(N):
            for m in ("t_emb_proj", "text_emb_proj"):
                specs += [(f"{m}_stage{s}/kernel", (FL, Fs[s])), (f"{m}_stage{s}/bias", (Fs[s],))]
        for s in range(N):
            for n in self._stage_blocks("encoder", s):
                specs += self._block_specs(n)
            if s < N - 1:
                m = f"patch_merger_{s}/"
                specs += [(m + "norm/scale", (4 * Fs[s],)), (m + "norm/bias", (4 * Fs[s],)),
                          (m + "projection/kernel", (4 * Fs[s], Fs[s + 1])), (m + "projection/bias", (Fs[s + 1],))]
        for s in range(N - 2, -1, -1):
            m = f"patch_expander_{s}/"
            specs += [(m + "projection/kernel", (Fs[s + 1], 4 * Fs[s])), (m + "projection/bias", (4 * Fs[s],)),
                      (m + "norm/scale", (4 * Fs[s],)), (m + "norm/bias", (4 * Fs[s],)),
                      (f"fusion_norm_{s}/scale", (2 * Fs[s],)), (f"fusion_norm_{s}/bias", (2 * Fs[s],)),
                      (f"fusion_dense_{s}/kernel", (2 * Fs[s], Fs[s])), (f"fusion_dense_{s}/bias", (Fs[s],))]
            for n in self._stage_blocks("decoder", s):
                specs += self._block_specs(n)
        specs += [("final_norm/scale", (Fs[0],)), ("final_norm/bias", (Fs[0],)),
                  ("final_proj/kernel", (Fs[0], nout)), ("final_proj/bias", (nout,))]
        return specs

    def _fourier_freqs(self, device) -> torch.Tensor:
        """time_embed_base's FourierEmbedding(F_last): normal(PRNGKey(42), F_last / 2) * 16."""
        from .. import utils
        key = ("freqs_base", str(device))
        if key not in self._consts:
            f = utils.normal(utils.PRNGKey(42), self.emb_features[-1] // 2) * 16.0
            self._consts[key] = torch.from_numpy(f.astype("float32")).to(device)
        return self._consts[key]

    # ------------------------------------------------------------------ forward program
    def forward(self, fp, x: torch.Tensor, temb: torch.Tensor, textcontext=None, save: bool = True):
        """x (B, H, W, 3) -> (F f32 (B, H, W, output_channels), tape or None)."""
        self._check_text(textcontext)
        B, H, W, _ = x.shape
        Fs, N, p, eps = self.emb_features, len(self.emb_features), self.patch_size, self.norm_epsilon
        q = p * 2 ** (N - 1)
        if H % q or W % q:
            raise FdxError(f"{type(self).__name__}: image {H}x{W} is not divisible by the coarsest patch size "
                           f"{p} * 2^{N - 1} = {q}")
        W32, W16 = fp.named, fp.shadow()
        dev = x.device
        HP, WP = H // p, W // p
        grids = [(HP >> s, WP >> s) for s in range(N)]

        # conditioning: the base time / text embeddings, then one [t_emb_s, text_emb_s] row per stage
        h2, tt = self._time_mlp_fwd("time_embed_base", temb, B, self._fourier_freqs(dev), W32, W16)
        tb16 = ops.linear_fwd(h2, W16["time_embed_base/layers_2/kernel"], bias=W32["time_embed_base/layers_2/bias"])
        tc16 = self._text_rows(textcontext, B)
        ctx16 = ops.cast_f32_bf16(ops.dit_token_mean(tc16)) if tc16.dim() == 3 else tc16
        xb16 = ops.linear_fwd(ctx16, W16["text_context_proj_base/kernel"], bias=W32["text_context_proj_base/bias"])
        conds = []
        for s in range(N):
            c16 = torch.empty((B, 2 * Fs[s]), dtype=torch.bfloat16, device=dev)
            ops.linear_fwd(tb16, W16[f"t_emb_proj_stage{s}/kernel"], bias=W32[f"t_emb_proj_stage{s}/bias"],
                           out=c16[:, :Fs[s]])
            ops.linear_fwd(xb16, W16[f"text_emb_proj_stage{s}/kernel"], bias=W32[f"text_emb_proj_stage{s}/bias"],
                           out=c16[:, Fs[s]:])
            conds.append(c16)

        order = self._order(HP, WP, dev)
        tok, rows = self._embed_fwd(x, W32, W16, HP, WP, order)
        recs, skips, merges = {}, [], []
        for s in range(N):                                                   # encoder, fine to coarse
            L = grids[s][0] * grids[s][1]
            for n in self._stage_blocks("encoder", s):
                tok, recs[n] = self._mm_block_fwd(n, tok, conds[s], W32, W16, B, L)
            skips.append(tok)
            if s < N - 1:
                m = f"patch_merger_{s}/"
                hc, wc = grids[s + 1]
                mg = ops.layernorm_rows_fwd(ops.LN_GATHER, tok, None, B * hc * wc, 4 * Fs[s], W32[m + "norm/scale"],
                                            W32[m + "norm/bias"], eps, grid=(hc, wc))
                tok = ops.linear_fwd(mg[0], W16[m + "projection/kernel"], bias=W32[m + "projection/bias"])
                merges.append(mg)
        dec = []
        for s in range(N - 2, -1, -1):                                       # decoder, coarse to fine
            hc, wc = grids[s + 1]
            L = grids[s][0] * grids[s][1]
            m = f"patch_expander_{s}/"
            u = ops.linear_fwd(tok, W16[m + "projection/kernel"], bias=W32[m + "projection/bias"])
            e, em, er = ops.layernorm_rows_fwd(ops.LN_SCATTER, u, None, B * hc * wc, 4 * Fs[s],
                                               W32[m + "norm/scale"], W32[m + "norm/bias"], eps, grid=(hc, wc))
            c, cm, cr = ops.layernorm_rows_fwd(ops.LN_CONCAT, e, skips[s], B * L, 2 * Fs[s],
                                               W32[f"fusion_norm_{s}/scale"], W32[f"fusion_norm_{s}/bias"], eps)
            dec.append((s, tok, u, em, er, e, c, cm, cr))
            tok = ops.linear_fwd(c, W16[f"fusion_dense_{s}/kernel"], bias=W32[f"fusion_dense_{s}/bias"])
            for n in self._stage_blocks("decoder", s):
                tok, recs[n] = self._mm_block_fwd(n, tok, conds[s], W32, W16, B, L)
        out, final = self._final_fwd(tok, W32, W16, B, H, W, grids[0][0] * grids[0][1], order)
        if not save:
            return out, None
        return out, {"B": B, "grids": grids, "order": order, "rows": rows, "cond": (tt, h2, tb16, ctx16, xb16, conds),
                     "recs": recs, "skips": skips, "merges": merges, "dec": dec, "final": final}

    # ------------------------------------------------------------------ backward program
    def backward(self, fp, saved: dict, dF: torch.Tensor, grads, on_ready=None):
        """As SimpleDiT.backward.  The stage-conditioning gradients collect over every block, so the gradients are
        announced final once, at the end (on_ready(0))."""
        W32, W16, Gd = fp.named, fp.shadow(), grads.named
        B, grids, recs, skips = saved["B"], saved["grids"], saved["recs"], saved["skips"]
        Fs, N = self.emb_features, len(self.emb_features)
        dev = dF.device
        tt, h2, tb16, ctx16, xb16, conds = saved["cond"]
        dconds = [torch.zeros((B, 2 * F), dtype=F32, device=dev) for F in Fs]
        dx = self._final_bwd(saved["final"], dF, saved["order"], W32, Gd, grids[0][0] * grids[0][1])
        dskips = [None] * N
        for s, tin, u, em, er, e, c, cm, cr in reversed(saved["dec"]):      # decoder, fine to coarse
            hc, wc = grids[s + 1]
            L = grids[s][0] * grids[s][1]
            for n in reversed(self._stage_blocks("decoder", s)):
                dx = self._mm_block_bwd(recs[n], dx, conds[s], dconds[s], W32, W16, Gd, B, L)
            _dense_wgrad(Gd[f"fusion_dense_{s}/kernel"], c, dx)
            ops.colsum_rows(dx, Gd[f"fusion_dense_{s}/bias"])
            dc = _dense_dgrad(dx, W16[f"fusion_dense_{s}/kernel"])
            de, dskips[s] = ops.layernorm_rows_bwd(ops.LN_CONCAT, e, skips[s], dc, B * L, 2 * Fs[s],
                                                   W32[f"fusion_norm_{s}/scale"], cm, cr,
                                                   Gd[f"fusion_norm_{s}/scale"], Gd[f"fusion_norm_{s}/bias"])
            m = f"patch_expander_{s}/"
            du, _ = ops.layernorm_rows_bwd(ops.LN_SCATTER, u, None, de, B * hc * wc, 4 * Fs[s],
                                           W32[m + "norm/scale"], em, er, Gd[m + "norm/scale"], Gd[m + "norm/bias"],
                                           grid=(hc, wc))
            _dense_wgrad(Gd[m + "projection/kernel"], tin, du)
            ops.colsum_rows(du, Gd[m + "projection/bias"])
            dx = _dense_dgrad(du, W16[m + "projection/kernel"])
        for s in range(N - 1, -1, -1):                                       # encoder, coarse to fine
            L = grids[s][0] * grids[s][1]
            if s < N - 1:
                # the skip's gradient is the fusion path's (in dskips[s]) plus the merge path's, added in place
                hc, wc = grids[s + 1]
                m = f"patch_merger_{s}/"
                mg, mm, mr = saved["merges"][s]
                _dense_wgrad(Gd[m + "projection/kernel"], mg, dx)
                ops.colsum_rows(dx, Gd[m + "projection/bias"])
                dmg = _dense_dgrad(dx, W16[m + "projection/kernel"])
                dx, _ = ops.layernorm_rows_bwd(ops.LN_GATHER, skips[s], None, dmg, B * hc * wc, 4 * Fs[s],
                                               W32[m + "norm/scale"], mm, mr, Gd[m + "norm/scale"],
                                               Gd[m + "norm/bias"], grid=(hc, wc), dx0=dskips[s], accumulate0=True)
            for n in reversed(self._stage_blocks("encoder", s)):
                dx = self._mm_block_bwd(recs[n], dx, conds[s], dconds[s], W32, W16, Gd, B, L)
        self._embed_bwd(saved["rows"], dx, Gd)

        # conditioning: the stage projections, then the base embeddings
        FL = Fs[-1]
        dtb = torch.zeros((B, FL), dtype=F32, device=dev)
        dxb = torch.zeros((B, FL), dtype=F32, device=dev)
        for s, F in enumerate(Fs):
            for half, (m, src, acc) in enumerate((("t_emb_proj", tb16, dtb), ("text_emb_proj", xb16, dxb))):
                d16 = ops.cast_f32_bf16(dconds[s][:, half * F:(half + 1) * F].contiguous())
                _dense_wgrad(Gd[f"{m}_stage{s}/kernel"], src, d16)
                ops.colsum_rows(d16, Gd[f"{m}_stage{s}/bias"])
                ops.gemm(GEMM_KK, d16, W16[f"{m}_stage{s}/kernel"], acc, B, FL, F, F, F, FL, atomic=True)
        te = "time_embed_base/layers_"
        dt16 = ops.cast_f32_bf16(dtb)
        _dense_wgrad(Gd[te + "2/kernel"], h2, dt16)
        ops.colsum_rows(dt16, Gd[te + "2/bias"])
        self._time_mlp_bwd("time_embed_base", tt, _dense_dgrad(dt16, W16[te + "2/kernel"]), W16, Gd)
        dx16 = ops.cast_f32_bf16(dxb)
        _dense_wgrad(Gd["text_context_proj_base/kernel"], ctx16, dx16)
        ops.colsum_rows(dx16, Gd["text_context_proj_base/bias"])
        if on_ready is not None:
            on_ready(0, [torch.cuda.current_stream()])
