"""CPU restatement of the reference's SimpleMMDiT (flaxdiff/models/simple_mmdit.py:17-331) in plain torch, from the
formulas of its modules; autograd gives the backward.  It runs in the dtype of the parameters (fp32 against the GPU,
float64 for gradcheck).  Parameters are a dict of flax names -> tensors in flaxdiff_b200's layout (dense kernels
(in, out), DenseGeneral kernels (in, heads, d) / (heads, d, out), the patch conv HWIO).

The text path is restated as the reference computes it - text_context_proj over every token, then MMAdaLNZero's mean
pooling and ada_text_proj per block (:44-72) - not in the engine's pool-first order, so that agreement also checks
that reordering."""
from __future__ import annotations

import math

import torch

from oracle.dit_ref import attention, dense, gelu_tanh, layernorm

CLIP = 10.0


class Clip10(torch.autograd.Function):
    """jnp.clip(v, -10, 10) (simple_mmdit.py:81-82) with JAX's derivative: clip = min(max(v, lo), hi), and
    lax.max / lax.min's JVP splits the cotangent evenly between equal operands, so the gradient is passed inside
    (-10, 10), zero outside and halved at exactly -10 or 10.  (Derived from that rule; not pinned against JAX.)"""

    @staticmethod
    def forward(ctx, v):
        ctx.save_for_backward(v)
        return v.clamp(-CLIP, CLIP)

    @staticmethod
    def backward(ctx, g):
        (v,) = ctx.saved_tensors
        inside = ((v > -CLIP) & (v < CLIP)).to(g.dtype)
        tie = ((v == -CLIP) | (v == CLIP)).to(g.dtype)
        return g * (inside + 0.5 * tie)


clip10 = Clip10.apply


def time_embed(P, t: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    """nn.Sequential([FourierEmbedding(F), TimeProjection(4F), Dense(F)]) (simple_mmdit.py:196-202)."""
    dt = P["time_embed/layers_2/kernel"].dtype
    arg = t.to(dt)[:, None] * (2 * math.pi * freqs.to(dt))[None, :]
    h = torch.cat([arg.sin(), arg.cos()], -1)
    h = gelu_tanh(dense(P, "time_embed/layers_1/DenseGeneral_0", h))
    h = gelu_tanh(dense(P, "time_embed/layers_1/DenseGeneral_1", h))
    return dense(P, "time_embed/layers_2", h)


def mm_adaln_zero(P, name, x, t_emb, text_emb, eps):
    """MMAdaLNZero (:17-90) -> (x_attn, gate_attn, x_mlp, gate_mlp)."""
    nx = layernorm(x, eps)
    t_emb = t_emb[:, None, :]
    if text_emb.dim() == 2:
        text_emb = text_emb[:, None, :]
    elif text_emb.shape[1] != x.shape[1]:
        text_emb = text_emb.mean(1, keepdim=True)
    t_params = dense(P, f"{name}/ada_t_proj", t_emb)
    text_params = dense(P, f"{name}/ada_text_proj", text_emb)
    if t_params.shape[1] != text_params.shape[1]:
        text_params = text_params.mean(1, keepdim=True)
    sc_m, sh_m, g_m, sc_a, sh_a, g_a = (t_params + text_params).chunk(6, -1)
    sc_m, sh_m = clip10(sc_m), clip10(sh_m)
    return nx * (1 + sc_a) + sh_a, g_a, nx * (1 + sc_m) + sh_m, g_m


def mmdit_block(P, name, x, t_emb, text_emb, heads, eps):
    """MMDiTBlock (:94-158): the attention and the MLP both read the one LayerNorm of the block input."""
    x_attn, g_a, x_mlp, g_m = mm_adaln_zero(P, f"{name}/ada_ln_zero", x, t_emb, text_emb, eps)
    x = x + g_a * attention(P, f"{name}/attention", x_attn, heads)
    h = dense(P, f"{name}/mlp/layers_2", gelu_tanh(dense(P, f"{name}/mlp/layers_0", x_mlp)))
    return x + g_m * h


def simple_mmdit_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, textcontext: torch.Tensor, *,
                         patch_size: int, num_layers: int, num_heads: int, output_channels: int = 3,
                         norm_epsilon: float = 1e-5, order=None):
    """SimpleMMDiT.__call__ (:257-331): x (B, H, W, C) -> (B, H, W, out).  order: the Hilbert patch order (token i is
    row-major patch order[i]) or None.  No position table: RoPE (on in both orders) is the only position signal."""
    dt = P["final_proj/kernel"].dtype
    B, H, W, C = x.shape
    p = patch_size
    HP, WP = H // p, W // p
    F = P["final_norm/scale"].shape[0]
    patches = x.to(dt).reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, HP * WP, p * p * C)
    if order is None:   # PatchEmbedding (vit_common.py:20-37): a p x p stride-p conv over (p1, p2, c) patches
        tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(p * p * C, F) + P["patch_embed/Conv_0/bias"]
    else:               # hilbert_patchify (hilbert.py:213-246) + hilbert_projection
        tok = dense(P, "hilbert_projection", patches[:, torch.as_tensor(order)])
    t_emb = time_embed(P, t, freqs)
    text_emb = dense(P, "text_context_proj", textcontext.to(dt))
    for i in range(num_layers):
        tok = mmdit_block(P, f"mmdit_block_{i}", tok, t_emb, text_emb, num_heads, norm_epsilon)
    out = layernorm(tok, norm_epsilon, P["final_norm/scale"], P["final_norm/bias"])
    out = dense(P, "final_proj", out)[..., :p * p * output_channels]        # learn_sigma keeps the first half
    if order is not None:  # hilbert_unpatchify: back to row-major
        inv = torch.empty(len(order), dtype=torch.long)
        inv[torch.as_tensor(order)] = torch.arange(len(order))
        out = out[:, inv]
    return out.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)


# ---------------------------------------------------------------------------------------------- HierarchicalMMDiT
def patch_merge(x: torch.Tensor, HP: int, WP: int) -> torch.Tensor:
    """PatchMerging's rearrange (:356-363): [B, HP*WP, C] -> [B, HP/2*WP/2, 4C], 'b (h p1) (w p2) c -> b h w (p1 p2 c)'."""
    B, _, C = x.shape
    x = x.reshape(B, HP // 2, 2, WP // 2, 2, C).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(B, (HP // 2) * (WP // 2), 4 * C)


def patch_expand(x: torch.Tensor, HP: int, WP: int) -> torch.Tensor:
    """PatchExpanding's rearrange (:415-427): [B, HP*WP, 4C] -> [B, 2HP*2WP, C], the inverse of patch_merge."""
    B, _, C4 = x.shape
    C = C4 // 4
    x = x.reshape(B, HP, WP, 2, 2, C).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(B, 4 * HP * WP, C)


def hierarchical_mmdit_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, textcontext: torch.Tensor,
                               *, base_patch_size: int, num_layers, num_heads, output_channels: int = 3,
                               norm_epsilon: float = 1e-5, order=None):
    """HierarchicalMMDiT.__call__ (:627-730): x (B, H, W, C) -> (B, H, W, out); freqs are time_embed_base's Fourier
    frequencies (drawn at the last stage's width).  order: the finest grid's Hilbert order or None."""
    dt = P["final_proj/kernel"].dtype
    eps = norm_epsilon
    B, H, W, C = x.shape
    p, N = base_patch_size, len(num_layers)
    HP, WP = H // p, W // p
    patches = x.to(dt).reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, HP * WP, p * p * C)
    if order is None:
        F0 = P["patch_embed/Conv_0/bias"].shape[0]
        tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(p * p * C, F0) + P["patch_embed/Conv_0/bias"]
    else:
        tok = dense(P, "hilbert_projection", patches[:, torch.as_tensor(order)])
    arg = t.to(dt)[:, None] * (2 * math.pi * freqs.to(dt))[None, :]
    h = torch.cat([arg.sin(), arg.cos()], -1)
    h = gelu_tanh(dense(P, "time_embed_base/layers_1/DenseGeneral_0", h))
    h = gelu_tanh(dense(P, "time_embed_base/layers_1/DenseGeneral_1", h))
    t_base = dense(P, "time_embed_base/layers_2", h)
    text_base = dense(P, "text_context_proj_base", textcontext.to(dt))
    t_embs = [dense(P, f"t_emb_proj_stage{s}", t_base) for s in range(N)]
    text_embs = [dense(P, f"text_emb_proj_stage{s}", text_base) for s in range(N)]
    skips, h_, w_ = {}, HP, WP
    for s in range(N):
        for i in range(num_layers[s]):
            tok = mmdit_block(P, f"encoder_block_stage{s}_{i}", tok, t_embs[s], text_embs[s], num_heads[s], eps)
        skips[s] = tok
        if s < N - 1:
            m = f"patch_merger_{s}"
            tok = layernorm(patch_merge(tok, h_, w_), eps, P[m + "/norm/scale"], P[m + "/norm/bias"])
            tok = dense(P, m + "/projection", tok)
            h_, w_ = h_ // 2, w_ // 2
    for s in range(N - 2, -1, -1):
        m = f"patch_expander_{s}"
        e = layernorm(dense(P, m + "/projection", tok), eps, P[m + "/norm/scale"], P[m + "/norm/bias"])
        tok = patch_expand(e, h_, w_)
        h_, w_ = h_ * 2, w_ * 2
        tok = torch.cat([tok, skips[s]], -1)
        tok = dense(P, f"fusion_dense_{s}", layernorm(tok, eps, P[f"fusion_norm_{s}/scale"],
                                                      P[f"fusion_norm_{s}/bias"]))
        for i in range(num_layers[s]):
            tok = mmdit_block(P, f"decoder_block_stage{s}_{i}", tok, t_embs[s], text_embs[s], num_heads[s], eps)
    out = layernorm(tok, eps, P["final_norm/scale"], P["final_norm/bias"])
    out = dense(P, "final_proj", out)[..., :p * p * output_channels]
    if order is not None:
        inv = torch.empty(len(order), dtype=torch.long)
        inv[torch.as_tensor(order)] = torch.arange(len(order))
        out = out[:, inv]
    return out.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)
