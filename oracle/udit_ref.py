"""CPU restatement of the reference's SimpleUDiT (flaxdiff/models/simple_vit.py:255-446) in plain torch, built on
oracle/dit_ref.py's DiTBlock; autograd gives the backward.  It runs in the dtype of the parameters (fp32 against the
GPU, float64 for gradcheck).  Parameters are a dict of flax names -> tensors in flaxdiff_b200's layout.

The text path is restated as the reference computes it - text_proj over every token, then the mean over tokens when the
text is 3-D - not in the engine's pool-first order, so that agreement also checks that reordering."""
from __future__ import annotations

import torch

from oracle.dit_ref import dense, dit_block, layernorm
from oracle.mmdit_ref import time_embed


def simple_udit_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, *, patch_size: int,
                        num_layers: int, num_heads: int, output_channels: int = 3, norm_epsilon: float = 1e-5,
                        textcontext=None, order=None):
    """SimpleUDiT.__call__: x (B, H, W, C) -> (B, H, W, out).  order: the Hilbert patch order (token i is row-major
    patch order[i]) or None.  No position table: RoPE, on in both orders, is the only position signal."""
    dt = P["final_proj/kernel"].dtype
    B, H, W, C = x.shape
    p = patch_size
    HP, WP = H // p, W // p
    F = P["final_norm/scale"].shape[0]
    patches = x.to(dt).reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, HP * WP, p * p * C)
    if order is None:   # PatchEmbedding: a p x p stride-p conv over (p1, p2, c) patches
        tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(p * p * C, F) + P["patch_embed/Conv_0/bias"]
    else:               # hilbert_patchify + hilbert_projection
        tok = dense(P, "hilbert_projection", patches[:, torch.as_tensor(order)])
    cond = time_embed(P, t, freqs)
    if textcontext is not None:
        text = dense(P, "text_proj", textcontext.to(dt))
        cond = cond + (text.mean(1) if text.dim() == 3 else text)
    half = num_layers // 2
    skips = []
    for i in range(half):
        tok = dit_block(P, f"down_block_{i}", tok, cond, num_heads, norm_epsilon)
        skips.append(tok)
    tok = dit_block(P, "mid_block", tok, cond, num_heads, norm_epsilon)
    for i in range(half):
        tok = dense(P, f"up_dense_{i}", torch.cat([tok, skips.pop()], -1))
        tok = dit_block(P, f"up_block_{i}", tok, cond, num_heads, norm_epsilon)
    out = layernorm(tok, norm_epsilon, P["final_norm/scale"], P["final_norm/bias"])
    out = dense(P, "final_proj", out)[..., :p * p * output_channels]        # learn_sigma keeps the mean half
    if order is not None:  # hilbert_unpatchify: back to row-major
        inv = torch.empty(len(order), dtype=torch.long)
        inv[torch.as_tensor(order)] = torch.arange(len(order))
        out = out[:, inv]
    return out.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)
