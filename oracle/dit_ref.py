"""fp32 CPU restatement of the reference's SimpleDiT (flaxdiff/models/simple_dit.py) in plain torch, from the formulas of
its modules; autograd gives the backward.  Parameters are a dict of flax names -> tensors (flaxdiff_b200's layout:
dense kernels (in, out), DenseGeneral kernels (in, heads, d) / (heads, d, out), the patch conv HWIO)."""
from __future__ import annotations

import math

import numpy as np
import torch


def sincos_2d(F: int, HP: int, WP: int) -> np.ndarray:
    """build_2d_sincos_pos_embed (hilbert.py:12-45): [HP*WP, F] in row-major patch order; the quarters are row-sin,
    row-cos, col-sin, col-cos with omega = 10000^(-i/quarter)."""
    quarter = F // 4
    omega = 1.0 / (10000.0 ** (np.arange(quarter, dtype=np.float32) / np.float32(quarter)))
    rows = np.arange(HP, dtype=np.float32)[:, None] * omega[None]
    cols = np.arange(WP, dtype=np.float32)[:, None] * omega[None]
    pos = np.zeros((HP, WP, F), dtype=np.float32)
    pos[..., 0:quarter] = np.sin(rows)[:, None, :]
    pos[..., quarter:2 * quarter] = np.cos(rows)[:, None, :]
    pos[..., 2 * quarter:3 * quarter] = np.sin(cols)[None, :, :]
    pos[..., 3 * quarter:4 * quarter] = np.cos(cols)[None, :, :]
    return pos.reshape(HP * WP, F)


def rope(x: torch.Tensor) -> torch.Tensor:
    """RotaryEmbedding + apply_rotary_embedding (vit_common.py:56-104) on x [B, L, heads, d]: position = token index,
    x*cos + rotate_half(x)*sin with cos / sin concatenated twice, rotate_half = concat(-x[d/2:], x[:d/2])."""
    L, d = x.shape[1], x.shape[3]
    inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    fr = torch.arange(L, dtype=torch.float32)[:, None] * inv[None]
    cos = torch.cat([fr.cos(), fr.cos()], -1)[None, :, None, :]
    sin = torch.cat([fr.sin(), fr.sin()], -1)[None, :, None, :]
    rot = torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1)
    return x * cos + rot * sin


def layernorm(x: torch.Tensor, eps: float, scale=None, bias=None) -> torch.Tensor:
    """nn.LayerNorm over the last axis (biased variance)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    if scale is not None:
        y = y * scale + bias
    return y


def gelu_tanh(z: torch.Tensor) -> torch.Tensor:
    """jax.nn.gelu (approximate=True, its default)."""
    return 0.5 * z * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (z + 0.044715 * z ** 3)))


def dense(P, name, x):
    return x @ P[name + "/kernel"] + P[name + "/bias"]


def time_embed(P, t: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    """nn.Sequential([FourierEmbedding(F), TimeProjection(4F), Dense(F)]) (simple_dit.py:146-152; common.py:97-124)."""
    arg = t.float()[:, None] * (2 * math.pi * freqs)[None, :]
    h = torch.cat([arg.sin(), arg.cos()], -1)
    h = gelu_tanh(dense(P, "time_embed/layers_1/DenseGeneral_0", h))
    h = gelu_tanh(dense(P, "time_embed/layers_1/DenseGeneral_1", h))
    return dense(P, "time_embed/layers_2", h)


def attention(P, base, x, heads):
    """RoPEAttention (vit_common.py:121-183) = NormalAttention (attention.py:117-177) with biases, q and k rotated."""
    B, L, F = x.shape
    d = F // heads
    q = torch.einsum("blf,fhd->blhd", x, P[base + "/to_q/kernel"]) + P[base + "/to_q/bias"]
    k = torch.einsum("blf,fhd->blhd", x, P[base + "/to_k/kernel"]) + P[base + "/to_k/bias"]
    v = torch.einsum("blf,fhd->blhd", x, P[base + "/to_v/kernel"]) + P[base + "/to_v/bias"]
    q, k = rope(q), rope(k)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(d)
    o = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v)
    return torch.einsum("blhd,hdf->blf", o, P[base + "/to_out_0/kernel"]) + P[base + "/to_out_0/bias"]


def dit_block(P, name, x, cond, heads, eps):
    """DiTBlock (simple_dit.py:23-92) with AdaLNParams (vit_common.py:240-261): ada_proj's 6F columns split as
    scale_mlp, shift_mlp, gate_mlp, scale_attn, shift_attn, gate_attn; LayerNorms without scale / bias."""
    ada = dense(P, f"{name}/ada_params_module/ada_proj", cond)[:, None, :]
    sc_m, sh_m, g_m, sc_a, sh_a, g_a = ada.chunk(6, -1)
    x = x + g_a * attention(P, f"{name}/attention", layernorm(x, eps) * (1 + sc_a) + sh_a, heads)
    h = layernorm(x, eps) * (1 + sc_m) + sh_m
    h = dense(P, f"{name}/mlp/layers_2", gelu_tanh(dense(P, f"{name}/mlp/layers_0", h)))
    return x + g_m * h


def simple_dit_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, *, patch_size: int, num_layers: int,
                       num_heads: int, output_channels: int = 3, norm_epsilon: float = 1e-5, textcontext=None):
    """SimpleDiT.__call__ (simple_dit.py:236-306), raster patch order: x (B, H, W, C) f32 -> (B, H, W, out) f32."""
    B, H, W, C = x.shape
    p = patch_size
    HP, WP = H // p, W // p
    F = P["patch_embed/Conv_0/bias"].shape[0]
    # PatchEmbedding (vit_common.py:20-37): a p x p stride-p conv = a dense layer over (p1, p2, c)-ordered patches
    patches = x.reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, HP * WP, p * p * C)
    tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(p * p * C, F) + P["patch_embed/Conv_0/bias"]
    tok = tok + torch.from_numpy(sincos_2d(F, HP, WP))[None]
    cond = time_embed(P, t, freqs)
    if textcontext is not None:
        cond = cond + dense(P, "text_context_proj", textcontext.float()).mean(1)
    for i in range(num_layers):
        tok = dit_block(P, f"dit_block_{i}", tok, cond, num_heads, norm_epsilon)
    out = layernorm(tok, norm_epsilon, P["final_norm/scale"], P["final_norm/bias"])
    out = dense(P, "final_proj", out)[..., :p * p * output_channels]        # learn_sigma keeps the first half
    # unpatchify (vit_common.py:10-17): 'B (h w) (p1 p2 C) -> B (h p1) (w p2) C'
    return out.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)
