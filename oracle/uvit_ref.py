"""CPU restatement of the reference's UViT (flaxdiff/models/simple_vit.py:18-250) in plain torch; autograd gives the
backward.  Test infrastructure: flaxdiff_b200 never imports it.  Parameters are a dict of flax names -> tensors in
flaxdiff_b200's layout.

It follows the reference's dtype flow.  With `round_bf16` (the default for float32 parameters) every output of a
module flax runs in bf16 is rounded to bf16 with an identity gradient: patch_embed / hilbert_projection, text_proj,
the time token, the RMSNorms, the attention projections, project_in / project_out, up_dense, final_norm, final_proj,
final_conv1, final_norm_conv and the activation.  The stream itself is float32 from the position add on, and the
feed-forward (FlaxFeedForward's default float32) and final_conv2 are float32.  The Hilbert input is gathered twice
(hilbert_patchify's order, then __call__'s `x_patches[:, idx]`) and the output goes back through inv_idx once.  In
float64 (gradcheck) nothing is rounded."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as tF

from oracle.dit_ref import gelu_tanh, layernorm
from oracle.unet_ref import conv_same, rms_norm


def _rounder(on: bool):
    if not on:
        return lambda v: v
    return lambda v: v + (v.to(torch.bfloat16).to(v.dtype) - v).detach()


def swish(z):
    return z * torch.sigmoid(z)


def mish(z):
    return z * torch.tanh(tF.softplus(z))


def time_token(P, t, freqs):
    """FourierEmbedding(F) -> TimeProjection(F): Dense, gelu, Dense, gelu, in float32 (common.py:97-124)."""
    arg = t.to(freqs.dtype)[:, None] * (2 * math.pi * freqs)[None, :]
    h = torch.cat([arg.sin(), arg.cos()], -1)
    te = "time_embed/layers_1/DenseGeneral_"
    h = gelu_tanh(h @ P[te + "0/kernel"] + P[te + "0/bias"])
    return gelu_tanh(h @ P[te + "1/kernel"] + P[te + "1/bias"])


def transformer_block(P, name, x, heads, eps, r, use_projection=False, use_self_and_cross=False, norm_inputs=False,
                      explicitly_add_residual=True):
    """TransformerBlock (attention.py:305-380) with only_pure_attention=False and no context: keys and values of
    Attention2 come from the (projected) input."""
    def dense16(v, w):
        return r(r(v) @ r(w))

    def mha(base, xq, ctx):
        d = xq.shape[-1] // heads
        q = r(torch.einsum("blc,chd->blhd", r(xq), r(P[f"{base}/to_q/kernel"])))
        k = r(torch.einsum("blc,chd->blhd", r(ctx), r(P[f"{base}/to_k/kernel"])))
        v = r(torch.einsum("blc,chd->blhd", r(ctx), r(P[f"{base}/to_v/kernel"])))
        w = torch.softmax(torch.einsum("blhd,bkhd->bhlk", q / math.sqrt(d), k), dim=-1)
        o = r(torch.einsum("bhlk,bkhd->blhd", w, v))
        return r(torch.einsum("blhd,hdc->blc", o, r(P[f"{base}/to_out_0/kernel"])))

    pre = f"{name}/Attention"
    if norm_inputs:
        x = r(rms_norm(x, P[f"{name}/RMSNorm_0/scale"], eps))
    px = dense16(x, P[f"{name}/project_in/kernel"]) if use_projection else x
    h = px
    if use_self_and_cross:
        n1 = r(rms_norm(h, P[f"{pre}/norm1/scale"], eps))
        h = h + mha(f"{pre}/Attention1", n1, n1)
    h = h + mha(f"{pre}/Attention2", r(rms_norm(h, P[f"{pre}/norm2/scale"], eps)), px)
    u = r(rms_norm(h, P[f"{pre}/norm3/scale"], eps)) @ P[f"{pre}/ff/net_0/proj/kernel"] + \
        P[f"{pre}/ff/net_0/proj/bias"]
    lin, gate = torch.chunk(u, 2, dim=-1)
    h = h + (lin * gelu_tanh(gate)) @ P[f"{pre}/ff/net_2/kernel"] + P[f"{pre}/ff/net_2/bias"]
    if use_projection:
        h = dense16(h, P[f"{name}/project_out/kernel"])
    return x + h if explicitly_add_residual else h


def uvit_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, *, patch_size: int, num_layers: int,
                 num_heads: int, output_channels: int = 3, norm_epsilon: float = 1e-5, textcontext=None, order=None,
                 use_projection: bool = False, use_self_and_cross: bool = False, norm_inputs: bool = False,
                 explicitly_add_residual: bool = True, add_residualblock_output: bool = False, activation="swish",
                 round_bf16=None):
    """UViT.__call__: x (B, H, W, 3) -> (B, H, W, out).  order: hilbert_indices(HP, WP) under use_hilbert, else None;
    textcontext [B, T, D] or None."""
    dt = P["final_norm/scale"].dtype
    r = _rounder(dt == torch.float32 if round_bf16 is None else round_bf16)
    B, H, W, C = x.shape
    p = patch_size
    HP, WP = H // p, W // p
    N = HP * WP
    F = P["final_norm/scale"].shape[0]
    xin = x.to(dt)
    patches = xin.reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, N, p * p * C)
    if order is None:   # PatchEmbedding: a p x p stride-p conv over (p1, p2, c) patches
        tok = r(r(patches) @ r(P["patch_embed/Conv_0/kernel"].reshape(p * p * C, F)) + P["patch_embed/Conv_0/bias"])
    else:               # hilbert_patchify's gather, hilbert_projection, then __call__'s second gather by idx
        idx = torch.as_tensor(order)
        tok = r(r(patches[:, idx]) @ r(P["hilbert_projection/kernel"]) + P["hilbert_projection/bias"])
        tok = tok[:, idx]
    tok = tok + P["pos_encoding"][:, :N]
    parts = [tok, r(time_token(P, t, freqs))[:, None, :]]
    if textcontext is not None:
        parts.append(r(r(textcontext.to(dt)) @ r(P["text_proj/kernel"]) + P["text_proj/bias"]))
    seq = torch.cat(parts, 1)
    kw = dict(use_projection=use_projection, use_self_and_cross=use_self_and_cross, norm_inputs=norm_inputs,
              explicitly_add_residual=explicitly_add_residual)
    half = num_layers // 2
    skips = []
    for i in range(half):
        seq = transformer_block(P, f"down_block_{i}", seq, num_heads, norm_epsilon, r, **kw)
        skips.append(seq)
    seq = transformer_block(P, "mid_block", seq, num_heads, norm_epsilon, r, **kw)
    for i in range(half):
        cat = torch.cat([seq, skips.pop()], -1)
        seq = r(r(cat) @ r(P[f"up_dense_{i}/kernel"]) + P[f"up_dense_{i}/bias"])
        seq = transformer_block(P, f"up_block_{i}", seq, num_heads, norm_epsilon, r, **kw)
    y = r(layernorm(seq, norm_epsilon, P["final_norm/scale"], P["final_norm/bias"]))[:, :N]
    y = r(r(y) @ r(P["final_proj/kernel"]) + P["final_proj/bias"])
    if order is not None:   # hilbert_unpatchify: row-major k <- sequence inv_idx[k]
        inv = torch.empty(N, dtype=torch.long)
        inv[torch.as_tensor(order)] = torch.arange(N)
        y = y[:, inv]
    img = y.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)
    if not add_residualblock_output:
        return img
    act = mish if activation == "mish" else swish
    z = torch.cat([r(xin), img], -1)
    z = r(conv_same(r(z), r(P["final_conv1/conv/kernel"]), P["final_conv1/conv/bias"]))
    z = r(layernorm(z, norm_epsilon, P["final_norm_conv/scale"], P["final_norm_conv/bias"]))
    z = r(act(z))
    return conv_same(z, P["final_conv2/conv/kernel"], P["final_conv2/conv/bias"])
