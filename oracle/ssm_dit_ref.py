"""fp32 CPU restatement of the reference's hybrid SSM-attention DiT (flaxdiff/models/ssm_dit.py) in plain torch, from
the formulas of its modules: S5Layer, BidirectionalS5Layer, SSMDiTBlock and HybridSSMAttentionDiT.  The S5 layer uses
complex tensors and an explicit sequential recurrence; torch's complex autograd gives the gradients of its real
parameters.  The attention blocks and the shared stem come from oracle/dit_ref.py.  Parameters are a dict of flax names
-> tensors, as in dit_ref."""
from __future__ import annotations

import math

import torch

from oracle import dit_ref


def s5_layer(P, base, u: torch.Tensor) -> torch.Tensor:
    """S5Layer.__call__ (ssm_dit.py:85-218) on u [B, L, F]: ZOH discretisation of A = -exp(log_A_real) + i A_imag
    with dt = exp(log_dt), then x_k = Abar x_{k-1} + Bbar u_k from x_{-1} = 0 and y_k = Re(C x_k) + D u_k.  Computes in
    u's precision (complex64 for f32, complex128 for f64)."""
    cdt = torch.complex128 if u.dtype == torch.float64 else torch.complex64
    dt = torch.exp(P[base + "/log_dt"])
    A = torch.complex(-torch.exp(P[base + "/log_A_real"]), P[base + "/A_imag"])
    Ab = torch.exp(A * dt)
    Bb = ((Ab - 1.0) / (A + 1e-8))[:, None] * torch.complex(P[base + "/B_re"], P[base + "/B_im"])
    C = torch.complex(P[base + "/C_re"], P[base + "/C_im"])
    Bu = torch.einsum("blf,nf->bln", u.to(cdt), Bb)
    h = torch.zeros(u.shape[0], Ab.shape[0], dtype=cdt)
    xs = []
    for k in range(u.shape[1]):
        h = Ab * h + Bu[:, k]
        xs.append(h)
    X = torch.stack(xs, 1)
    return torch.einsum("fn,bln->blf", C, X).real + P[base + "/D"] * u


def ssm(P, name, u: torch.Tensor, bidirectional: bool) -> torch.Tensor:
    """BidirectionalS5Layer (ssm_dit.py:243-286): the forward layer on u, the backward layer on u reversed in token
    order (its output reversed back), concatenated and projected by out_proj; or the single S5Layer."""
    if not bidirectional:
        return s5_layer(P, f"{name}/ssm", u)
    yf = s5_layer(P, f"{name}/ssm/s5_forward", u)
    yb = s5_layer(P, f"{name}/ssm/s5_backward", u.flip(1)).flip(1)
    return dit_ref.dense(P, f"{name}/ssm/out_proj", torch.cat([yf, yb], -1))


def ssm_block(P, name, x, cond, eps, bidirectional: bool):
    """SSMDiTBlock.__call__ (ssm_dit.py:504-538): DiTBlock's adaLN / gate / MLP skeleton with the S5 layer in place
    of the attention."""
    ada = dit_ref.dense(P, f"{name}/ada_params_module/ada_proj", cond)[:, None, :]
    sc_m, sh_m, g_m, sc_a, sh_a, g_a = ada.chunk(6, -1)
    x = x + g_a * ssm(P, name, dit_ref.layernorm(x, eps) * (1 + sc_a) + sh_a, bidirectional)
    h = dit_ref.layernorm(x, eps) * (1 + sc_m) + sh_m
    h = dit_ref.dense(P, f"{name}/mlp/layers_2", dit_ref.gelu_tanh(dit_ref.dense(P, f"{name}/mlp/layers_0", h)))
    return x + g_m * h


def dit_block_without_rope(P, name, x, cond, heads, eps):
    """DiTBlock under the Hilbert / zigzag orders, where the reference passes cos = 1, sin = 0 (ssm_dit.py:756-759):
    dit_ref.dit_block with the rotation left out."""
    ada = dit_ref.dense(P, f"{name}/ada_params_module/ada_proj", cond)[:, None, :]
    sc_m, sh_m, g_m, sc_a, sh_a, g_a = ada.chunk(6, -1)
    h = dit_ref.layernorm(x, eps) * (1 + sc_a) + sh_a
    B, L, F = h.shape
    base = f"{name}/attention"
    q = torch.einsum("blf,fhd->blhd", h, P[base + "/to_q/kernel"]) + P[base + "/to_q/bias"]
    k = torch.einsum("blf,fhd->blhd", h, P[base + "/to_k/kernel"]) + P[base + "/to_k/bias"]
    v = torch.einsum("blf,fhd->blhd", h, P[base + "/to_v/kernel"]) + P[base + "/to_v/bias"]
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(F // heads)
    o = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v)
    x = x + g_a * (torch.einsum("blhd,hdf->blf", o, P[base + "/to_out_0/kernel"]) + P[base + "/to_out_0/bias"])
    h = dit_ref.layernorm(x, eps) * (1 + sc_m) + sh_m
    h = dit_ref.dense(P, f"{name}/mlp/layers_2", dit_ref.gelu_tanh(dit_ref.dense(P, f"{name}/mlp/layers_0", h)))
    return x + g_m * h


def hybrid_forward(P, x: torch.Tensor, t: torch.Tensor, freqs: torch.Tensor, *, patch_size: int, pattern, num_heads: int,
                   output_channels: int = 3, norm_epsilon: float = 1e-5, textcontext=None, order=None,
                   bidirectional: bool = True):
    """HybridSSMAttentionDiT.__call__ (ssm_dit.py:700-779): x (B, H, W, C) f32 -> (B, H, W, out) f32.  `order` is the
    patch order as row-major patch indices (the Hilbert / zigzag table; None = raster): the patch rows and the sin-cos
    table follow it, hilbert_projection embeds the patches, RoPE is off, and the output rows go back to raster order."""
    B, H, W, C = x.shape
    p = patch_size
    HP, WP = H // p, W // p
    patches = x.reshape(B, HP, p, WP, p, C).permute(0, 1, 3, 2, 4, 5).reshape(B, HP * WP, p * p * C)
    pos = torch.from_numpy(dit_ref.sincos_2d(P["final_norm/scale"].shape[0], HP, WP))
    if order is None:
        tok = patches @ P["patch_embed/Conv_0/kernel"].reshape(p * p * C, -1) + P["patch_embed/Conv_0/bias"]
    else:
        idx = torch.as_tensor(order, dtype=torch.long)
        patches, pos = patches[:, idx], pos[idx]
        tok = dit_ref.dense(P, "hilbert_projection", patches)
    tok = tok + pos[None].to(tok.dtype)
    cond = dit_ref.time_embed(P, t, freqs)
    if textcontext is not None:
        cond = cond + dit_ref.dense(P, "text_context_proj", textcontext.float()).mean(1)
    for i, kind in enumerate(pattern):
        if kind == "ssm":
            tok = ssm_block(P, f"ssm_block_{i}", tok, cond, norm_epsilon, bidirectional)
        elif order is None:
            tok = dit_ref.dit_block(P, f"dit_block_{i}", tok, cond, num_heads, norm_epsilon)
        else:
            tok = dit_block_without_rope(P, f"dit_block_{i}", tok, cond, num_heads, norm_epsilon)
    out = dit_ref.layernorm(tok, norm_epsilon, P["final_norm/scale"], P["final_norm/bias"])
    out = dit_ref.dense(P, "final_proj", out)[..., :p * p * output_channels]
    if order is not None:
        inv = torch.empty_like(idx)
        inv[idx] = torch.arange(idx.numel())
        out = out[:, inv]
    return out.reshape(B, HP, WP, p, p, output_channels).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, output_channels)
