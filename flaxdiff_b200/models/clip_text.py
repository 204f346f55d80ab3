"""The CLIP text tower on the engine: the FlaxCLIPTextModel that the reference's text-conditioned trainer runs in bf16
inside its jitted train_step (flaxdiff/inputs/encoders.py, trainer/general_diffusion_trainer.py:266-275), built from
a `transformers` CLIPTextModel (or its config and state dict) and evaluated forward only: the tower is frozen.

    h = bf16(tok[ids] + pos)                                   fdx_token_embed
    per layer:
      x = LN1(h);  qkv = x Wqkv + bqkv                         fdx_layernorm_fwd, fdx_gemm (bias epilogue)
      o = attention(q, k, v), causal + attention_mask          fdx_attention_fwd_masked (q, k, v: ld = 3D views)
      h = o Wo + bo + h                                        fdx_gemm (bias + residual epilogue)
      x = LN2(h);  u = act(x W1 + b1)                          fdx_layernorm_fwd, fdx_gemm, fdx_bias_act
      h = u W2 + b2 + h                                        fdx_gemm (bias + residual epilogue)
    last_hidden_state = LN_final(h)                            bf16 [B, T, D]

The hidden state between layers is bf16, as in the reference's bf16 tower; the weights live in one device buffer:
linear kernels bf16 in the (in, out) layout of flax Dense, LayerNorm parameters, biases and embedding tables f32.
Every kernel computes each sequence on its own, so a sequence encodes to the same bits alone or inside any batch.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from .. import ops
from .._lib import ACT_GELU, ACT_QUICK_GELU, FdxError

_ACTS = {"quick_gelu": ACT_QUICK_GELU, "gelu": ACT_GELU}
_ALIGN = 256                  # byte alignment of every tensor inside the packed weight buffer


def _cfg(config, name):
    return config[name] if isinstance(config, dict) else getattr(config, name)


class CLIPTextTower:
    """Frozen CLIP text tower.  `config` is a transformers CLIPTextConfig (or a dict with its fields), `state_dict`
    the CLIPTextModel's (keys with or without the `text_model.` prefix).  `seq_len` = the token length the tower
    is used at (the tokenizer's model_max_length, 77 for CLIP)."""

    def __init__(self, config, state_dict: Dict[str, torch.Tensor], device=None, seq_len: Optional[int] = None):
        self.D = int(_cfg(config, "hidden_size"))
        self.inner = int(_cfg(config, "intermediate_size"))
        self.layers = int(_cfg(config, "num_hidden_layers"))
        self.heads = int(_cfg(config, "num_attention_heads"))
        self.max_pos = int(_cfg(config, "max_position_embeddings"))
        self.vocab = int(_cfg(config, "vocab_size"))
        self.eps = float(_cfg(config, "layer_norm_eps"))
        self.seq_len = self.max_pos if seq_len is None else int(seq_len)
        act = _cfg(config, "hidden_act")
        if act not in _ACTS:
            raise FdxError(f"CLIPTextTower: hidden_act {act!r} is not supported (quick_gelu or gelu)")
        self.act = _ACTS[act]
        if self.D % self.heads or self.D // self.heads not in (32, 64):
            raise FdxError(f"CLIPTextTower: head width {self.D / self.heads:g} (hidden_size {self.D} / "
                           f"{self.heads} heads) must be 32 or 64")
        if self.D % 64 or self.D > 1280:
            raise FdxError(f"CLIPTextTower: hidden_size {self.D} must be a multiple of 64, <= 1280")
        if self.inner % 64:
            raise FdxError(f"CLIPTextTower: intermediate_size {self.inner} must be a multiple of 64")
        if not 0 < self.seq_len <= self.max_pos:
            raise FdxError(f"CLIPTextTower: sequence length {self.seq_len} exceeds max_position_embeddings "
                           f"{self.max_pos}")
        self.dh = self.D // self.heads
        self.scale = 1.0 / math.sqrt(self.dh)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._pack({k[len("text_model."):] if k.startswith("text_model.") else k: v for k, v in state_dict.items()})

    @staticmethod
    def from_transformers(model, device=None, seq_len: Optional[int] = None) -> "CLIPTextTower":
        return CLIPTextTower(model.config, model.state_dict(), device, seq_len)

    # ------------------------------------------------------------------ weights
    def _pack(self, sd: Dict[str, torch.Tensor]) -> None:
        get = state_getter(sd, "CLIPTextTower")
        D = self.D
        entries = [("tok", get("embeddings.token_embedding.weight", (self.vocab, D)), torch.float32),
                   ("pos", get("embeddings.position_embedding.weight", (self.max_pos, D)), torch.float32)]
        entries += layer_entries(get, self.layers, D, self.inner)
        entries += [("lnf_g", get("final_layer_norm.weight", (D,)), torch.float32),
                    ("lnf_b", get("final_layer_norm.bias", (D,)), torch.float32)]
        self.buffer, self.w = pack(entries, self.device)

    # ------------------------------------------------------------------ forward
    def encode(self, ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """last_hidden_state bf16 [B, T, D] of token ids [B, T] (attention_mask [B, T] of 0 / 1, or None)."""
        if ids.dim() != 2:
            raise FdxError(f"CLIPTextTower: ids must be [B, T], got {tuple(ids.shape)}")
        B, T = ids.shape
        if T > self.max_pos:
            raise FdxError(f"CLIPTextTower: sequence length {T} exceeds max_position_embeddings {self.max_pos}")
        ids = ids.to(self.device, torch.int32).contiguous()
        mask = None
        if attention_mask is not None:
            if tuple(attention_mask.shape) != (B, T):
                raise FdxError(f"CLIPTextTower: attention_mask {tuple(attention_mask.shape)} does not match ids")
            mask = attention_mask.to(self.device, torch.int32).contiguous()
        h = ops.token_embed(ids, self.w["tok"], self.w["pos"])
        encoder_layers(h, self.w, self.layers, self.heads, self.inner, self.eps, self.act, causal=True, key_mask=mask)
        if out is None:
            out = torch.empty((B, T, self.D), dtype=torch.bfloat16, device=self.device)
        return ops.layernorm_fwd(h, self.w["lnf_g"], self.w["lnf_b"], self.eps, out=out)


def state_getter(sd: Dict[str, torch.Tensor], who: str):
    """get(name, shape) -> the f32 CPU copy of sd[name], or FdxError when it is missing or has another shape."""
    def get(name, shape):
        if name not in sd:
            raise FdxError(f"{who}: state dict has no {name!r}")
        t = sd[name].detach().to("cpu", torch.float32)
        if tuple(t.shape) != tuple(shape):
            raise FdxError(f"{who}: {name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
        return t
    return get


def layer_entries(get, layers: int, D: int, I: int):
    """The packed weights of CLIPEncoder's layers (shared by the text and vision towers): linear kernels bf16 in the
    (in, out) layout, q / k / v fused into one [D, 3D] kernel; LayerNorm parameters and biases f32."""
    entries = []
    for i in range(layers):
        p = f"encoder.layers.{i}."
        wq, wk, wv = (get(p + f"self_attn.{n}_proj.weight", (D, D)) for n in "qkv")
        bq, bk, bv = (get(p + f"self_attn.{n}_proj.bias", (D,)) for n in "qkv")
        entries += [
            (f"{i}.ln1_g", get(p + "layer_norm1.weight", (D,)), torch.float32),
            (f"{i}.ln1_b", get(p + "layer_norm1.bias", (D,)), torch.float32),
            (f"{i}.wqkv", torch.cat([wq.t(), wk.t(), wv.t()], dim=1), torch.bfloat16),
            (f"{i}.bqkv", torch.cat([bq, bk, bv]), torch.float32),
            (f"{i}.wo", get(p + "self_attn.out_proj.weight", (D, D)).t(), torch.bfloat16),
            (f"{i}.bo", get(p + "self_attn.out_proj.bias", (D,)), torch.float32),
            (f"{i}.ln2_g", get(p + "layer_norm2.weight", (D,)), torch.float32),
            (f"{i}.ln2_b", get(p + "layer_norm2.bias", (D,)), torch.float32),
            (f"{i}.w1", get(p + "mlp.fc1.weight", (I, D)).t(), torch.bfloat16),
            (f"{i}.b1", get(p + "mlp.fc1.bias", (I,)), torch.float32),
            (f"{i}.w2", get(p + "mlp.fc2.weight", (D, I)).t(), torch.bfloat16),
            (f"{i}.b2", get(p + "mlp.fc2.bias", (D,)), torch.float32)]
    return entries


def pack(entries, device):
    """One device buffer holding every (name, tensor, dtype) entry at a 256-byte aligned offset -> (buffer, {name:
    view})."""
    offsets, total = [], 0
    for _, t, dt in entries:
        offsets.append(total)
        nbytes = t.numel() * (2 if dt == torch.bfloat16 else 4)
        total += (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
    host = torch.zeros(total, dtype=torch.uint8)
    for (_, t, dt), off in zip(entries, offsets):
        b = t.to(dt).contiguous().view(torch.uint8).reshape(-1)
        host[off:off + b.numel()] = b
    buffer = host.to(device)
    w = {}
    for (name, t, dt), off in zip(entries, offsets):
        n = t.numel() * (2 if dt == torch.bfloat16 else 4)
        w[name] = buffer[off:off + n].view(dt).view(tuple(t.shape))
    return buffer, w


def encoder_layers(h: torch.Tensor, w, layers: int, heads: int, inner: int, eps: float, act: int,
                   causal: bool = False, key_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """CLIPEncoder's pre-LN layers over the bf16 hidden state h [B, T, D], in place.  The text tower's attention is
    causal under its attention mask (fdx_attention_fwd_masked), the vision tower's attends to every token
    (fdx_attention_fwd)."""
    B, T, D = h.shape
    dh = D // heads
    scale = 1.0 / math.sqrt(dh)
    h2 = h.view(B * T, D)
    x = torch.empty((B * T, D), dtype=torch.bfloat16, device=h.device)
    qkv = torch.empty((B, T, 3 * D), dtype=torch.bfloat16, device=h.device)
    o = torch.empty((B, T, D), dtype=torch.bfloat16, device=h.device)
    u = torch.empty((B * T, inner), dtype=torch.bfloat16, device=h.device)
    masked = causal or key_mask is not None
    for i in range(layers):
        ops.layernorm_fwd(h2, w[f"{i}.ln1_g"], w[f"{i}.ln1_b"], eps, out=x)
        ops.linear_fwd(x, w[f"{i}.wqkv"], out=qkv.view(B * T, 3 * D), bias=w[f"{i}.bqkv"])
        q, k, v = qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]
        if masked:
            ops.attention_fwd_masked(q, k, v, heads, dh, scale, causal, key_mask, out=o)
        else:
            ops.attention_fwd(q, k, v, heads, dh, scale, out=o)
        ops.linear_fwd(o.view(B * T, D), w[f"{i}.wo"], out=h2, bias=w[f"{i}.bo"], res=h2)
        ops.layernorm_fwd(h2, w[f"{i}.ln2_g"], w[f"{i}.ln2_b"], eps, out=x)
        ops.linear_fwd(x, w[f"{i}.w1"], out=u)
        ops.bias_act(u, w[f"{i}.b1"], act, out=u)
        ops.linear_fwd(u, w[f"{i}.w2"], out=h2, bias=w[f"{i}.b2"], res=h2)
    return h
