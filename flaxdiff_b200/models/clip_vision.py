"""CLIP's vision tower and the image-text pair of the reference's validation metrics (flaxdiff/metrics/images.py:32-112)
on the engine, built from a `transformers` CLIPModel (or its config and state dict) and evaluated forward only.

    patches = prep(samples)         quantise to uint8, PIL bicubic resize,  fdx_clip_image_prep
                                    centre crop, normalise, patchify
    e = patches Wpatch              the patch Conv2d as a GEMM (f32 out)    fdx_gemm
    h = LN_pre([cls; e] + pos)                                              fdx_clip_vision_embed
    CLIPEncoder layers, unmasked attention                                  clip_text.encoder_layers
    image_embeds = LN_post(h[:, 0]) Wvis                                    fdx_clip_pool, fdx_gemm (f32 out)
    text_embeds = last_hidden_state[b, argmax(ids[b])] Wtext                CLIPTextTower, fdx_clip_pool, fdx_gemm
    cos = <a / (|a| + 1e-6), t / (|t| + 1e-6)>                              fdx_clip_similarity

The preprocessing is CLIPImageProcessorPil's (the reference's AutoProcessor(use_fast=False)), computed bit for bit:
the resize tables below restate Pillow's precompute_coeffs / normalize_coeffs_8bpc (Resample.c) for the BICUBIC
filter, and the normalisation table is the processor's f32 arithmetic on each of the 256 levels.  The towers run in
bf16 with f32 accumulation, the embeddings, norms and the cosine in f32.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from .. import ops
from .._lib import FdxError
from .clip_text import _ACTS, CLIPTextTower, _cfg, encoder_layers, layer_entries, pack, state_getter

PRECISION_BITS = 22           # Pillow's 8-bit resample accumulators: 32 - 8 - 2 fraction bits
PIL_BICUBIC = 3               # PIL.Image.Resampling.BICUBIC


def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def axis_coeffs(in_size: int, out_size: int):
    """Pillow's BICUBIC coefficients of one axis resized from in_size to out_size -> (ksize, first [out], count [out],
    taps int32 [out, ksize]) with PRECISION_BITS fraction bits.  The support widens by the scale when downscaling."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    first = np.zeros(out_size, np.int32)
    count = np.zeros(out_size, np.int32)
    taps = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic(((x + xmin) - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        taps[xx, :xmax] = [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
                           for v in w]
        first[xx], count[xx] = xmin, xmax
    return ksize, first, count, taps


def resize_shape(H: int, W: int, shortest_edge: int) -> Tuple[int, int]:
    """transformers' get_resize_output_image_size(default_to_square=False): the short edge becomes shortest_edge, the
    long edge int(shortest_edge * long / short)."""
    short, long = (W, H) if W <= H else (H, W)
    new_long = int(shortest_edge * long / short)
    return (new_long, shortest_edge) if W <= H else (shortest_edge, new_long)


def crop_tables(H: int, W: int, shortest_edge: int, crop: int) -> Tuple[np.ndarray, int, int]:
    """fdx_clip_image_prep's int32 tables for [H, W] images: the crop window's output rows, then its columns, each
    [first, count, taps...].  An axis PIL leaves alone (same size) gets one tap of 1.0 -> (tables, ksize_y,
    ksize_x)."""
    parts, ks = [], []
    for n_in, n_out in zip((H, W), resize_shape(H, W, shortest_edge)):
        off = (n_out - crop) // 2
        idx = np.arange(off, off + crop)
        if n_out == n_in:
            k, first, count, taps = 1, idx.astype(np.int32), np.ones(crop, np.int32), \
                np.full((crop, 1), 1 << PRECISION_BITS, np.int32)
        else:
            k, first, count, taps = axis_coeffs(n_in, n_out)
            first, count, taps = first[idx], count[idx], taps[idx]
        parts.append(np.concatenate([first[:, None], count[:, None], taps], axis=1).reshape(-1))
        ks.append(k)
    return np.concatenate(parts).astype(np.int32), ks[0], ks[1]


def normalise_lut(rescale_factor: float, mean, std) -> np.ndarray:
    """f32 [3, 256]: CLIPImageProcessorPil's rescale (uint8 -> float64 * factor -> f32) and normalise ((x - mean) /
    std in f32) of every level of every channel."""
    x = (np.arange(256, dtype=np.float64) * rescale_factor).astype(np.float32)
    m, s = np.asarray(mean, np.float32), np.asarray(std, np.float32)
    return ((x[None, :] - m[:, None]) / s[:, None]).astype(np.float32)


class CLIPVisionTower:
    """Frozen CLIP vision transformer.  `config` is a transformers CLIPVisionConfig (or a dict with its fields),
    `state_dict` the CLIPVisionModel's (keys with or without the `vision_model.` prefix).  encode() takes the patch
    matrix of fdx_clip_image_prep and returns the pooled output (post_layernorm of the class token), bf16 [B, D]."""

    def __init__(self, config, state_dict: Dict[str, torch.Tensor], device=None):
        self.D = int(_cfg(config, "hidden_size"))
        self.inner = int(_cfg(config, "intermediate_size"))
        self.layers = int(_cfg(config, "num_hidden_layers"))
        self.heads = int(_cfg(config, "num_attention_heads"))
        self.eps = float(_cfg(config, "layer_norm_eps"))
        self.image_size = int(_cfg(config, "image_size"))
        self.patch = int(_cfg(config, "patch_size"))
        act = _cfg(config, "hidden_act")
        if act not in _ACTS:
            raise FdxError(f"CLIPVisionTower: hidden_act {act!r} is not supported (quick_gelu or gelu)")
        self.act = _ACTS[act]
        if int(_cfg(config, "num_channels")) != 3:
            raise FdxError(f"CLIPVisionTower: num_channels {_cfg(config, 'num_channels')} is not supported (3)")
        if self.D % self.heads or self.D // self.heads not in (32, 64, 128):
            raise FdxError(f"CLIPVisionTower: head width {self.D / self.heads:g} (hidden_size {self.D} / "
                           f"{self.heads} heads) must be 32, 64 or 128")
        if self.D % 64 or self.D > 1280:
            raise FdxError(f"CLIPVisionTower: hidden_size {self.D} must be a multiple of 64, <= 1280")
        if self.inner % 64:
            raise FdxError(f"CLIPVisionTower: intermediate_size {self.inner} must be a multiple of 64")
        if self.patch <= 0 or self.image_size % self.patch:
            raise FdxError(f"CLIPVisionTower: image_size {self.image_size} is not a multiple of patch_size "
                           f"{self.patch}")
        self.G = self.image_size // self.patch
        self.K = 3 * self.patch * self.patch          # one patch row, (c, ky, kx) as the conv weight stores it
        self.ld = (self.K + 7) // 8 * 8               # row stride of the patch matrix: TMA needs 16-byte rows
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._pack({k[len("vision_model."):] if k.startswith("vision_model.") else k: v for k, v in state_dict.items()})

    def _pack(self, sd: Dict[str, torch.Tensor]) -> None:
        get = state_getter(sd, "CLIPVisionTower")
        D, p = self.D, self.patch
        entries = [("wpatch", get("embeddings.patch_embedding.weight", (D, 3, p, p)).reshape(D, self.K).t(),
                    torch.bfloat16),
                   ("cls", get("embeddings.class_embedding", (D,)), torch.float32),
                   ("pos", get("embeddings.position_embedding.weight", (self.G * self.G + 1, D)), torch.float32),
                   ("pre_g", get("pre_layrnorm.weight", (D,)), torch.float32),
                   ("pre_b", get("pre_layrnorm.bias", (D,)), torch.float32)]
        entries += layer_entries(get, self.layers, D, self.inner)
        entries += [("post_g", get("post_layernorm.weight", (D,)), torch.float32),
                    ("post_b", get("post_layernorm.bias", (D,)), torch.float32)]
        self.buffer, self.w = pack(entries, self.device)

    def encode(self, patches: torch.Tensor) -> torch.Tensor:
        """pooler_output bf16 [B, D] of the bf16 patch matrix [B * G^2, ld]."""
        rows = patches.shape[0]
        B = rows // (self.G * self.G)
        if rows != B * self.G * self.G or patches.shape[1] != self.ld:
            raise FdxError(f"CLIPVisionTower: patch matrix {tuple(patches.shape)} is not [B * {self.G * self.G}, "
                           f"{self.ld}]")
        w = self.w
        e = ops.linear_fwd(patches[:, :self.K], w["wpatch"], out_dtype=torch.float32)
        h = ops.clip_vision_embed(e, B, w["cls"], w["pos"], w["pre_g"], w["pre_b"], self.eps)
        encoder_layers(h, w, self.layers, self.heads, self.inner, self.eps, self.act)
        return ops.clip_pool(h, None, w["post_g"], w["post_b"], self.eps)


def _proc(processor, name):
    return processor[name] if isinstance(processor, dict) else getattr(processor, name)


class CLIPPair:
    """Both towers of a CLIPModel, its two projections and the preprocessing of its CLIPImageProcessorPil (or a dict
    with the processor's fields).  image_embeds / text_embeds are CLIPModel's image_embeds / text_embeds (f32, not
    normalised); similarity() the cosine of the reference's metrics and both of their batch means."""

    def __init__(self, config, state_dict: Dict[str, torch.Tensor], processor, device=None):
        tcfg, vcfg = _cfg(config, "text_config"), _cfg(config, "vision_config")
        self.P = int(_cfg(config, "projection_dim"))
        if self.P % 32:
            raise FdxError(f"CLIPPair: projection_dim {self.P} must be a multiple of 32")
        if _proc(processor, "resample") != PIL_BICUBIC:
            raise FdxError(f"CLIPPair: processor resample {_proc(processor, 'resample')!r} is not BICUBIC")
        for flag in ("do_resize", "do_center_crop", "do_rescale", "do_normalize"):
            if not _proc(processor, flag):
                raise FdxError(f"CLIPPair: the processor's {flag} is off; the engine's preprocessing always does it")
        size, crop = _proc(processor, "size"), _proc(processor, "crop_size")
        self.shortest_edge, self.crop = int(size["shortest_edge"] or 0), int(crop["height"] or 0)
        if int(crop["width"] or 0) != self.crop or self.crop <= 0 or self.shortest_edge < self.crop:
            raise FdxError(f"CLIPPair: crop {dict(crop)} must be square and fit the resized short edge "
                           f"{self.shortest_edge}")
        if self.crop != int(_cfg(vcfg, "image_size")):
            raise FdxError(f"CLIPPair: processor crop {self.crop} differs from the vision tower's image_size "
                           f"{_cfg(vcfg, 'image_size')}")
        self.vision = CLIPVisionTower(vcfg, state_dict, device)
        self.device = self.vision.device
        self.text = CLIPTextTower(tcfg, state_dict, self.device)
        get = state_getter(state_dict, "CLIPPair")
        self.buffer, self.w = pack(
            [("vproj", get("visual_projection.weight", (self.P, self.vision.D)).t(), torch.bfloat16),
             ("tproj", get("text_projection.weight", (self.P, self.text.D)).t(), torch.bfloat16),
             ("lut", torch.from_numpy(normalise_lut(float(_proc(processor, "rescale_factor")),
                                                    _proc(processor, "image_mean"), _proc(processor, "image_std"))),
              torch.float32)], self.device)
        self._tables: Dict[Tuple[int, int], Tuple[torch.Tensor, int, int]] = {}

    @staticmethod
    def from_transformers(model, processor, device=None) -> "CLIPPair":
        return CLIPPair(model.config, model.state_dict(), processor, device)

    def _prep_tables(self, H: int, W: int):
        """Resize tables of one input shape, built on the host and copied to the device once."""
        if (H, W) not in self._tables:
            tab, ky, kx = crop_tables(H, W, self.shortest_edge, self.crop)
            self._tables[(H, W)] = (torch.from_numpy(tab).to(self.device), ky, kx)
        return self._tables[(H, W)]

    def preprocess(self, samples: torch.Tensor, u8_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """bf16 patch matrix [B * G^2, ld] of f32 samples [B, H, W, 3] in [-1, 1] (out-of-range values clamp, NaN
        counts as -1); u8_out uint8 [B, crop, crop, 3] receives the processor's uint8 image."""
        if samples.dim() != 4 or samples.shape[-1] != 3:
            raise FdxError(f"CLIPPair: samples must be [B, H, W, 3], got {tuple(samples.shape)}")
        x = samples.to(self.device, torch.float32).contiguous()
        tab, ky, kx = self._prep_tables(x.shape[1], x.shape[2])
        return ops.clip_image_prep(x, tab, ky, kx, self.w["lut"], self.crop, self.vision.patch, self.vision.ld,
                                   u8_out)

    def image_embeds(self, samples: torch.Tensor) -> torch.Tensor:
        """f32 [B, P] image embeddings of samples [B, H, W, 3] in [-1, 1]."""
        return ops.linear_fwd(self.vision.encode(self.preprocess(samples)), self.w["vproj"], out_dtype=torch.float32)

    def text_embeds(self, ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """f32 [B, P] text embeddings of token ids [B, T]: the final-LayerNorm row at argmax(ids), projected."""
        ids = ids.to(self.device, torch.int32).contiguous()
        pooled = ops.clip_pool(self.text.encode(ids, attention_mask), ids)
        return ops.linear_fwd(pooled, self.w["tproj"], out_dtype=torch.float32)

    def similarity(self, samples, ids, attention_mask=None):
        """-> (cos f32 [B], f32 [2] = (clip_similarity = mean(1 - cos), clip_score = mean(100 max(cos, 0))))."""
        img = self.image_embeds(samples)
        txt = self.text_embeds(ids, attention_mask)
        if img.shape[0] != txt.shape[0]:
            raise FdxError(f"CLIPPair: {img.shape[0]} samples but {txt.shape[0]} token sequences")
        return ops.clip_similarity(img, txt)
