"""References of the CLIP metrics' pieces (csrc/fdx_clip.cu, models/clip_vision.py, flaxdiff_b200/metrics): PIL's
8-bit two-pass resize restated in numpy from the engine's tables, float64 references of the embedding, pooling and
cosine kernels with the first-order error bound `delta` of their f32 arithmetic (the tolerance model of
tests/elementwise_ref.py), and the seeded random CLIP models the tests build."""
from __future__ import annotations

import math

import numpy as np
import torch

from clip_text_ref import layernorm_ref
from elementwise_ref import U32, gamma
from flaxdiff_b200.models.clip_vision import PRECISION_BITS, axis_coeffs, resize_shape


# ----------------------------------------------------------------------------------------------- preprocessing
def quantise_np(x: np.ndarray) -> np.ndarray:
    """uint8(((x + 1) / 2) * 255) in f32, clamped to [0, 255], NaN -> 0."""
    t = ((x.astype(np.float32) + np.float32(1)) / np.float32(2)) * np.float32(255)
    t = np.where(np.isnan(t), np.float32(0), t)
    return np.clip(t, 0, 255).astype(np.uint8)


def _pass(img: np.ndarray, axis: int, n_out: int) -> np.ndarray:
    _, first, count, taps = axis_coeffs(img.shape[axis], n_out)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((n_out,) + src.shape[1:], np.int64)
    for i in range(n_out):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for t in range(count[i]):
            acc += src[first[i] + t] * int(taps[i, t])
        out[i] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis).astype(np.uint8)


def pil_resize_np(u8: np.ndarray, new_h: int, new_w: int) -> np.ndarray:
    """Image.resize((new_w, new_h), BICUBIC) of a uint8 [H, W, 3] image: the horizontal pass, then the vertical one,
    each clipped to uint8, a pass skipped where its axis keeps its size (Resample.c's ImagingResampleInner)."""
    out = u8
    if new_w != u8.shape[1]:
        out = _pass(out, 1, new_w)
    if new_h != u8.shape[0]:
        out = _pass(out, 0, new_h)
    return out


def processor_u8(u8: np.ndarray, shortest_edge: int = 224, crop: int = 224) -> np.ndarray:
    """CLIPImageProcessorPil's resized and centre-cropped uint8 image, restated with pil_resize_np."""
    H, W, _ = u8.shape
    nh, nw = resize_shape(H, W, shortest_edge)
    r = pil_resize_np(u8, nh, nw)
    top, left = (nh - crop) // 2, (nw - crop) // 2
    return r[top:top + crop, left:left + crop]


def patchify(pixel_values: torch.Tensor, p: int) -> torch.Tensor:
    """[B, 3, S, S] -> [B * (S / p)^2, 3 p p] rows in the (c, ky, kx) order of the patch conv weight."""
    B, C, S, _ = pixel_values.shape
    G = S // p
    return pixel_values.reshape(B, C, G, p, G, p).permute(0, 2, 4, 1, 3, 5).reshape(B * G * G, C * p * p)


# ----------------------------------------------------------------------------------------------- kernels, float64
def vision_embed_ref(patch, cls, pos, g, b, eps):
    """LN([cls; patch] + pos) per image -> (value, delta): one f32 addition before layernorm_ref's bound."""
    B = patch.shape[0] // (pos.shape[0] - 1)
    x = torch.cat([cls.view(1, 1, -1).expand(B, 1, -1), patch.view(B, pos.shape[0] - 1, -1)], 1) + pos.unsqueeze(0)
    y, d = layernorm_ref(x, g, b, eps)
    rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + eps)
    return y, d + g.abs() * rstd * U32 * 2 * x.abs().amax(-1, keepdim=True)


def pool_rows(ids, B):
    """Row 0, or the first position of each sequence's largest id."""
    if ids is None:
        return torch.zeros(B, dtype=torch.long, device="cpu")
    return ids.long().cpu().argmax(1)


def similarity_ref(img, txt):
    """cos [B], mean(1 - cos), mean(100 max(cos, 0)) in float64 -> (cos, out2, delta_cos, delta_out2).  The three
    sums over P are lane-serial fmas and a 5-level warp tree (depth P / 32 + 5); two square roots, + 1e-6 and two
    divisions add 5u relative.  The means: depth B / 32 + 5 additions of terms each carrying their own cos error."""
    B, P = img.shape
    na, nt = img.norm(dim=1), txt.norm(dim=1)
    dot = (img * txt).sum(1)
    cos = dot / (na + 1e-6) / (nt + 1e-6)
    gs = gamma(math.ceil(P / 32) + 5)
    abs_dot = (img.abs() * txt.abs()).sum(1) / (na + 1e-6) / (nt + 1e-6)
    d_cos = gs * abs_dot + (gs + 6 * U32) * cos.abs()
    out2 = torch.stack([(1 - cos).mean(), (100 * cos.clamp_min(0)).mean()])
    gm = gamma(math.ceil(B / 32) + 6)
    d2 = torch.stack([d_cos.mean() + gm * (1 + cos.abs()).mean() + U32,
                      100 * d_cos.mean() + gm * (100 * cos.clamp_min(0)).mean() + 100 * U32 * cos.abs().mean()])
    return cos, out2, d_cos, d2


# ----------------------------------------------------------------------------------------------- models
def clip_pair_config(kind: str):
    """Seeded CLIPConfigs: a tiny pair (p = 14 on 224^2, two heads of 32 / 64), and CLIP ViT-L/14's shape (1024
    wide, 24 layers, 16 heads, p = 14; the 768-wide 12-layer text tower; 768 projection).  eos_token_id = 2 makes
    transformers pool the argmax(input_ids) row, as FlaxCLIP does."""
    from transformers import CLIPConfig
    if kind == "tiny":
        text = dict(vocab_size=1000, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
                    max_position_embeddings=77, eos_token_id=2)
        vision = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
                      image_size=224, patch_size=14)
        return CLIPConfig(text_config=text, vision_config=vision, projection_dim=64)
    if kind == "vit-l":
        text = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                    num_attention_heads=12, max_position_embeddings=77, eos_token_id=2)
        vision = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                      image_size=224, patch_size=14)
        return CLIPConfig(text_config=text, vision_config=vision, projection_dim=768)
    raise ValueError(kind)


def clip_pair_model(kind: str, seed: int = 0):
    """transformers' CLIPModel with random weights (CPU, fp32, eager attention)."""
    from transformers import CLIPModel
    torch.manual_seed(seed)
    cfg = clip_pair_config(kind)
    cfg._attn_implementation = "eager"
    cfg.text_config._attn_implementation = "eager"
    cfg.vision_config._attn_implementation = "eager"
    return CLIPModel(cfg).eval()


def save_tiny(path, seed: int = 0) -> str:
    """A tiny CLIPModel and a default CLIPImageProcessorPil saved under `path` (a local model directory)."""
    from transformers.models.clip import CLIPImageProcessorPil
    clip_pair_model("tiny", seed).save_pretrained(str(path))
    CLIPImageProcessorPil().save_pretrained(str(path))
    return str(path)


def metric_ref(model, processor, samples: np.ndarray, ids, mask):
    """flaxdiff/metrics/images.py:32-112 in torch fp32: quantise, CLIPImageProcessorPil, CLIPModel, the cosine with
    1e-6 added to the norms -> (clip_similarity, clip_score, cos)."""
    u8 = (((samples + np.float32(1)) / np.float32(2)) * np.float32(255)).astype(np.uint8)
    pv = processor(images=list(u8), return_tensors="pt")["pixel_values"]
    with torch.no_grad():
        out = model(pixel_values=pv, input_ids=ids, attention_mask=mask)
    a = out.image_embeds / (out.image_embeds.norm(dim=-1, keepdim=True) + 1e-6)
    t = out.text_embeds / (out.text_embeds.norm(dim=-1, keepdim=True) + 1e-6)
    cos = (a * t).sum(-1)
    return float((1 - cos).mean()), float((100 * cos.clamp_min(0)).mean()), cos
