"""CLIP metrics of generated images against their prompts (flaxdiff/metrics/images.py:32-112), computed on the
engine: CLIPImageProcessorPil's preprocessing, both CLIP towers, the projections and the cosine run as libfdx kernels
(models/clip_vision.py).

Samples are quantised as the reference does, uint8(((x + 1) / 2) * 255) in f32 with truncation; values the samplers'
clipping would never produce are defined here: the result clamps to [0, 255] and NaN maps to 0.  The prompts'
embedding is the final-LayerNorm row at argmax(input_ids) (FlaxCLIP's end-of-text rule).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from .._lib import FdxError
from .common import EvaluationMetric

# One engine model per model name, shared by every metric built from it (both CLIP metrics of a run load the
# weights once).
_clip_cache: Dict[str, object] = {}


def _get_clip(modelname: str):
    """The cached CLIPPair of `modelname`: a Hugging Face model id in the local cache, or a directory holding a
    CLIPModel and its CLIPImageProcessorPil.  Nothing is downloaded."""
    if modelname not in _clip_cache:
        try:
            from transformers import CLIPModel
            from transformers.models.clip import CLIPImageProcessorPil
            model = CLIPModel.from_pretrained(modelname, local_files_only=True)
            processor = CLIPImageProcessorPil.from_pretrained(modelname, local_files_only=True)
        except Exception as e:  # noqa: BLE001
            raise FdxError(f"CLIP metrics: cannot load {modelname!r} from the local Hugging Face cache "
                           f"({type(e).__name__}); pass a local directory holding the model and its processor") from e
        from ..models.clip_vision import CLIPPair
        _clip_cache[modelname] = CLIPPair.from_transformers(model, processor)
    return _clip_cache[modelname]


def _tensor(x):
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def _similarity(pair, generated, batch):
    """(clip_similarity, clip_score) of samples [B, H, W, 3] in [-1, 1] against batch['text']'s tokens, f32 [2]."""
    text = batch["text"]
    mask = text.get("attention_mask")
    _, out2 = pair.similarity(_tensor(generated), _tensor(text["input_ids"]), None if mask is None else _tensor(mask))
    return out2


def get_clip_metric(modelname: str = "openai/clip-vit-large-patch14") -> EvaluationMetric:
    """clip_similarity = mean(1 - cos(image, text)): lower is better."""
    pair = _get_clip(modelname)

    def clip_metric(generated, batch) -> float:
        return float(_similarity(pair, generated, batch)[0])

    return EvaluationMetric(function=clip_metric, name="clip_similarity")


def get_clip_score_metric(modelname: str = "openai/clip-vit-large-patch14") -> EvaluationMetric:
    """CLIPScore (Hessel et al. 2021) = mean(100 max(cos(image, text), 0)): higher is better."""
    pair = _get_clip(modelname)

    def clip_score_metric(generated, batch) -> float:
        return float(_similarity(pair, generated, batch)[1])

    return EvaluationMetric(function=clip_score_metric, name="clip_score", higher_is_better=True)
