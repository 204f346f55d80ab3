"""Validation metrics (flaxdiff/metrics): the CLIP image-text metrics of the reference's training script."""
from .common import EvaluationMetric
from .images import get_clip_metric, get_clip_score_metric

__all__ = ["EvaluationMetric", "get_clip_metric", "get_clip_score_metric"]
