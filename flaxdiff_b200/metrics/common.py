"""EvaluationMetric (flaxdiff/metrics/common.py): what GeneralDiffusionTrainer.validation_loop evaluates."""
from dataclasses import dataclass
from typing import Callable


@dataclass
class EvaluationMetric:
    """`function(generated, batch)` -> scalar, with generated the validation samples [B, H, W, C] and batch the
    validation batch; the trainer tracks it as `val/<name>`, its maximum when higher_is_better, else its minimum."""
    function: Callable
    name: str
    higher_is_better: bool = False
