"""flaxdiff.inference-compatible surface (flaxdiff/inference/__init__.py): from a run's checkpoint and config to
images."""
from .pipeline import DiffusionInferencePipeline, InferencePipeline
from .utils import (get_wandb_run, load_from_checkpoint, load_from_wandb_registry, load_from_wandb_run,
                    parse_config)
