"""Conditioning-input configuration (API of flaxdiff/inputs/__init__.py:15-172).

Only the contract the samplers / trainer need is kept: which batch key feeds which model
kwarg, the cached unconditional ("null") embedding, and the per-sample null mixing used for
classifier-free-guidance training.  `CLIPTextEncoder` is the reference's text tower on the torch backend of
`transformers` (weights must be in the local cache); BASELINE config 4 uses frozen random text embeddings:
`RandomEmbeddingEncoder`.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Tuple

import torch


class ConditioningEncoder:
    """Maps raw conditioning (e.g. strings) to an embedding tensor (B, T, D)."""
    key = "text"

    def __call__(self, data) -> torch.Tensor:
        raise NotImplementedError

    def encode_from_tokens(self, tokens) -> torch.Tensor:
        raise NotImplementedError

    def serialize(self) -> dict:
        return {}


class RandomEmbeddingEncoder(ConditioningEncoder):
    """Frozen random embeddings keyed by hash of the input (stand-in for CLIPTextEncoder,
    flaxdiff/inputs/encoders.py:61-94)."""

    def __init__(self, seq_len: int = 77, features: int = 768, key: str = "text", device=None, seed: int = 0):
        self.seq_len, self.features, self.key, self.seed = seq_len, features, key, seed
        self.device = device

    def _one(self, item) -> torch.Tensor:
        g = torch.Generator()
        import zlib
        g.manual_seed((zlib.crc32(str(item).encode()) ^ self.seed) & 0x7FFFFFFF)
        return torch.randn(self.seq_len, self.features, generator=g)

    def __call__(self, data) -> torch.Tensor:
        if isinstance(data, torch.Tensor):
            return data
        out = torch.stack([self._one(d) for d in data])
        return out.to(self.device) if self.device is not None else out

    def encode_from_tokens(self, tokens):
        return self(tokens)

    def serialize(self):
        return {"seq_len": self.seq_len, "features": self.features, "seed": self.seed}

    @staticmethod
    def deserialize(serialized_config: dict):
        return RandomEmbeddingEncoder(seq_len=serialized_config.get("seq_len", 77),
                                      features=serialized_config.get("features", 768),
                                      seed=serialized_config.get("seed", 0))


class CLIPTextEncoder(ConditioningEncoder):
    """`CLIPTextEncoder` of the reference (flaxdiff/inputs/encoders.py:53-94) on the torch backend of
    `transformers` (SURVEY $8 f3): tokenizer(padding="max_length", max_length=model_max_length, truncation=True)
    -> CLIPTextModel -> last_hidden_state (B, 77, 768), frozen, evaluated under no_grad.  The text tower is
    conditioning PRE-processing, not the hot path: it runs as stock PyTorch modules; its output feeds the UNet's
    cross-attention as a bf16 CUDA tensor.  backend="fdx" runs the same weights as the engine's text tower
    (models/clip_text.py), which the trainer then evaluates inside its training step.  `model` / `tokenizer` may be
    injected (tests, custom towers); `from_modelname` needs the weights in the local Hugging Face cache."""
    key = "text"

    def __init__(self, model, tokenizer, modelname: str = "openai/clip-vit-large-patch14", backend: str = "torch",
                 device=None, dtype: torch.dtype = torch.bfloat16):
        self.model, self.tokenizer, self.modelname, self.backend = model, tokenizer, modelname, backend
        self.device, self.dtype = device, dtype
        self.tower = None
        if hasattr(model, "eval"):
            model.eval()
        if backend == "fdx":
            # the engine's tower: the weights are packed onto the GPU once, the transformers model stays on the host
            from ..models.clip_text import CLIPTextTower
            self.tower = CLIPTextTower.from_transformers(model, device, seq_len=tokenizer.model_max_length)
        elif device is not None and hasattr(model, "to"):
            model.to(device)

    @staticmethod
    def from_modelname(modelname: str = "openai/clip-vit-large-patch14", backend: str = "torch", device=None):
        from .._lib import FdxError
        if backend not in ("torch", "pt", "fdx"):
            raise FdxError(f"CLIPTextEncoder backend {backend!r}: only the torch backend and the engine's 'fdx' "
                           "tower exist here (JAX is not installed)")
        try:
            from transformers import AutoTokenizer, CLIPTextModel
            model = CLIPTextModel.from_pretrained(modelname, local_files_only=True)
            tokenizer = AutoTokenizer.from_pretrained(modelname, local_files_only=True)
        except Exception as e:  # noqa: BLE001
            raise FdxError(f"CLIPTextEncoder: cannot load {modelname!r} from the local Hugging Face cache "
                           f"({type(e).__name__}); pass model= / tokenizer= or use RandomEmbeddingEncoder") from e
        return CLIPTextEncoder(model, tokenizer, modelname, "fdx" if backend == "fdx" else "torch", device)

    def tokenize(self, data):
        return self.tokenizer(list(data), padding="max_length", max_length=self.tokenizer.model_max_length,
                              truncation=True, return_tensors="pt")

    def encode_from_tokens(self, tokens) -> torch.Tensor:
        ids, mask = tokens["input_ids"], tokens["attention_mask"]
        if self.tower is not None:
            return self.tower.encode(ids, mask)         # bf16 on the GPU
        if self.device is not None:
            ids, mask = ids.to(self.device), mask.to(self.device)
        with torch.no_grad():
            out = self.model(input_ids=ids, attention_mask=mask).last_hidden_state
        return out.to(self.dtype)

    def __call__(self, data) -> torch.Tensor:
        if isinstance(data, torch.Tensor):          # already embedded
            return data
        return self.encode_from_tokens(self.tokenize(data))

    def serialize(self) -> dict:
        return {"modelname": self.modelname, "backend": self.backend}

    @staticmethod
    def deserialize(serialized_config: dict):
        return CLIPTextEncoder.from_modelname(serialized_config["modelname"], serialized_config.get("backend", "torch"))


CONDITIONAL_ENCODERS_REGISTRY = {"text": CLIPTextEncoder}


@dataclass
class ConditionalInputConfig:
    encoder: ConditioningEncoder
    conditioning_data_key: str = None
    pretokenized: bool = False
    unconditional_input: Any = None
    model_key_override: Optional[str] = None

    def __post_init__(self):
        null = self.unconditional_input if self.unconditional_input is not None else ""
        self._uncond = self.encoder([null])

    def __call__(self, batch_data):
        key = self.conditioning_data_key if self.conditioning_data_key else self.encoder.key
        if self.pretokenized:
            return self.encoder.encode_from_tokens(batch_data[key])
        return self.encoder(batch_data[key])

    def get_unconditional(self):
        return self._uncond

    def serialize(self):
        return {"encoder": self.encoder.serialize(), "encoder_key": self.encoder.key,
                "conditioning_data_key": self.conditioning_data_key,
                "unconditional_input": self.unconditional_input,
                "model_key_override": self.model_key_override}

    @staticmethod
    def deserialize(serialized_config: dict, registry: Optional[Dict[str, Any]] = None):
        """inputs/__init__.py:55-74: rebuild the encoder through the registry (`encoder_key` -> class with a
        `deserialize`), then the config.  `registry` extends / overrides CONDITIONAL_ENCODERS_REGISTRY (e.g.
        {"text": RandomEmbeddingEncoder} where the CLIP weights are not available)."""
        reg = dict(CONDITIONAL_ENCODERS_REGISTRY)
        reg.update(registry or {})
        encoder_key = serialized_config["encoder_key"]
        encoder_class = reg.get(encoder_key)
        if encoder_class is None:
            raise ValueError(f"Unknown encoder type: {encoder_key}")
        encoder = encoder_class.deserialize(serialized_config["encoder"])
        return ConditionalInputConfig(encoder=encoder,
                                      conditioning_data_key=serialized_config.get("conditioning_data_key"),
                                      unconditional_input=serialized_config.get("unconditional_input"),
                                      model_key_override=serialized_config.get("model_key_override"))


@dataclass
class DiffusionInputConfig:
    sample_data_key: str
    sample_data_shape: Tuple[int, ...]
    conditions: List[ConditionalInputConfig] = field(default_factory=list)

    def get_input_shapes(self, autoencoder=None, sample_model_key: str = 'x',
                         time_embeddings_model_key: str = 'temb') -> Dict[str, Tuple[int, ...]]:
        if len(self.sample_data_shape) == 3:
            H, W, C = self.sample_data_shape
        elif len(self.sample_data_shape) == 4:
            _, H, W, C = self.sample_data_shape
        else:
            raise ValueError(f"Unsupported shape for sample data {self.sample_data_shape}")
        shapes = {sample_model_key: (H, W, C), time_embeddings_model_key: ()}
        for cond in self.conditions:
            key = cond.model_key_override if cond.model_key_override else cond.encoder.key
            shapes[key] = tuple(cond.get_unconditional()[0].shape)
        return shapes

    def get_unconditionals(self):
        return [c.get_unconditional() for c in self.conditions]

    def process_conditioning(self, batch_data, uncond_mask: Optional[torch.Tensor] = None):
        """Per-sample null mixing (inputs/__init__.py:123-146)."""
        results = []
        for cond in self.conditions:
            emb = cond(batch_data)
            if uncond_mask is not None:
                assert len(uncond_mask) == len(emb), "Unconditional mask length must match the batch size."
                null = cond.get_unconditional().to(emb.device).expand_as(emb)
                mask = uncond_mask.to(emb.device).reshape([len(uncond_mask)] + [1] * (emb.dim() - 1))
                emb = torch.where(mask.bool(), null, emb)
            results.append(emb)
        return results

    def serialize(self):
        return {"sample_data_key": self.sample_data_key, "sample_data_shape": self.sample_data_shape,
                "conditions": [c.serialize() for c in self.conditions]}

    @staticmethod
    def deserialize(serialized_config: dict, registry: Optional[Dict[str, Any]] = None):
        """inputs/__init__.py:157-173."""
        return DiffusionInputConfig(
            sample_data_key=serialized_config["sample_data_key"],
            sample_data_shape=tuple(serialized_config["sample_data_shape"]),
            conditions=[ConditionalInputConfig.deserialize(c, registry) for c in serialized_config["conditions"]])
