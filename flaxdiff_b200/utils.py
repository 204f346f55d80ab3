"""Host utilities mirroring flaxdiff/utils.py for the hot path.

`RandomMarkovState` (flaxdiff/utils.py:95-99) threads a functional PRNG key through the
trainer and samplers.  Keys here are threefry2x32 keys with JAX's `split` / `fold_in`
semantics (jax/_src/prng.py; JAX is not installable here, so the construction is a
restatement checked against the published Random123 known-answer vectors in
tests/test_prng.py).

Which stream a key draws from is chosen where the key is made, by its type:
  * a plain tuple (`PRNGKey(seed)`, the default everywhere) draws bulk device tensors with a
    torch.Generator seeded from the key: statistically equivalent, not bit-identical, to
    `jax.random.normal` - parity tests therefore inject identical (x0, eps, t) tensors on both
    sides, as SURVEY.md $8(c) says;
  * a `ThreefryKey` (`jax_key(seed)`, same two words) draws them with the libfdx kernels of
    csrc/fdx_random.cu, which restate jax.random.{bits, uniform, normal, randint, bernoulli} of
    JAX 0.4.28 (jax_threefry_partitionable=False).  `split`, `fold_in` and
    `RandomMarkovState.get_random_key` return the type they were given, so the choice flows through
    samplers, schedulers and the trainer.  `uniform`, `normal_f32`, `randint` and `bernoulli` below
    are the host restatements those kernels are held to, bit for bit.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch

from . import ops
from ._lib import FdxError

_U32 = np.uint32
_ROT = ((13, 15, 26, 6), (17, 29, 16, 24))


def _rotl(x: np.ndarray, r: int) -> np.ndarray:
    return ((x << _U32(r)) | (x >> _U32(32 - r))).astype(_U32)


def threefry2x32(key: Tuple[int, int], x0: np.ndarray, x1: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Threefry-2x32, 20 rounds (Salmon et al., Random123), as used by jax.random."""
    with np.errstate(over="ignore"):
        k0, k1 = _U32(key[0]), _U32(key[1])
        ks = (k0, k1, _U32(k0 ^ k1 ^ _U32(0x1BD11BDA)))
        x0 = (np.asarray(x0, dtype=_U32) + ks[0]).astype(_U32)
        x1 = (np.asarray(x1, dtype=_U32) + ks[1]).astype(_U32)
        for i in range(5):
            for r in _ROT[i % 2]:
                x0 = (x0 + x1).astype(_U32)
                x1 = _rotl(x1, r)
                x1 = (x1 ^ x0).astype(_U32)
            x0 = (x0 + ks[(i + 1) % 3]).astype(_U32)
            x1 = (x1 + ks[(i + 2) % 3] + _U32(i + 1)).astype(_U32)
    return x0, x1


def _random_bits32(key: Tuple[int, int], n: int) -> np.ndarray:
    """jax threefry_random_bits for 32-bit output of length n (counter = iota, split in halves)."""
    m = (n + 1) // 2
    counts = np.arange(2 * m, dtype=_U32)
    a, b = threefry2x32(key, counts[:m], counts[m:])
    return np.concatenate([a, b])[:n]


def PRNGKey(seed: int) -> Tuple[int, int]:
    seed = int(seed)
    return ((seed >> 32) & 0xFFFFFFFF, seed & 0xFFFFFFFF)


class ThreefryKey(tuple):
    """A threefry key (two uint32 words) whose device draws are jax.random's own streams."""
    __slots__ = ()

    def __new__(cls, words):
        k0, k1 = (int(w) & 0xFFFFFFFF for w in words)
        return super().__new__(cls, (k0, k1))

    def __repr__(self):
        return f"ThreefryKey(({self[0]}, {self[1]}))"


def jax_key(seed: int) -> ThreefryKey:
    """`jax.random.PRNGKey(seed)`: the words of `PRNGKey(seed)`, drawing from JAX's streams."""
    return ThreefryKey(PRNGKey(seed))


def key_like(key, words):
    """A key with `words`, of the stream `key` draws from."""
    words = (int(words[0]), int(words[1]))
    return ThreefryKey(words) if isinstance(key, ThreefryKey) else words


def split(key: Tuple[int, int], num: int = 2):
    bits = _random_bits32(key, 2 * num).reshape(num, 2)
    return [key_like(key, r) for r in bits]


def fold_in(key: Tuple[int, int], data: int) -> Tuple[int, int]:
    a, b = threefry2x32(key, np.array([0], dtype=_U32), np.array([int(data) & 0xFFFFFFFF], dtype=_U32))
    return key_like(key, (a[0], b[0]))


def uniform01(key: Tuple[int, int], n: int) -> np.ndarray:
    """jax.random.uniform(key, (n,)) in [0,1): mantissa trick on 32 random bits."""
    bits = _random_bits32(key, n)
    f = ((bits >> _U32(9)) | _U32(0x3F800000)).view(np.float32) - np.float32(1.0)
    return f


def normal(key: Tuple[int, int], n: int) -> np.ndarray:
    """jax.random.normal(key, (n,), float32) = sqrt(2) * erfinv(uniform(-1+ulp, 1))."""
    from scipy.special import erfinv  # host-side, tiny n only (FourierEmbedding freqs)
    lo = np.nextafter(np.float32(-1.0), np.float32(0.0))
    hi = np.float32(1.0)
    u = uniform01(key, n) * (hi - lo) + lo
    u = np.maximum(lo, u).astype(np.float32)
    return (np.float32(np.sqrt(2.0)) * erfinv(u.astype(np.float64)).astype(np.float32)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------
# host restatements of jax.random's draws (JAX 0.4.28): the specification of csrc/fdx_random.cu
# ---------------------------------------------------------------------------------------------------------
_F32 = np.float32
_NORMAL_LO = np.nextafter(_F32(-1.0), _F32(0.0))
# Giles (2010), "Approximating the erfinv function", single precision, as XLA's erf_inv evaluates it
_ERFINV_CENTRAL = (2.81022636e-08, 3.43273939e-07, -3.5233877e-06, -4.39150654e-06, 0.00021858087,
                   -0.00125372503, -0.00417768164, 0.246640727, 1.50140941)
_ERFINV_TAIL = (-0.000200214257, 0.000100950558, 0.00134934322, -0.00367342844, 0.00573950773,
                -0.0076224613, 0.00943887047, 1.00167406, 2.83297682)


def uniform(key: Tuple[int, int], n: int, minval=0.0, maxval=1.0) -> np.ndarray:
    """jax.random.uniform(key, (n,), float32, minval, maxval): every operation rounded to float32."""
    minval, maxval = _F32(minval), _F32(maxval)
    return np.maximum(minval, uniform01(key, n) * _F32(maxval - minval) + minval).astype(_F32)


def erfinv_f32(u: np.ndarray) -> np.ndarray:
    """XLA's float32 erf_inv for |u| < 1, one float32 rounding per operation (no fused multiply-add)."""
    u = np.asarray(u, dtype=_F32)
    w = -np.log1p(-u * u).astype(_F32)
    central = w < _F32(5.0)
    with np.errstate(invalid="ignore"):
        w = np.where(central, w - _F32(2.5), np.sqrt(w) - _F32(3.0)).astype(_F32)
    p = np.where(central, _F32(_ERFINV_CENTRAL[0]), _F32(_ERFINV_TAIL[0])).astype(_F32)
    for c, t in zip(_ERFINV_CENTRAL[1:], _ERFINV_TAIL[1:]):
        p = (np.where(central, _F32(c), _F32(t)).astype(_F32) + p * w).astype(_F32)
    return (p * u).astype(_F32)


def normal_f32(key: Tuple[int, int], n: int) -> np.ndarray:
    """jax.random.normal(key, (n,), float32) with XLA's float32 erf_inv polynomial instead of SciPy's float64
    erfinv (`normal` above): what the device kernel computes."""
    return (_F32(np.sqrt(2.0)) * erfinv_f32(uniform(key, n, _NORMAL_LO, 1.0))).astype(_F32)


def randint(key: Tuple[int, int], n: int, minval: int, maxval: int) -> np.ndarray:
    """jax.random.randint(key, (n,), minval, maxval, int32) for minval < maxval: two 32-bit draws combined so
    that the modulo bias is that of a 64-bit draw.  Restated from jax/_src/random.py; no JAX was at hand to pin
    it against."""
    if not minval < maxval:
        raise ValueError(f"randint: minval={minval} must be below maxval={maxval}")
    k1, k2 = split(key)
    hi, lo = _random_bits32(k1, n), _random_bits32(k2, n)
    span = _U32((int(maxval) - int(minval)) & 0xFFFFFFFF)
    mult = _U32(65536) % span
    with np.errstate(over="ignore"):
        mult = _U32(mult * mult) % span
        off = ((hi % span) * mult + (lo % span)).astype(_U32) % span
        return (off + _U32(int(minval) & 0xFFFFFFFF)).astype(_U32).view(np.int32)


def bernoulli(key: Tuple[int, int], p: float, n: int) -> np.ndarray:
    """jax.random.bernoulli(key, p, (n,)) = uniform(key, (n,)) < p."""
    return uniform(key, n) < _F32(p)


def key_to_seed(key: Tuple[int, int]) -> int:
    return ((int(key[0]) << 32) | int(key[1])) & 0x7FFFFFFFFFFFFFFF


class DeviceKey:
    """The two words of a `ThreefryKey` in device memory (a (2,) int32 tensor): a captured CUDA graph draws
    from whatever key those 8 bytes hold when it is replayed."""

    def __init__(self, words: torch.Tensor):
        self.words = words


def _threefry_words(key):
    """The `ops.random_*` key argument for a key that draws from JAX's streams, else None."""
    if isinstance(key, DeviceKey):
        return key.words
    return key if isinstance(key, ThreefryKey) else None


def _f32_only(dtype):
    if dtype != torch.float32:
        raise FdxError(f"a ThreefryKey draws float32 only, not {dtype}")


def device_normal(key: Tuple[int, int], shape, device, dtype=torch.float32) -> torch.Tensor:
    words = _threefry_words(key)
    if words is not None:
        _f32_only(dtype)
        return ops.random_normal(words, shape, device=device)
    g = torch.Generator(device=device)
    g.manual_seed(key_to_seed(key))
    return torch.randn(shape, generator=g, device=device, dtype=dtype)


def device_uniform(key: Tuple[int, int], shape, device, dtype=torch.float32) -> torch.Tensor:
    words = _threefry_words(key)
    if words is not None:
        _f32_only(dtype)
        return ops.random_uniform(words, shape, device=device)
    g = torch.Generator(device=device)
    g.manual_seed(key_to_seed(key))
    return torch.rand(shape, generator=g, device=device, dtype=dtype)


def device_randint(key: Tuple[int, int], shape, low: int, high: int, device) -> torch.Tensor:
    words = _threefry_words(key)
    if words is not None:
        return ops.random_randint(words, shape, low, high, device=device)
    g = torch.Generator(device=device)
    g.manual_seed(key_to_seed(key))
    return torch.randint(low, high, shape, generator=g, device=device, dtype=torch.int32)


def device_bernoulli(key: Tuple[int, int], p: float, shape, device) -> torch.Tensor:
    """jax.random.bernoulli: `uniform < p`, on the stream `key` draws from."""
    return device_uniform(key, shape, device) < p


class MarkovState:
    pass


@dataclass(frozen=True)
class RandomMarkovState(MarkovState):
    """flaxdiff/utils.py:95-99: `get_random_key()` -> (new_state, subkey)."""
    rng: Tuple[int, int]

    def get_random_key(self):
        rng, subkey = split(self.rng)
        return RandomMarkovState(rng), subkey


def clip_images(images: torch.Tensor, clip_min=-1, clip_max=1) -> torch.Tensor:
    """flaxdiff/utils.py:101-112."""
    return torch.clamp(images, clip_min, clip_max)


def denormalize_images(images: torch.Tensor, target_type=torch.uint8, source_range=(-1, 1),
                       target_range=(0, 255)) -> torch.Tensor:
    """flaxdiff/utils.py:114-142."""
    src_min, src_max = source_range
    tgt_min, tgt_max = target_range
    images = clip_images(images, src_min, src_max)
    images = (images - src_min) / (src_max - src_min)
    images = images * (tgt_max - tgt_min) + tgt_min
    if target_type is not None:
        images = images.to(target_type)
    return images


# ---------------------------------------------------------------------------------------------------------
# configuration / checkpoint helpers of flaxdiff/utils.py:40-90, 239-263 (host side, no device work)
# ---------------------------------------------------------------------------------------------------------
DTYPE_MAP = {"bfloat16": torch.bfloat16, "float32": torch.float32, "float16": torch.float16, "None": None, None: None}
# jax.lax.Precision names of the reference's configs: there is one matmul precision here (bf16 operands, f32
# accumulation), so they all map to None ("backend default")
PRECISION_MAP = {"high": None, "HIGH": None, "default": None, "DEFAULT": None, "highest": None, "HIGHEST": None,
                 "None": None, None: None}
# the reference maps names to jax.nn functions; the Unet here takes the NAME (swish / silu and mish are implemented;
# relu and gelu pass through so that the Unet refuses them by name)
ACTIVATION_MAP = {"swish": "swish", "silu": "swish", "jax._src.nn.functions.silu": "swish", "mish": "mish",
                  "relu": "relu", "gelu": "gelu"}


def map_nested_config(config: dict) -> dict:
    """flaxdiff/utils.py:40-58: turn the strings of a serialised (wandb) model config back into objects - dtype
    names into torch dtypes, precision names into None, activation names into the activation key, 'None' into
    None; nested dicts recursively; other values are dropped exactly as the reference drops them."""
    out = {}
    for key, value in config.items():
        if isinstance(value, dict):
            out[key] = map_nested_config(value)
        elif isinstance(value, str):
            if value in DTYPE_MAP:
                out[key] = DTYPE_MAP[value]
            elif value in PRECISION_MAP:
                out[key] = PRECISION_MAP[value]
            elif value in ACTIVATION_MAP:
                out[key] = ACTIVATION_MAP[value]
            elif value == "None":
                out[key] = None
    return out


def serialize_model(model) -> dict:
    """flaxdiff/utils.py:60-82: the public attributes of a model object as a plain dict, callables (activation,
    initialisers) and dtypes replaced by their names, nested dicts / lists of dicts handled recursively."""
    def conv(v):
        if isinstance(v, dict):
            return {k: conv(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return type(v)(conv(x) for x in v)
        if isinstance(v, torch.dtype):
            return str(v).split(".")[-1]
        if callable(v):
            return getattr(v, "__name__", str(v).split(".")[-1])
        return v
    return {k: conv(v) for k, v in vars(model).items() if not k.startswith("_")}


def get_latest_checkpoint(checkpoint_path: str) -> str:
    """flaxdiff/utils.py:84-90: the step directory with the largest number under `checkpoint_path`."""
    import os
    steps = sorted(int(d) for d in os.listdir(checkpoint_path) if d.isdigit())
    if not steps:
        raise FileNotFoundError(f"no step directories under {checkpoint_path}")
    return os.path.join(checkpoint_path, str(steps[-1]))


class AutoTextTokenizer:
    """flaxdiff/utils.py:239-257: AutoTokenizer with CLIP's padding contract; returns input_ids, attention_mask and
    the captions.  The tokenizer files must be in the local Hugging Face cache (no network here); a tokenizer
    object may be passed instead."""

    def __init__(self, tensor_type: str = "pt", modelname: str = "openai/clip-vit-large-patch14", tokenizer=None):
        if tokenizer is None:
            from transformers import AutoTokenizer
            tokenizer = AutoTokenizer.from_pretrained(modelname, local_files_only=True)
        self.tokenizer = tokenizer
        self.tensor_type = tensor_type

    def __call__(self, inputs):
        tokens = self.tokenizer(inputs, padding="max_length", max_length=self.tokenizer.model_max_length,
                                truncation=True, return_tensors=self.tensor_type)
        return {"input_ids": tokens["input_ids"], "attention_mask": tokens["attention_mask"], "caption": inputs}

    def __repr__(self):
        return self.__class__.__name__ + "()"


def defaultTextEncodeModel(modelname: str = "openai/clip-vit-large-patch14", backend: str = "torch"):
    """flaxdiff/utils.py:261-263 (the torch backend is the only one here)."""
    from .inputs import CLIPTextEncoder
    return CLIPTextEncoder.from_modelname(modelname=modelname, backend=backend)
