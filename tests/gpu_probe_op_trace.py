"""Probe (a script, not a test): the sequence of libfdx calls one UNet forward plus backward issues, for every
attention-block configuration of tests/test_attention_launches_gpu.py (pure and full blocks, with and without
projections, self-attention and a 77 x 768 text context, true head widths 16 / 64 / 80 / 128).

    python tests/gpu_probe_op_trace.py [--unet PATH] > trace.txt

Every public function of flaxdiff_b200.ops is wrapped by name, as bench.py wraps them, and each call that reaches
libfdx (a wrapped call that makes no wrapped call of its own) prints as one line: its name and every parameter,
defaults included - scalars by value, tensors by dtype, shape, strides and storage offset.  No pointers, so two runs
of the same program print the same text.  gemm reads only the addresses of its operands (M, N, K and the leading
dimensions are its scalar arguments), so its tensors print as the memory they span, contiguous dimensions merged.
Each configuration ends with the libfdx launch count of its forward plus backward.  `--unet` runs the Unet of another copy of
models/simple_unet.py (e.g. `git show <commit>:flaxdiff_b200/models/simple_unet.py`) on this build, so the traces of
two commits can be diffed.  It needs a GPU and fails without one; it changes no device setting."""
import argparse
import importlib.util
import inspect
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200.models import simple_unet  # noqa: E402
import test_attention_launches_gpu as cases  # noqa: E402


def merged(t: torch.Tensor):
    """(shape, strides) of the memory t spans: size-1 dimensions dropped, contiguous neighbours merged."""
    shape, strides = [], []
    for n, s in zip(t.shape, t.stride()):
        if n == 1:
            continue
        if shape and strides[-1] == n * s:
            shape[-1] *= n
            strides[-1] = s
        else:
            shape.append(n)
            strides.append(s)
    return tuple(shape), tuple(strides)


def describe(x, flat: bool) -> str:
    if isinstance(x, torch.Tensor):
        shape, strides = merged(x) if flat else (tuple(x.shape), x.stride())
        return f"{str(x.dtype)[6:]}{list(shape)}/{list(strides)}+{x.storage_offset()}"
    if isinstance(x, (tuple, list)):
        return "(" + ", ".join(describe(v, flat) for v in x) + ")"
    if x is None or isinstance(x, (bool, int, float, str, torch.dtype)):
        return repr(x)
    return type(x).__name__


def traced(fn):
    """Run fn() with every public ops function wrapped; -> the lines of the calls that reach libfdx."""
    names = [n for n, f in vars(ops).items()
             if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")]
    orig = {n: getattr(ops, n) for n in names}
    calls, stack = [], []

    def wrap(name, f):
        sig = inspect.signature(f)

        def inner(*a, **k):
            if stack:
                stack[-1][2] = True
            bound = sig.bind(*a, **k)
            bound.apply_defaults()         # a default passed explicitly prints as if left out
            rec = [name, ", ".join(f"{p}={describe(v, name == 'gemm')}" for p, v in bound.arguments.items()), False]
            calls.append(rec)
            stack.append(rec)
            try:
                return f(*a, **k)
            finally:
                stack.pop()
        return inner
    try:
        for n in names:
            setattr(ops, n, wrap(n, orig[n]))
        fn()
    finally:
        for n in names:
            setattr(ops, n, orig[n])
    return [f"{n}({a})" for n, a, nested in calls if not nested]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unet", default=None, help="a models/simple_unet.py to run instead of this tree's")
    args = ap.parse_args()
    unet = simple_unet
    if args.unet:
        spec = importlib.util.spec_from_file_location("flaxdiff_b200.models._probe_unet", args.unet)
        unet = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(unet)
    dev = torch.device("cuda")
    for block, _, _ in cases.BLOCKS:
        for d in sorted(cases.WIDTHS):
            before = cases.launch_count()
            lines = traced(lambda: cases.unet_fwd_bwd(block, d, dev, unet.Unet))
            torch.cuda.synchronize()
            print(f"== {block} d={d}")
            print("\n".join(lines))
            print(f"launches {cases.launch_count() - before}")


if __name__ == "__main__":
    main()
