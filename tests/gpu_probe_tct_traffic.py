"""GPU probe for the transposed convolution engine (run directly on a GPU machine; not a pytest file).

Prints the card's name and power limit, then runs one eager training step of the C2 workload (EDM UNet 64 x 64,
B = 256) with every convolution wrapper recorded, keeps the calls that ran `fdx_tct_kernel`, and times each
distinct call shape alone: the same call on the same tensors (slot views and strides included), CUDA events over
`--iters` launches after warm-up, as min / median / max over `--rounds` windows.  Per shape it prints the number of
such calls in the step, microseconds per call, the algorithmic HBM bytes (every activation the call reads or
writes once, plus the weights; computed from the shapes below), GB/s, the fraction of the 3.35 TB/s of the H100
SXM data sheet, and TFLOP/s; then the step's total over all recorded calls, weighted by their count.

usage: python tests/gpu_probe_tct_traffic.py [--batch 256] [--iters 20] [--rounds 3]"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200 import _lib, ops  # noqa: E402

dev = torch.device("cuda")
HBM_BYTES_PER_S = 3.35e12
OPS = ("conv3x3_fwd", "conv3x3_dgrad", "conv3x3_dgrad_gn", "conv1x1_fwd", "conv1x1_dgrad")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        out = f"{torch.cuda.get_device_name(0)}, power limit unknown"
    return out


def nbytes(t):
    return 0 if t is None else t.numel() * t.element_size()


def arg(a, k, i, name, default=None):
    return a[i] if len(a) > i else k.get(name, default)


def cost(name, a, k):
    """(algorithmic HBM bytes, FLOPs, label) of one call, from its arguments' shapes."""
    if name == "conv3x3_fwd":
        x, w, res, out = a[0], a[1], arg(a, k, 4, "res"), arg(a, k, 5, "out")
        taps = 9
        extra = [s for s, v in (("bias", arg(a, k, 2, "bias")), ("row", arg(a, k, 3, "rowvec")), ("res", res),
                                ("colsum", arg(a, k, 7, "colstats"))) if v is not None]
        byt = nbytes(x) + nbytes(res) + nbytes(out) + nbytes(w)
        cin, cout, dst = x.shape[3], out.shape[3], out
        kind = f"3x3 fwd s{arg(a, k, 6, 'stride', 1)}"
    elif name in ("conv3x3_dgrad", "conv3x3_dgrad_gn"):
        dy, w, dst = a[0], a[1], a[2]
        if name == "conv3x3_dgrad_gn":
            byt = nbytes(dy) + nbytes(dst) + nbytes(a[3]) + nbytes(w)
            extra = ["gnb"]
        else:
            acc = bool(arg(a, k, 4, "accumulate", False))
            byt = nbytes(dy) + nbytes(dst) * (2 if acc else 1) + nbytes(w)
            extra = ["acc"] if acc else []
        cin, cout = dst.shape[3], dy.shape[3]
        kind = f"3x3 dgrad s{arg(a, k, 3, 'stride', 1) if name == 'conv3x3_dgrad' else 1}"
        # FLOPs at the resolution of dy (the forward's output), as bench.py counts them
        return byt, 2.0 * dy.shape[0] * dy.shape[1] * dy.shape[2] * 9 * cin * cout, label_of(kind, dst, cin, cout,
                                                                                              extra)
    elif name == "conv1x1_fwd":
        x, w, res, out = a[0], a[1], arg(a, k, 3, "res"), arg(a, k, 4, "out")
        extra = [s for s, v in (("bias", arg(a, k, 2, "bias")), ("res", res)) if v is not None]
        byt = nbytes(x) + nbytes(res) + nbytes(out) + nbytes(w)
        cin, cout, dst, taps = x.shape[3], out.shape[3], out, 1
        kind = "1x1 fwd"
    else:
        dy, w, dst = a[0], a[1], a[2]
        acc = bool(arg(a, k, 3, "accumulate", False))
        byt = nbytes(dy) + nbytes(dst) * (2 if acc else 1) + nbytes(w)
        extra = ["acc"] if acc else []
        cin, cout, taps = dst.shape[3], dy.shape[3], 1
        kind = "1x1 dgrad"
    return byt, 2.0 * dst.shape[0] * dst.shape[1] * dst.shape[2] * taps * cin * cout, label_of(kind, dst, cin, cout,
                                                                                                extra)


def label_of(kind, dst, cin, cout, extra):
    """e.g. '3x3 dgrad s1 64x64 64->320 [gnb]': layer input -> output channels of the forward convolution"""
    slot = "" if dst.is_contiguous() else f" slot(pix_stride {dst.stride(2)})"
    return f"{kind} {dst.shape[1]}x{dst.shape[2]} {cin}->{cout} [{'+'.join(extra) or 'plain'}]{slot}"


def key_of(name, a, k):
    def d(v):
        if isinstance(v, torch.Tensor):
            return (tuple(v.shape), tuple(v.stride()), str(v.dtype))
        if isinstance(v, tuple):
            return tuple(d(x) for x in v)
        if isinstance(v, ops.ColStats):
            return ("colstats", v.channels)
        return v
    return (name, tuple(d(v) for v in a), tuple(sorted((kk, d(v)) for kk, v in k.items())))


def record_step(B):
    from flaxdiff_b200.inputs import DiffusionInputConfig
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.schedulers import EDMNoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    lib = _lib.load()
    res = 64
    model = Unet(attention_configs=(None, None, None, None), dtype=torch.bfloat16)
    trainer = GeneralDiffusionTrainer(
        model, adamw(2.7e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
        DiffusionInputConfig("image", (res, res, 3), []), rngs=4, name="probe",
        model_output_transform=KarrasPredictionTransform(sigma_data=0.5), ema_decay=0.999, device=dev,
        use_cuda_graph=False)
    gen = torch.Generator().manual_seed(1234)
    images = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8, generator=gen).to(dev)
    noise = torch.randn(B, res, res, 3, device=dev)
    t = torch.randn(B, device=dev)
    os.environ["FDX_NO_SIDE"] = "1"
    trainer._overlap = False
    trainer._fwd_bwd(images, noise, t)                 # warm-up: module load, first launches
    torch.cuda.synchronize()
    orig = {n: getattr(ops, n) for n in OPS}
    calls = {}

    def wrap(name, fn):
        def inner(*a, **k):
            r = fn(*a, **k)
            if lib.fdx_last_kernel_kind() == 1:        # FDX_KERNEL_TCT
                key = key_of(name, a, k)
                if key in calls:
                    calls[key][3] += 1
                else:
                    calls[key] = [name, a, k, 1]
            return r
        return inner
    try:
        for n in OPS:
            setattr(ops, n, wrap(n, orig[n]))
        trainer._fwd_bwd(images, noise, t)
        torch.cuda.synchronize()
    finally:
        for n in OPS:
            setattr(ops, n, orig[n])
    return [tuple(v) for v in calls.values()], orig


def timed(fn, iters, rounds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    us = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        us.append(a.elapsed_time(b) * 1e3 / iters)
    return min(us), statistics.median(us), max(us)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    print(f"card: {info}", flush=True)
    calls, orig = record_step(args.batch)
    rows, total_us, total_floor = [], 0.0, 0.0
    for name, a, k, count in calls:
        byt, fl, label = cost(name, a, k)
        t = timed(lambda: orig[name](*a, **k), args.iters, args.rounds)
        med = t[1]
        floor_us = byt / HBM_BYTES_PER_S * 1e6
        total_us += med * count
        total_floor += floor_us * count
        rows.append((med * count, f"{label:58s} x{count:<2d} {t[0]:8.1f} / {med:8.1f} / {t[2]:8.1f} us  "
                                  f"{byt / 1e6:8.1f} MB  {byt / med / 1e3:7.1f} GB/s  "
                                  f"{floor_us / med:5.1%} of HBM  {fl / med / 1e6:6.1f} TF/s"))
    for _, r in sorted(rows, key=lambda r: -r[0]):
        print(f"[{info}] {r}", flush=True)
    print(f"[{info}] fdx_tct_kernel calls of one C2 step (B={args.batch}): {sum(c[3] for c in calls)} calls, "
          f"{total_us / 1e3:.2f} ms timed alone (HBM floor {total_floor / 1e3:.2f} ms)", flush=True)


if __name__ == "__main__":
    main()
