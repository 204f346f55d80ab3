"""Sampling the UNet with its inference forward on one H100: the Euler step's time and peak memory through
forward(save=False), which keeps no tape, against the same step through the training forward, which keeps it
(alternated in one process, three times each).  Each round builds one sampler, captures its graphs, times it
and releases it before the other forward's round: the training forward's two graphs (the whole step and the last
evaluation) each keep a private pool of a training forward's activations, and at 256x256 with CFG they alone fill
most of the card.

    python tests/gpu_probe_unet_sampling.py --which all [--out f.json]     # every case below, one after the other
    python tests/gpu_probe_unet_sampling.py --which c2                     # one case (also c2-cfg, c5, c5-b64, c4-cfg)

Cases: the C2 UNet (bench.py's c2, no attention) at 64x64 with B = 256, with and without CFG; the C3 / C5 UNet
(8-head self-attention at the 32x32 level) at 256x256 with B = 32 and B = 64; C4 (8-head cross-attention on a random
[B, 77, 768] text context at the last three levels, CFG) at 256x256 with B = 32.  CFG (guidance 3) doubles the model
batch.  B = 64 at 256x256 is the largest model batch bench.py's workloads run there (C4's, with CFG), so every kernel
has run at its tensor sizes; `memory_fit_B` is the batch the card's memory would hold by the inference forward's
measured per-image peak, which is not run: kernels index activations of up to [64, 256, 256, 128] elements today,
and larger ones have not been audited for 32-bit offsets.  The Euler step is the sampler's whole-step CUDA graph:
(time of 7 steps - time of 2 steps) / 5.  Its peak is torch.cuda.max_memory_allocated() above what was allocated
before the sampler's first call (the parameters and their bf16 shadow), the capture of its graphs included; `held`
is torch.cuda.max_memory_reserved() above what was reserved before: what the sampler's graph pools keep from other
work while it lives.  The card's name, power limit and maximum SM clock are read in the same run."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder  # noqa: E402
from flaxdiff_b200.models.simple_unet import Unet  # noqa: E402
from flaxdiff_b200.predictors import KarrasPredictionTransform  # noqa: E402
from flaxdiff_b200.samplers import EulerSampler  # noqa: E402
from flaxdiff_b200.schedulers import KarrasVENoiseScheduler  # noqa: E402

dev = torch.device("cuda") if torch.cuda.is_available() else None
GB = 2 ** 30
ATTN = {  # bench.py's WORKLOADS attention configurations
    "c2": (None, None, None, None),
    "c5": (None, None, None, {"heads": 8}),
    "c4": (None, {"heads": 8}, {"heads": 8}, {"heads": 8}),
}
CASES = {  # case -> (UNet, resolution, B, guidance)
    "c2": ("c2", 64, 256, 0.0),
    "c2-cfg": ("c2", 64, 256, 3.0),
    "c5": ("c5", 256, 32, 0.0),
    "c5-b64": ("c5", 256, 64, 0.0),
    "c4-cfg": ("c4", 256, 32, 3.0),
}
HEADROOM = 6 * GB      # kept free in memory_fit_B: the allocator's rounding, the CUDA context


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def seconds(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e-3


class Setup:
    """One UNet, its parameters and (C4) text context, shared by the samplers of both forwards."""

    def __init__(self, unet, res, B, guidance):
        text = unet == "c4"
        self.model = Unet(attention_configs=ATTN[unet], dtype=torch.bfloat16, context_dim=768 if text else None)
        self.fp = self.model.init(4, device=dev)
        self.res, self.B, self.guidance = res, B, guidance
        self.enc = RandomEmbeddingEncoder(77, 768, device=dev) if text else None
        self.ctx = (self.enc([f"prompt {i}" for i in range(B)]).to(dev),) if text else ()

    def sampler(self, keep_tape):
        model = self.model
        if keep_tape:           # the same step through the training forward: the tape is built, then dropped
            model = _TrainingForward(model)
        conds = [ConditionalInputConfig(self.enc)] if self.enc is not None else []
        cfg = DiffusionInputConfig("image", (self.res, self.res, 3), conds)
        smp = EulerSampler(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev),
                           KarrasPredictionTransform(0.5), cfg, guidance_scale=self.guidance)

        def gen(n):
            return smp.generate_samples(self.fp, self.B, self.res, diffusion_steps=n, start_step=1000, device=dev,
                                        model_conditioning_inputs=self.ctx)
        return gen


class _TrainingForward:
    def __init__(self, model):
        self.model = model

    def __getattr__(self, name):
        return getattr(self.model, name)

    def forward(self, *a, **k):
        k["save"] = True
        return self.model.forward(*a, **k)


def round_(setup, keep_tape):
    """(peak bytes above what was allocated before, peak bytes reserved above what was reserved before, Euler step
    ms) of one sampler, which is then released."""
    gen = setup.sampler(keep_tape)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base, held = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
    gen(2)                                  # captures the whole-step and the last-evaluation graphs
    gen(7)
    peak, held = torch.cuda.max_memory_allocated() - base, torch.cuda.max_memory_reserved() - held
    ms = round((seconds(lambda: gen(7)) - seconds(lambda: gen(2))) / 5 * 1e3, 2)
    del gen
    gc.collect()
    torch.cuda.empty_cache()
    return peak, held, ms


def alternate(case):
    unet, res, B, g = CASES[case]
    s = Setup(unet, res, B, g)
    params = torch.cuda.memory_allocated()
    row = {"unet": unet, "res": res, "B": B, "cfg": g > 0, "model_batch": B * (2 if g > 0 else 1),
           "params_gb": round(params / GB, 3)}
    peaks, helds, times = {}, {}, {}
    for _ in range(3):
        for k in ("training_forward", "inference_forward"):
            peak, held, ms = round_(s, k == "training_forward")
            peaks[k], helds[k] = max(peaks.get(k, 0), peak), max(helds.get(k, 0), held)
            times.setdefault(k, []).append(ms)
    row["peak_above_params_gb"] = {k: round(v / GB, 3) for k, v in peaks.items()}
    row["held_gb"] = {k: round(v / GB, 3) for k, v in helds.items()}
    row["euler_step_ms"] = times
    row["memory_fit_B"] = int((torch.cuda.mem_get_info()[1] - params - HEADROOM) // (peaks["inference_forward"] / B))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", required=True, choices=["all", *CASES])
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if dev is None:
        raise SystemExit("gpu_probe_unet_sampling.py needs a GPU")
    res = {"card": card()}
    for c in (list(CASES) if args.which == "all" else [args.which]):
        res[c] = alternate(c)
        print(json.dumps({c: res[c]}), flush=True)
        gc.collect()            # each case's model, samplers and graphs are released before the next one
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
