"""Probe (a script, not a test): what jax.random's streams cost on the device, and what the whole-step graph
gives the Euler-ancestral sampler.

    python tests/gpu_probe_prng.py [--reps 200] [--rounds 3]

Prints, with the card's name, power limit and clocks read in the same run:
  * fdx_random_normal next to torch.randn at 3 145 728, 6 291 456 and 100 663 296 float32 elements: microseconds per
    launch (CUDA events over `reps` launches, the two alternated `rounds` times) and GB/s of output written;
  * EulerAncestralSampler steps/s at 64x64, B = 256, 50 steps and at 256x256, text CFG, B = 32, 30 steps, with a plain
    tuple key (per-evaluation graph, torch.Generator noise) and a ThreefryKey (whole-step graph), alternated, and
    the launches the host makes per step (graph replays + libfdx launches outside a graph) for both.
It needs a GPU and fails without one; it changes no device setting."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flaxdiff_b200 import _lib, ops, utils  # noqa: E402
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder  # noqa: E402
from flaxdiff_b200.models.simple_unet import Unet  # noqa: E402
from flaxdiff_b200.predictors import KarrasPredictionTransform  # noqa: E402
from flaxdiff_b200.samplers import EulerAncestralSampler  # noqa: E402
from flaxdiff_b200.schedulers import KarrasVENoiseScheduler  # noqa: E402


def timed(fn, reps):
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(reps):
        fn()
    s1.record()
    torch.cuda.synchronize()
    return s0.elapsed_time(s1) / reps * 1e3          # microseconds per call


def probe_normal(dev, reps, rounds):
    key = utils.jax_key(0)
    gen = torch.Generator(device=dev).manual_seed(0)
    print("normal draws, float32: microseconds per launch | GB/s written   (best of the alternated rounds)")
    for n in (3_145_728, 6_291_456, 100_663_296):
        out = torch.empty(n, dtype=torch.float32, device=dev)
        r = max(10, reps * 3_145_728 // n)
        ours = lambda: ops.random_normal(key, (n,), out=out)                    # noqa: E731
        theirs = lambda: torch.randn((n,), generator=gen, out=out)  # noqa: E731
        for f in (ours, theirs):
            timed(f, 5)                                                         # warm-up of this shape
        best = [float("inf"), float("inf")]
        for _ in range(rounds):
            for i, f in enumerate((ours, theirs)):
                best[i] = min(best[i], timed(f, r))
        print(f"  n={n:>11,d}  fdx_random_normal {best[0]:9.1f} us {4e-3 * n / best[0]:7.0f} GB/s   "
              f"torch.randn {best[1]:9.1f} us {4e-3 * n / best[1]:7.0f} GB/s   ({r} launches per timing)")


def probe_sampler(dev, name, res, B, steps, acfg, text, rounds):
    sched = KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev)
    conds, cond, kw = [], (), {}
    if text:
        enc = RandomEmbeddingEncoder(77, 768, device=dev)
        conds, cond, kw = [ConditionalInputConfig(enc)], (enc([f"prompt {i}" for i in range(B)]).to(dev),), \
            {"context_dim": 768}
    cfg = DiffusionInputConfig("image", (res, res, 3), conds)
    model = Unet(attention_configs=acfg, dtype=torch.bfloat16, **kw)
    params = model.init(4, device=dev)
    smp = EulerAncestralSampler(model, sched, KarrasPredictionTransform(0.5), cfg, guidance_scale=3.0 if text else 0.0)
    lib = _lib.load()
    replays = [0]
    orig = torch.cuda.CUDAGraph.replay

    def counted(self):
        replays[0] += 1
        return orig(self)

    def run(key, n):
        return smp.generate_samples(params, B, res, diffusion_steps=n, start_step=1000, device=dev,
                                    rngstate=utils.RandomMarkovState(key), model_conditioning_inputs=cond)
    keys = {"tuple key (per-evaluation graph)": utils.PRNGKey(42), "ThreefryKey (whole-step graph)": utils.jax_key(42)}
    best, launches = {k: float("inf") for k in keys}, {}
    for label, key in keys.items():
        run(key, 3)                                                             # warm-up + graph capture
        torch.cuda.CUDAGraph.replay = counted
        replays[0], before = 0, lib.fdx_launch_count()
        run(key, steps)
        launches[label] = (replays[0] / steps, (lib.fdx_launch_count() - before) / steps)
        torch.cuda.CUDAGraph.replay = orig
    torch.cuda.synchronize()
    for _ in range(rounds):
        for label, key in keys.items():
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            img = run(key, steps)
            s1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(img).all()
            best[label] = min(best[label], s0.elapsed_time(s1))
    print(f"EulerAncestral {name}: {res}x{res}, B={B}, {steps} steps{', text CFG g=3' if text else ''}")
    for label in keys:
        print(f"  {label:34s} {best[label]:9.1f} ms  {steps / best[label] * 1e3:8.2f} steps/s   per step: "
              f"{launches[label][0]:.2f} graph replays + {launches[label][1]:.1f} libfdx launches outside a graph")
    del smp, params, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-256", action="store_true", help="leave out the 256x256 text-CFG sampling shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_probe_prng: no CUDA device; nothing is measured without one")
    dev = torch.device("cuda", 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem",
                        "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    print("card (name, power limit, max SM clock, SM clock now, memory clock now):", q.stdout.strip() or q.stderr.strip())
    probe_normal(dev, args.reps, args.rounds)
    probe_sampler(dev, "C2 shape", 64, 256, 50, (None, None, None, None), False, args.rounds)
    if not args.skip_256:
        probe_sampler(dev, "C4 shape", 256, 32, 30, (None, {"heads": 8}, {"heads": 8}, {"heads": 8}), True, args.rounds)


if __name__ == "__main__":
    main()
