"""GPU probe for the mish activation (run directly on a GPU machine; not a pytest file).

Prints the card's name and power limit, then
  * the C2 training step (EDM UNet 64x64x3, B = 256, CUDA graph) and one Euler sampling step at B = 256, swish and
    mish alternating in this process, `--runs` runs each: ms per step;
  * each GroupNorm apply / backward call shape of the C2 UNet with act = silu and act = mish: ms per call;
  * each transposed-engine data-gradient shape of the C2 UNet (Cin, Cout): fdx_conv3x3_dgrad_gn (silu) and
    fdx_conv3x3_dgrad_gn_act (mish) alone, and the whole mish backward fused (data gradient with the GroupNorm
    first pass in its epilogue + one pass) against two-pass (data gradient + the two-pass GroupNorm backward).
Kernel-level times are min / median over CUDA-event windows of `--iters` calls.

usage: python tests/gpu_probe_mish.py [--runs 4] [--steps 20] [--iters 50]"""
import argparse
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200 import ops  # noqa: E402

dev = torch.device("cuda")
BF16 = torch.bfloat16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        out = f"{torch.cuda.get_device_name(0)}, power limit unknown"
    return out


def timed(fn, iters, rounds=3):
    """ms per call: (min, median) over `rounds` CUDA-event windows of `iters` calls each."""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return min(ms), statistics.median(ms)


def step_level(args):
    from flaxdiff_b200.inputs import DiffusionInputConfig
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.samplers import EulerSampler
    from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    res, B = 64, 256
    runs = {}
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).to(dev)
    for act in ("swish", "mish"):
        model = Unet(attention_configs=(None,) * 4, dtype=BF16, activation=act)
        tr = GeneralDiffusionTrainer(model, adamw(2.7e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                     DiffusionInputConfig("image", (res, res, 3), []), rngs=4, name="probe",
                                     model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                     use_cuda_graph=True)
        smp = EulerSampler(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev),
                           KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (res, res, 3), []))
        runs[act] = [tr, tr._define_train_step(B), smp, [], []]
        for _ in range(3):
            tr.state, _, tr.rngstate = runs[act][1](tr.state, tr.rngstate, {"image": img}, 0)
        smp.generate_samples(tr.state.ema_params, B, res, diffusion_steps=4, start_step=1000, device=dev)
    torch.cuda.synchronize()
    for _ in range(args.runs):
        for act in ("swish", "mish"):
            tr, step, smp, t_train, t_euler = runs[act]
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                tr.state, loss, tr.rngstate = step(tr.state, tr.rngstate, {"image": img}, 0)
            b.record()
            b.synchronize()
            t_train.append(a.elapsed_time(b) / args.steps)
            a.record()
            out = smp.generate_samples(tr.state.ema_params, B, res, diffusion_steps=args.steps, start_step=1000,
                                       device=dev)
            b.record()
            b.synchronize()
            t_euler.append(a.elapsed_time(b) / args.steps)
            assert math.isfinite(loss.item()) and torch.isfinite(out).all()
    for act in ("swish", "mish"):
        t_train, t_euler = runs[act][3], runs[act][4]
        print(f"C2 train step {act:5s}: " + " ".join(f"{v:.2f}" for v in t_train) +
              f" ms (median {statistics.median(t_train):.2f})")
        print(f"C2 Euler step {act:5s}: " + " ".join(f"{v:.2f}" for v in t_euler) +
              f" ms (median {statistics.median(t_euler):.2f})")
    del runs
    torch.cuda.empty_cache()


# GroupNorm inputs of the C2 UNet (B = 256): (H, W, C)
GN_SHAPES = [(64, 64, 64), (64, 64, 128), (64, 64, 192), (32, 32, 128), (32, 32, 192), (32, 32, 256),
             (32, 32, 384), (16, 16, 256), (16, 16, 384), (16, 16, 512), (16, 16, 768), (8, 8, 512), (8, 8, 1024)]
# data gradients of the C2 UNet that the transposed engine takes: (H, W, Cin, Cout)
DGRAD_SHAPES = [(64, 64, 64, 64), (64, 64, 128, 64), (64, 64, 192, 64), (32, 32, 128, 128), (32, 32, 192, 128),
                (32, 32, 384, 128), (16, 16, 384, 256), (16, 16, 448, 256)]


def kernel_level(args):
    N, G, eps = 256, 8, 1e-4
    print("GroupNorm calls, ms min / median (silu | mish):")
    for H, W, C in GN_SHAPES:
        x = torch.randn(N, H, W, C, device=dev).to(BF16)
        dy = torch.randn(N, H, W, C, device=dev).to(BF16)
        gamma, beta = 1 + 0.1 * torch.randn(C, device=dev), 0.1 * torch.randn(C, device=dev)
        st = ops.groupnorm_stats(x, G)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
        ci, ct = torch.empty(N, C, device=dev), torch.empty(C, device=dev)
        row = []
        for a in (ops.ACT_SILU, ops.ACT_MISH):
            row.append(timed(lambda: ops.groupnorm_apply(x, G, st, gamma, beta, eps, a, out=y), args.iters))
            row.append(timed(lambda: ops.groupnorm_bwd(x, dy, G, st, gamma, beta, eps, a, dg, db, dx,
                                                       csum_img=ci, csum_tot=ct), args.iters))
        print(f"  {N}x{H}x{W}x{C:4d}  apply {row[0][0]:.3f}/{row[0][1]:.3f} | {row[2][0]:.3f}/{row[2][1]:.3f}"
              f"   bwd {row[1][0]:.3f}/{row[1][1]:.3f} | {row[3][0]:.3f}/{row[3][1]:.3f}")
        del x, dy, y, dx
    print("data gradient + GroupNorm backward, ms min / median:")
    for H, W, C, Co in DGRAD_SHAPES:
        x = torch.randn(N, H, W, C, device=dev).to(BF16)
        dy = torch.randn(N, H, W, Co, device=dev).to(BF16)
        w = (torch.randn(3, 3, C, Co, device=dev) / math.sqrt(9 * C)).to(BF16)
        gamma, beta = 1 + 0.1 * torch.randn(C, device=dev), 0.1 * torch.randn(C, device=dev)
        st = ops.groupnorm_stats(x, G)
        ab = ops.groupnorm_coeffs(st, gamma, beta, H * W, eps)
        dz, dx = torch.empty_like(x), torch.empty_like(x)
        dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
        assert ops._gn_fuse_default(x, dy)
        e_silu = timed(lambda: ops.conv3x3_dgrad_gn(dy, w, dz, x, ab), args.iters)
        e_mish = timed(lambda: ops.conv3x3_dgrad_gn(dy, w, dz, x, ab, act_fn=ops.ACT_MISH), args.iters)
        full = {}
        for name, a, fused in (("silu fused", ops.ACT_SILU, None), ("mish fused", ops.ACT_MISH, True),
                               ("mish two-pass", ops.ACT_MISH, False)):
            full[name] = timed(lambda: ops.conv_dgrad_groupnorm_bwd(dy, w, x, G, st, gamma, beta, eps, dg, db, dx,
                                                                    fused=fused, act_fn=a), args.iters)
        print(f"  {N}x{H}x{W} Cin {C:3d} Cout {Co:3d}  dgrad_gn silu {e_silu[0]:.3f}/{e_silu[1]:.3f}  "
              f"mish {e_mish[0]:.3f}/{e_mish[1]:.3f}   whole backward: " +
              "  ".join(f"{k} {v[0]:.3f}/{v[1]:.3f}" for k, v in full.items()))
        del x, dy, dz, dx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--skip-steps", action="store_true")
    args = ap.parse_args()
    print("card:", card())
    if not args.skip_steps:
        step_level(args)
    kernel_level(args)


if __name__ == "__main__":
    main()
