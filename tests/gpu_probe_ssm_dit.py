"""HybridSSMAttentionDiT on one H100: the S5 scan kernels against their HBM floor, one SSM block against one attention
block (forward + backward) at the same shapes, and graphed training-step and Euler-step throughput of hybrid 3:1 next
to SimpleDiT at the same widths.

    python tests/gpu_probe_ssm_dit.py [--out results.json]

Configs: B/2 at 64x64 (L = 1024), B = 256, and B/4 at 256x256 (L = 4096), B = 32; F = 768, 12 layers, 12 heads,
ssm_state_dim = 64, bidirectional.  Times are CUDA events around warmed-up work; the card's name and power limit are
read in the same run."""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200.inputs import DiffusionInputConfig  # noqa: E402
from flaxdiff_b200.models.simple_dit import SimpleDiT  # noqa: E402
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT  # noqa: E402
from flaxdiff_b200.predictors import KarrasPredictionTransform  # noqa: E402
from flaxdiff_b200.samplers import EulerSampler  # noqa: E402
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler  # noqa: E402
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw  # noqa: E402
from gpu_probe_dit import HBM, card, timed  # noqa: E402

dev = torch.device("cuda")
CONFIGS = [("B/2 64x64", 2, 64, 256), ("B/4 256x256", 4, 256, 32)]
BASE = dict(emb_features=768, num_layers=12, num_heads=12)
N = 64


def scans(B, L):
    """fdx_ssm_scan / _scan_bwd (both directions, N = 64): seconds and share of the HBM floor.  Each pass must read
    its f32 input once and write its outputs once: the scan reads Bu and writes the f32 and bf16 states (10 bytes per
    real column), the adjoint reads dx, the f32 states and Bu and writes bf16 lambda (14 bytes)."""
    S2 = 4 * N
    M = B * L
    chunk = ops.ssm_chunk(B, L, 2 * N, dev)
    adt = torch.empty(S2, device=dev)
    adt[:N] = adt[2 * N:3 * N] = -0.01 * (torch.arange(N, device=dev) + 0.5)
    adt[N:2 * N] = adt[3 * N:] = 0.01 * torch.arange(N, device=dev)
    bu = torch.randn(M, S2, device=dev) * 1e-3
    x, _ = ops.ssm_scan(bu, adt, B, N, 2, chunk)
    dx = torch.randn(M, S2, device=dev)
    out = {"chunk": chunk}
    for k, fn, nbytes in (("scan", lambda: ops.ssm_scan(bu, adt, B, N, 2, chunk, out=x), 10 * M * S2),
                          ("scan_bwd", lambda: ops.ssm_scan_bwd(dx, x, bu, adt, B, N, 2, chunk), 14 * M * S2)):
        s = timed(fn, 20)
        out[k] = {"us": round(s * 1e6, 1), "hbm_floor_share": round(nbytes / HBM / s, 3)}
    return out


def blocks(B, L):
    """One bidirectional SSM block and one attention block, forward + backward, at the same shapes (ms)."""
    model = HybridSSMAttentionDiT(patch_size=2, emb_features=768, num_layers=2, num_heads=12, ssm_state_dim=N,
                                  block_pattern=["ssm", "attn"])
    fp = model.init(0, device=dev)
    W32, W16, G = fp.named, fp.shadow(), fp.zeros_like()
    x = torch.randn(B * L, 768, device=dev).bfloat16()
    cond16 = torch.randn(B, 768, device=dev).bfloat16()
    dcond = torch.zeros(B, 768, device=dev)
    dx2 = torch.randn_like(x)
    out = {}
    for (n, fwd, bwd) in model._blocks():
        def run():
            _, rec = fwd(n, x, cond16, W32, W16, B, L)
            bwd(rec, dx2, cond16, dcond, W32, W16, G.named, B, L)
        out[n.split("_block")[0] + "_block_fwd_bwd_ms"] = round(timed(run, 5) * 1e3, 2)
    return out


def throughput(model, r, B, iters):
    row = {}
    try:
        tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                     DiffusionInputConfig("image", (r, r, 3), []), rngs=4,
                                     model_output_transform=KarrasPredictionTransform(0.5), device=dev)
        step = tr._define_train_step()
        batch = {"image": torch.randint(0, 256, (B, r, r, 3), dtype=torch.uint8, device=dev)}
        st = [tr.state, tr.rngstate]

        def train():
            st[0], _, st[1] = step(st[0], st[1], batch)
        s = timed(train, iters)
        row["train_step_ms"] = round(s * 1e3, 2)
        row["train_img_per_s"] = round(B / s, 1)
        row["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    except torch.cuda.OutOfMemoryError as e:
        row["train_error"] = f"out of memory: {str(e)[:120]}"
    tr = step = st = train = None
    gc.collect()
    torch.cuda.empty_cache()
    try:
        fp = model.init(0, device=dev)
        smp = EulerSampler(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev),
                           KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (r, r, 3), []))
        s12 = timed(lambda: smp.generate_samples(fp, B, r, diffusion_steps=12, start_step=1000, device=dev), 2, warm=1)
        s2 = timed(lambda: smp.generate_samples(fp, B, r, diffusion_steps=2, start_step=1000, device=dev), 2, warm=1)
        row["euler_step_ms"] = round((s12 - s2) / 10 * 1e3, 2)
        row["euler_img_steps_per_s"] = round(B / ((s12 - s2) / 10), 1)
    except torch.cuda.OutOfMemoryError as e:
        row["euler_error"] = f"out of memory: {str(e)[:120]}"
    smp = fp = None
    gc.collect()
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    res = {"card": card(), "configs": {}}
    print(res["card"], flush=True)
    for name, p, r, B in CONFIGS:
        L = (r // p) ** 2
        row = {"scans": scans(B, L)}
        gc.collect()
        torch.cuda.empty_cache()
        row["blocks"] = blocks(B, L)
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        row["hybrid_3to1"] = throughput(HybridSSMAttentionDiT(patch_size=p, ssm_state_dim=N, **BASE), r, B, args.iters)
        torch.cuda.reset_peak_memory_stats()
        row["simple_dit"] = throughput(SimpleDiT(patch_size=p, **BASE), r, B, args.iters)
        res["configs"][name] = row
        print(name, json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
