"""UViT on one H100: graphed training-step throughput and peak memory of UViT-B/2 at 64x64 (B = 256) and UViT-B/4 at
256x256 (B = 32, with and without the convolutional output head), SimpleUDiT-B/2 at 64x64 for comparison, and the C2
UNet training step from bench.py alternated between this tree and a parent tree.

    python tests/gpu_probe_uvit.py --which uvit-b2|uvit-b4|uvit-b4-head|udit-b2 [--batch B] [--out f.json]
    python tests/gpu_probe_uvit.py --which c2 --parent DIR [--rounds 2] [--out f.json]

Shapes: F = 768, 12 layers, 12 heads, a random [B, 77, 768] text context (L = N + 1 + 77 tokens).  pos_encoding alone
is 65536 x 768 f32 at p = 2 (192 MiB, plus its gradient and two Adam moments).  Each --which runs in its own process.
Times are CUDA events around warmed-up work; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flaxdiff_b200.models.udit import SimpleUDiT  # noqa: E402
from flaxdiff_b200.models.uvit import UViT  # noqa: E402
from gpu_probe_dit import card  # noqa: E402
from gpu_probe_mmdit import throughput  # noqa: E402

BASE = dict(emb_features=768, num_layers=12, num_heads=12, context_dim=768)
SHAPES = {"b2": (2, 64, 256), "b4": (4, 256, 32)}


def c2(parent: str, rounds: int):
    """bench.py's C2 UNet training step (--workload c2), alternating this tree and `parent`, one process per run."""
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = {"this": [], "parent": []}
    for _ in range(rounds):
        for key, root in (("parent", parent), ("this", here)):
            r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "30", "--warmup", "5",
                                "--workload", "c2", "--no-cpu-baseline"], cwd=root, capture_output=True, text=True)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            out[key].append(json.loads(line[-1]).get("value") if line else f"failed: {r.stderr[-300:]}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", required=True, choices=("uvit-b2", "uvit-b4", "uvit-b4-head", "udit-b2", "c2"))
    ap.add_argument("--parent", default=None, help="a built checkout of the parent commit (for --which c2)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=0, help="override the shape's batch")
    args = ap.parse_args()
    res = {"card": card()}
    if args.which == "c2":
        res["c2_img_per_s"] = c2(args.parent, args.rounds)
    else:
        name, shape = args.which.split("-")[:2]
        p, r, B = SHAPES[shape]
        B = args.batch or B
        if name == "udit":
            model = SimpleUDiT(patch_size=p, **BASE)
        else:
            model = UViT(patch_size=p, add_residualblock_output=args.which.endswith("head"), **BASE)
        res["shape"] = f"{type(model).__name__}-B/{p} {r}x{r}, B = {B}" + (" + head" if args.which.endswith("head")
                                                                            else "")
        torch.cuda.reset_peak_memory_stats()
        res[type(model).__name__] = throughput(model, r, B, args.iters, False)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
