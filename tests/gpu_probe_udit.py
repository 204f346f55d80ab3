"""SimpleUDiT on one H100: graphed training-step and Euler-step throughput against SimpleDiT at the same widths,
fdx_gemm_cat against torch.cat + fdx_gemm at the up_dense shape, and the split-weight float32 final projection against
the bf16 one.

    python tests/gpu_probe_udit.py --which gemm|udit-b2|dit-b2|udit-b4|dit-b4|udit-b2-euler|dit-b2-euler [--out f.json]

Shapes: B/2 at 64x64 (L = 1024) with B = 256 and B/4 at 256x256 (L = 4096) with B = 32 for training, B = 64 for the
Euler step; F = 768, 12 layers, 12 heads (SimpleUDiT: 13 blocks and 6 up_dense layers), a random [B, 77, 768] text
context for both models.  The up_dense shape is 262144 x 1536 -> 768 (B/2 at 64x64, B = 256).  Each --which runs in its
own process.  Times are CUDA events around warmed-up work; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200._lib import GEMM_KMN  # noqa: E402
from flaxdiff_b200.models.simple_dit import SimpleDiT  # noqa: E402
from flaxdiff_b200.models.udit import SimpleUDiT  # noqa: E402
from gpu_probe_dit import card, timed  # noqa: E402
from gpu_probe_mmdit import throughput  # noqa: E402

dev = torch.device("cuda")
BASE = dict(emb_features=768, num_layers=12, num_heads=12, context_dim=768)
SHAPES = {"b2": (2, 64, 256), "b4": (4, 256, 32)}
EULER_BATCH = 64


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def gemm():
    """up_dense forward at 262144 x [768 | 768] -> 768: fdx_gemm_cat against torch.cat + fdx_gemm (time and the peak
    memory the call adds over its inputs); the final projection [xf | xf] x [W_hi; W_lo] (K = 1536) against the bf16
    one (K = 768), N = 32 (p*p*3 = 12 padded)."""
    M, F = 262144, 768
    g = torch.Generator(device=dev).manual_seed(0)
    x, skip = (torch.randn(M, F, generator=g, device=dev).bfloat16() for _ in range(2))
    W = (torch.randn(2 * F, F, generator=g, device=dev) / (2 * F) ** 0.5).bfloat16()
    bias = torch.zeros(F, device=dev)

    def cat_gemm():
        y = torch.empty(M, F, dtype=torch.bfloat16, device=dev)
        return ops.gemm(GEMM_KMN, torch.cat([x, skip], 1), W, y, M, F, 2 * F, 2 * F, F, F, bias=bias)
    two = lambda: ops.linear_cat_fwd(x, skip, W, bias=bias)  # noqa: E731
    flop = 2.0 * M * F * 2 * F
    out = {}
    for k, fn in (("gemm_cat", two), ("torch_cat_plus_gemm", cat_gemm)):
        s = timed(fn, 20)
        out[k] = {"ms": round(s * 1e3, 3), "tflops": round(flop / s / 1e12, 1), "added_peak_gb": round(peak(fn), 3)}
    N = 32
    wsplit = (torch.randn(2 * F, N, generator=g, device=dev) * 0.02).bfloat16()
    yf = torch.empty(M, N, dtype=torch.float32, device=dev)
    split = lambda: ops.gemm_cat(GEMM_KMN, x, x, wsplit, yf, M, N, 2 * F, F, F, F, N, N)  # noqa: E731
    plain = lambda: ops.gemm(GEMM_KMN, x, wsplit[:F], yf, M, N, F, F, N, N)  # noqa: E731
    out["final_proj_split_f32_ms"] = round(timed(split, 20) * 1e3, 3)
    out["final_proj_bf16_ms"] = round(timed(plain, 20) * 1e3, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", required=True,
                    choices=("gemm", "udit-b2", "dit-b2", "udit-b4", "dit-b4", "udit-b2-euler", "dit-b2-euler"))
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    res = {"card": card()}
    if args.which == "gemm":
        res["gemm"] = gemm()
    else:
        name, shape = args.which.split("-")[:2]
        p, r, B = SHAPES[shape]
        sample = args.which.endswith("euler")
        B = EULER_BATCH if sample else B
        cls = SimpleUDiT if name == "udit" else SimpleDiT
        res["shape"] = f"{cls.__name__}-B/{p} {r}x{r}, B = {B}"
        torch.cuda.reset_peak_memory_stats()
        res[cls.__name__] = throughput(cls(patch_size=p, **BASE), r, B, args.iters, sample)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
