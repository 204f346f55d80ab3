"""use_remat on one H100: graphed training-step throughput and peak memory of the transformer denoisers with and
without the flag, at 64x64 with patch size 2.

    python tests/gpu_probe_remat.py [--rounds 1] [--iters 10] [--out f.json]
    python tests/gpu_probe_remat.py --which uvit|dit|udit --batch B --remat 0|1       (one case, in this process)

Cases: UViT-B/2 at B = 256 with the flag (without it this shape does not fit in 80 GB); SimpleDiT-B/2 and
SimpleUDiT-B/2 at B = 256, and UViT-B/2 and SimpleDiT-B/2 at B = 128, each with and without the flag.  Shapes are
gpu_probe_uvit.py's: F = 768, 12 layers, 12 heads, a random [B, 77, 768] text context.  Each case runs in its own
process (a fresh allocator, so its peak is its own), warmed up before the timed steps, and the two settings of a case
run back to back, their order alternating from case to case and round to round.  Times are CUDA events around warmed-up
graphed steps; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flaxdiff_b200.models.simple_dit import SimpleDiT  # noqa: E402
from flaxdiff_b200.models.udit import SimpleUDiT  # noqa: E402
from flaxdiff_b200.models.uvit import UViT  # noqa: E402
from gpu_probe_dit import card  # noqa: E402
from gpu_probe_mmdit import throughput  # noqa: E402

BASE = dict(patch_size=2, emb_features=768, num_layers=12, num_heads=12, context_dim=768)
CLASSES = {"uvit": UViT, "dit": SimpleDiT, "udit": SimpleUDiT}
# (model, batch, settings to run)
CASES = [("uvit", 256, (True,)), ("dit", 256, (False, True)), ("udit", 256, (False, True)),
         ("uvit", 128, (False, True)), ("dit", 128, (False, True))]
RES = 64


def one(which: str, batch: int, remat: bool, iters: int) -> dict:
    model = CLASSES[which](use_remat=remat, **BASE)
    torch.cuda.reset_peak_memory_stats()
    return throughput(model, RES, batch, iters, False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", choices=sorted(CLASSES), default=None)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--remat", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if args.which:
        print(json.dumps(one(args.which, args.batch, bool(args.remat), args.iters)), flush=True)
        return
    res = {"card": card(), "shape": f"B/2 {RES}x{RES}, F = 768, 12 layers, 12 heads, 77 text tokens", "runs": []}
    flip = False
    for _ in range(args.rounds):
        for which, batch, settings in CASES:
            order = settings[::-1] if flip else settings
            flip = not flip
            for remat in order:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--which", which, "--batch",
                                    str(batch), "--remat", str(int(remat)), "--iters", str(args.iters)],
                                   capture_output=True, text=True)
                line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                row = json.loads(line[-1]) if line else {"error": r.stderr[-400:]}
                res["runs"].append({"model": f"{CLASSES[which].__name__}-B/2", "batch": batch, "use_remat": remat,
                                    **row})
                print(json.dumps(res["runs"][-1]), flush=True)
    res["card_after"] = card()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
