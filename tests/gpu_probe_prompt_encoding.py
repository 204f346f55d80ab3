"""Measure what encoding prompts adds to a DiffusionInferencePipeline.generate_samples call (not a test; run by hand on
an H100):

    python tests/gpu_probe_prompt_encoding.py [--out results.json]

A CLIP ViT-L/14-shaped text tower (12 x 768, 12 heads, MLP 3072, 77 tokens, random weights) on the engine at B = 32,
with CUDA events around each call after warm-up: the tower alone (CLIPTextTower.encode on device tokens) and the
whole CLIPTextEncoder call a raw prompt list takes (host tokenizer stand-in, token upload, tower).  Compare with
bench.py's `sample_256_text_cfg` (30 CFG Euler-ancestral steps, B = 32, 256 x 256).  The card's name and power limit
are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from clip_text_ref import Tok, clip_model  # noqa: E402

from flaxdiff_b200.inputs import CLIPTextEncoder  # noqa: E402


def timed_ms(fn, reps):
    times = []
    for _ in range(reps):
        s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        fn()
        s1.record()
        torch.cuda.synchronize()
        times.append(s0.elapsed_time(s1))
    times.sort()
    return {"median_ms": times[len(times) // 2], "min_ms": times[0], "max_ms": times[-1], "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    enc = CLIPTextEncoder(clip_model("clip-l"), Tok(49408), modelname="clip-l-random", backend="fdx",
                          device=torch.device("cuda"))
    prompts = [f"a photograph of object number {i} on a wooden table, studio light" for i in range(args.batch)]
    tok = enc.tokenize(prompts)
    ids = tok["input_ids"].to("cuda", torch.int32).contiguous()
    mask = tok["attention_mask"].to("cuda", torch.int32).contiguous()
    for _ in range(5):
        enc.tower.encode(ids, mask)
        enc(prompts)
    torch.cuda.synchronize()
    res = {"gpu": gpu, "batch": args.batch,
           "tower_encode": timed_ms(lambda: enc.tower.encode(ids, mask), args.reps),
           "encoder_call_with_tokenizer": timed_ms(lambda: enc(prompts), args.reps)}
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
