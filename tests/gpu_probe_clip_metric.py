"""Measure the CLIP metrics on the engine against transformers on the same GPU (not a test; run by hand on an H100):

    python tests/gpu_probe_clip_metric.py [--out results.json]

1. One metric evaluation (samples -> clip_similarity and clip_score) with CLIP ViT-L/14's shapes (random weights) at
   B = 32 and 256 on 64^2 and 256^2 samples: the engine (CLIPPair.similarity, preprocessing included), and
   transformers' CLIPModel in f32 and in bf16 fed by CLIPImageProcessorPil on the host (the reference's path: quantise,
   processor, copy, model, cosine).  Variants alternate in rounds after warm-up; a host clock around work that ends
   in a device synchronise.  The vision tower is 2 (4 D^2 + 2 D I) + 4 L D FLOP per token and layer, L = 257.
2. One validation_loop of a text-conditioned trainer (64^2 UNet, B = 32, 20 Euler steps) with and without both
   metrics, alternated.
The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from clip_metric_ref import clip_pair_model  # noqa: E402
from clip_text_ref import Tok, clip_model, token_batch  # noqa: E402

from flaxdiff_b200.models.clip_vision import CLIPPair  # noqa: E402

dev = torch.device("cuda")


def vision_flop_per_image(cfg):
    D, I, L = cfg.hidden_size, cfg.intermediate_size, (cfg.image_size // cfg.patch_size) ** 2 + 1
    return cfg.num_hidden_layers * L * (2 * (4 * D * D + 2 * D * I) + 4 * L * D) + 2 * (L - 1) * 3 * \
        cfg.patch_size ** 2 * D


def wall(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def transformers_metric(model, proc, dtype):
    def run(x, ids, mask):
        u8 = (((x.cpu().numpy() + np.float32(1)) / np.float32(2)) * np.float32(255)).astype(np.uint8)
        pv = proc(images=list(u8), return_tensors="pt")["pixel_values"].to(dev, dtype)
        with torch.no_grad():
            out = model(pixel_values=pv, input_ids=ids, attention_mask=mask)
        a = out.image_embeds.float() / (out.image_embeds.float().norm(dim=-1, keepdim=True) + 1e-6)
        t = out.text_embeds.float() / (out.text_embeds.float().norm(dim=-1, keepdim=True) + 1e-6)
        cos = (a * t).sum(-1)
        return (1 - cos).mean().item(), (100 * cos.clamp_min(0)).mean().item()
    return run


def metric_alone(pair, m32, m16, proc, B, res, rounds=3, reps=2):
    g = torch.Generator().manual_seed(B + res)
    x = (torch.rand(B, res, res, 3, generator=g) * 2 - 1).to(dev)
    ids, mask = token_batch(49408, [int(n) for n in torch.arange(B) * 7 % 76], seed=B)
    ids, mask = ids.to(dev), mask.to(dev)
    variants = {"engine": lambda: pair.similarity(x, ids, mask)[1].tolist(),
                "transformers_f32": lambda: transformers_metric(m32, proc, torch.float32)(x, ids, mask),
                "transformers_bf16": lambda: transformers_metric(m16, proc, torch.bfloat16)(x, ids, mask)}
    values = {k: f() for k, f in variants.items()}
    times = {k: [] for k in variants}
    for _ in range(rounds):
        for k, f in variants.items():
            times[k].append(wall(f, reps))
    return {k: {"ms_median": float(np.median(v)), "ms_all": v, "metrics": values[k]} for k, v in times.items()}


def validation(pair_name):
    from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig
    from flaxdiff_b200.metrics import get_clip_metric, get_clip_score_metric
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.samplers import EulerSampler
    from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    enc = CLIPTextEncoder(clip_model("clip-l"), Tok(49408), modelname="clip-l-random", backend="fdx")
    cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True, unconditional_input="")
    torch.manual_seed(0)
    model = Unet(attention_configs=(None, None, {"heads": 8}, {"heads": 8}), dtype=torch.bfloat16)
    tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (64, 64, 3), [cond]), rngs=4,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev)
    step = tr._define_validation_step(EulerSampler, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5))
    ids, mask = token_batch(49408, [int(n) for n in torch.arange(32) * 5 % 76], seed=1)

    def val_ds():
        while True:
            yield {"text": {"input_ids": ids, "attention_mask": mask}}

    metrics = [get_clip_metric(pair_name), get_clip_score_metric(pair_name)]
    runs = {"without_metrics": None, "with_metrics": metrics}
    times = {k: [] for k in runs}
    for r in range(4):
        for k, m in runs.items():
            tr.eval_metrics = m
            t = wall(lambda: tr.validation_loop(tr.state, step, val_ds, 1, 0, 20), 1)
            if r:                                              # round 0 warms up (graph capture)
                times[k].append(t)
    return {k: {"ms_median": float(np.median(v)), "ms_all": v} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    from transformers.models.clip import CLIPImageProcessorPil

    from flaxdiff_b200.metrics import images
    proc = CLIPImageProcessorPil()
    m32 = clip_pair_model("vit-l")
    pair = CLIPPair.from_transformers(m32, proc, dev)
    m16 = clip_pair_model("vit-l").to(dev, torch.bfloat16)
    m32 = m32.to(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"gpu": gpu, "vision_gflop_per_image": vision_flop_per_image(m32.config.vision_config) / 1e9, "metric": {}}
    for B in (32, 256):
        for r in (64, 256):
            res["metric"][f"B{B}_{r}px"] = metric_alone(pair, m32, m16, proc, B, r)
            print(f"B={B} {r}px:", {k: round(v["ms_median"], 2) for k, v in res["metric"][f"B{B}_{r}px"].items()},
                  flush=True)
    del m32, m16
    torch.cuda.empty_cache()
    images._clip_cache["vit-l-random"] = pair
    res["validation_loop"] = validation("vit-l-random")
    print("validation_loop:", {k: round(v["ms_median"], 1) for k, v in res["validation_loop"].items()})
    print("gpu:", gpu)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
