"""Measure the CLIP text tower on the engine against transformers on the same GPU (not a test; run by hand on an H100):

    python tests/gpu_probe_clip_text.py [--out results.json] [--skip-train]

1. The tower alone, CLIP ViT-L/14 text shapes (12 x 768, 12 heads, MLP 3072, 77 tokens, random weights) at B = 32
   and 256: the engine (CLIPTextTower.encode), transformers' CLIPTextModel in f32 (what CLIPTextEncoder(device=
   "cuda") runs) and in bf16, alternated in rounds after warm-up, CUDA events around each call.  TFLOP/s from
   2 (3 D^2 + D^2 + 2 D I) + 4 T D FLOP per token and layer.
2. Where the engine's time goes: CUDA events around each kernel of one encode at B = 256.
3. One text-conditioned training step (C4's UNet at 256 x 256, B = 32, pretokenized batches, CUDA graph) with the
   text tower in transformers f32 outside the graph (backend "torch") and on the engine inside it (backend "fdx").
The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from clip_text_ref import Tok, clip_model, token_batch  # noqa: E402

from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200.models.clip_text import CLIPTextTower  # noqa: E402

dev = torch.device("cuda")


def flop_per_seq(cfg, T=77):
    D, I = cfg.hidden_size, cfg.intermediate_size
    return cfg.num_hidden_layers * T * (2 * (4 * D * D + 2 * D * I) + 4 * T * D)


def timed(fn, reps):
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(reps):
        fn()
    s1.record()
    torch.cuda.synchronize()
    return s0.elapsed_time(s1) / reps


def tower_alone(model, tower, B, rounds=5, reps=5):
    ids, mask = token_batch(model.config.vocab_size, [int(n) for n in torch.arange(B) * 7 % 76], seed=B)
    ids, mask = ids.to(dev), mask.to(dev)
    m32 = model.to(dev)
    m16 = clip_model("clip-l").to(dev, torch.bfloat16)
    variants = {
        "engine": lambda: tower.encode(ids, mask),
        "transformers_f32": lambda: m32(input_ids=ids, attention_mask=mask).last_hidden_state,
        "transformers_bf16": lambda: m16(input_ids=ids, attention_mask=mask).last_hidden_state,
    }
    with torch.no_grad():
        for f in variants.values():
            f(), f()
        torch.cuda.synchronize()
        ms = {k: [] for k in variants}
        for _ in range(rounds):
            for k, f in variants.items():
                ms[k].append(timed(f, reps))
    fl = flop_per_seq(model.config) * B
    out = {}
    for k, v in ms.items():
        best, med = min(v), sorted(v)[len(v) // 2]
        out[k] = {"ms_median": med, "ms_min": best, "tflops_median": fl / (med / 1e3) / 1e12}
    m32.to("cpu")
    del m16
    return out


def engine_breakdown(model, tower, B=256, reps=10):
    """CUDA events around every launch of one encode (the loop of CLIPTextTower.encode, instrumented)."""
    ids, mask = token_batch(model.config.vocab_size, [int(n) for n in torch.arange(B) * 7 % 76], seed=1)
    ids, mask = ids.to(dev, torch.int32), mask.to(dev, torch.int32)
    T, D, w = 77, tower.D, tower.w
    acc = {}

    def ev(name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        acc.setdefault(name, []).append((a, b))

    for it in range(reps + 2):
        if it == 2:
            acc.clear()
        h = ops.token_embed(ids, w["tok"], w["pos"])
        h2 = h.view(B * T, D)
        x = torch.empty((B * T, D), dtype=torch.bfloat16, device=dev)
        qkv = torch.empty((B, T, 3 * D), dtype=torch.bfloat16, device=dev)
        o = torch.empty((B, T, D), dtype=torch.bfloat16, device=dev)
        u = torch.empty((B * T, tower.inner), dtype=torch.bfloat16, device=dev)
        ev("token_embed", lambda: ops.token_embed(ids, w["tok"], w["pos"], out=h))
        for i in range(tower.layers):
            ev("layernorm", lambda: ops.layernorm_fwd(h2, w[f"{i}.ln1_g"], w[f"{i}.ln1_b"], tower.eps, out=x))
            ev("gemm_qkv", lambda: ops.linear_fwd(x, w[f"{i}.wqkv"], out=qkv.view(B * T, 3 * D), bias=w[f"{i}.bqkv"]))
            ev("attention_masked", lambda: ops.attention_fwd_masked(qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:],
                                                                    tower.heads, tower.dh, tower.scale, True, mask,
                                                                    out=o))
            ev("gemm_out_proj", lambda: ops.linear_fwd(o.view(B * T, D), w[f"{i}.wo"], out=h2, bias=w[f"{i}.bo"],
                                                       res=h2))
            ev("layernorm", lambda: ops.layernorm_fwd(h2, w[f"{i}.ln2_g"], w[f"{i}.ln2_b"], tower.eps, out=x))
            ev("gemm_fc1", lambda: ops.linear_fwd(x, w[f"{i}.w1"], out=u))
            ev("bias_act", lambda: ops.bias_act(u, w[f"{i}.b1"], tower.act, out=u))
            ev("gemm_fc2", lambda: ops.linear_fwd(u, w[f"{i}.w2"], out=h2, bias=w[f"{i}.b2"], res=h2))
        ev("layernorm", lambda: ops.layernorm_fwd(h2, w["lnf_g"], w["lnf_b"], tower.eps))
    torch.cuda.synchronize()
    return {k: sum(a.elapsed_time(b) for a, b in v) / reps for k, v in acc.items()}


def train_step_compare(steps=10, rounds=2):
    from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.schedulers import EDMNoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    res, B = 256, 32
    conds = {}
    for backend in ("torch", "fdx"):
        enc = CLIPTextEncoder(clip_model("clip-l"), Tok(49408), modelname="random-clip-l", backend=backend,
                              device=dev)
        conds[backend] = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True,
                                                unconditional_input="")
    model = Unet(attention_configs=(None, {"heads": 8}, {"heads": 8}, {"heads": 8}), dtype=torch.bfloat16)
    cfg = DiffusionInputConfig("image", (res, res, 3), [conds["fdx"]])
    tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5), cfg,
                                 rngs=4, unconditional_prob=0.12, model_output_transform=KarrasPredictionTransform(0.5),
                                 device=dev, use_cuda_graph=True)
    g = torch.Generator().manual_seed(0)
    ids, mask = token_batch(49408, [int(n) for n in torch.randint(0, 76, (B,), generator=g)], seed=2)
    batch = {"image": torch.randint(0, 256, (B, res, res, 3), generator=g, dtype=torch.uint8),
             "text": {"input_ids": ids, "attention_mask": mask}}
    step = tr._define_train_step()
    rng = tr.rngstate
    ms = {k: [] for k in conds}
    for _ in range(rounds):
        for backend, cond in conds.items():
            cfg.conditions[0] = cond
            tr._graph, tr._null_tokens = None, None          # recapture for this encoder
            for _ in range(2):
                _, loss, rng = step(tr.state, rng, batch)
            torch.cuda.synchronize()
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(steps):
                _, loss, rng = step(tr.state, rng, batch)
            s1.record()
            torch.cuda.synchronize()
            ms[backend].append(s0.elapsed_time(s1) / steps)
    return {k: {"ms_per_step": sorted(v)[len(v) // 2], "all": v} for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_probe_clip_text needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    model = clip_model("clip-l")
    tower = CLIPTextTower.from_transformers(model, dev)
    res = {"card": card, "gflop_per_sequence": flop_per_seq(model.config) / 1e9, "tower": {}}
    for B in (32, 256):
        res["tower"][B] = tower_alone(model, tower, B)
        print(f"tower B={B}:", json.dumps(res["tower"][B]), flush=True)
    res["engine_ms_per_kernel_B256"] = engine_breakdown(model, tower)
    print("engine per kernel (ms, B=256):", json.dumps(res["engine_ms_per_kernel_B256"]), flush=True)
    if not args.skip_train:
        res["train_step_c4_256_B32"] = train_step_compare()
        print("train step:", json.dumps(res["train_step_c4_256_B32"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
