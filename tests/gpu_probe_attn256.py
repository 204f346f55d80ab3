"""GPU probe for attention at head width 256 (run directly on a GPU machine; not a pytest file).

Prints the card's name and power limit, then, at the UNet shapes of 2-head attention on 512 channels (256-wide
heads): self-attention at L = Lk = 64, 256 and 1024 (the 8², 16² and 32² levels) and cross-attention from 1024
queries to 77 text keys, with B as in the C2 (64², B = 256) and C3 (256², B = 32) workloads:
  - the fused kernels (fdx_attention_fwd, and forward + fdx_attention_bwd),
  - torch.nn.functional.scaled_dot_product_attention on the same bf16 tensors (the yardstick),
as milliseconds per call (min / median / max over CUDA-event windows) and TFLOP/s (forward 4 B h L Lk d, forward
+ backward 14 B h L Lk d: the FlashAttention count with the recomputed logits).  Then one EDM training step at the
C2 shape (64², B = 256) of the default UNet with 2-head attention at levels 1-3 against the same UNet with 8 heads,
and a 256² step (B = 8) of the 2-head UNet.

usage: python tests/gpu_probe_attn256.py [--iters 20] [--rounds 3]"""
import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200 import ops  # noqa: E402

dev = torch.device("cuda")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        out = f"{torch.cuda.get_device_name(0)}, power limit unknown"
    return out


def timed(fn, iters, rounds):
    """ms per call: (min, median, max) over `rounds` CUDA-event windows of `iters` calls each."""
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
    return min(ms), statistics.median(ms), max(ms)


def fmt(t, flop):
    return f"{t[0]:8.3f} {t[1]:8.3f} {t[2]:8.3f} ms  {flop / t[1] / 1e9:6.1f} TFLOP/s"


def attention(B, heads, L, Lk, iters, rounds):
    d = 256
    HD = heads * d
    q = torch.randn(B, L, HD, device=dev).bfloat16()
    k = torch.randn(B, Lk, HD, device=dev).bfloat16()
    v = torch.randn(B, Lk, HD, device=dev).bfloat16()
    do = torch.randn(B, L, HD, device=dev).bfloat16()
    sc = d ** -0.5
    o, lse = ops.attention_fwd(q, k, v, heads, d, sc)
    fl_f, fl_fb = 4 * B * heads * L * Lk * d, 14 * B * heads * L * Lk * d

    def fused_fb():
        o2, l2 = ops.attention_fwd(q, k, v, heads, d, sc)
        ops.attention_bwd(q, k, v, o2, l2, do, heads, d, sc)
    t_f = timed(lambda: ops.attention_fwd(q, k, v, heads, d, sc), iters, rounds)
    t_fb = timed(fused_fb, iters, rounds)
    # SDPA on [B, h, L, d] views of the same tensors
    qs = q.view(B, L, heads, d).transpose(1, 2).detach().requires_grad_(True)
    ks = k.view(B, Lk, heads, d).transpose(1, 2).detach().requires_grad_(True)
    vs = v.view(B, Lk, heads, d).transpose(1, 2).detach().requires_grad_(True)
    dos = do.view(B, L, heads, d).transpose(1, 2)

    def sdpa_f():
        with torch.no_grad():
            return F.scaled_dot_product_attention(qs, ks, vs, scale=sc)

    def sdpa_fb():
        out = F.scaled_dot_product_attention(qs, ks, vs, scale=sc)
        torch.autograd.grad(out, (qs, ks, vs), dos)
    s_f = timed(sdpa_f, iters, rounds)
    s_fb = timed(sdpa_fb, iters, rounds)
    ref = sdpa_f().transpose(1, 2).reshape(B, L, HD).float()
    err = ((o.float() - ref).norm() / ref.norm()).item()
    tag = f"B={B:3d} h={heads} L={L:4d} Lk={Lk:4d}"
    print(f"{tag}  fused fwd     {fmt(t_f, fl_f)}   sdpa fwd     {fmt(s_f, fl_f)}   rel(o, sdpa)={err:.1e}")
    print(f"{tag}  fused fwd+bwd {fmt(t_fb, fl_fb)}   sdpa fwd+bwd {fmt(s_fb, fl_fb)}")


def train_step(levels, res, B, iters, rounds):
    from flaxdiff_b200.inputs import DiffusionInputConfig
    from flaxdiff_b200.models.simple_unet import Unet
    from flaxdiff_b200.predictors import KarrasPredictionTransform
    from flaxdiff_b200.schedulers import EDMNoiseScheduler
    from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
    model = Unet(attention_configs=levels, dtype=torch.bfloat16)
    tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 DiffusionInputConfig("image", (res, res, 3), []), rngs=4,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 use_cuda_graph=True)
    step = tr._define_train_step(B)
    img = torch.randint(0, 256, (B, res, res, 3), dtype=torch.uint8, device=dev)
    box = {}

    def one():
        tr.state, box["loss"], tr.rngstate = step(tr.state, tr.rngstate, {"image": img}, 0)
    t = timed(one, iters, rounds)
    print(f"train step {res}x{res} B={B} heads={levels[1]['heads']}: {t[0]:.2f} / {t[1]:.2f} / {t[2]:.2f} ms  "
          f"({B / t[1] * 1e3:.0f} img/s)  loss {float(box['loss']):.4f}")
    del tr, model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print(card())
    for B, L, Lk in ((256, 64, 64), (32, 256, 256), (32, 1024, 1024), (32, 1024, 77), (256, 64, 77)):
        attention(B, 2, L, Lk, a.iters, a.rounds)
    two = (None, {"heads": 2}, {"heads": 2}, {"heads": 2})
    eight = (None, {"heads": 8}, {"heads": 8}, {"heads": 8})
    train_step(two, 64, 256, 5, a.rounds)
    train_step(eight, 64, 256, 5, a.rounds)
    train_step(two, 256, 8, 3, a.rounds)


if __name__ == "__main__":
    main()
