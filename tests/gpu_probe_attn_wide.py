"""GPU probe for attention at head width 128 (run directly on a GPU machine; not a pytest file).

Prints the card's name and power limit, then the fused kernels (fdx_attention_fwd / fdx_attention_bwd at stored
width 128) and an unfused attention core (QK^T GEMM, f32 logits and bf16 probabilities in HBM, softmax, PV GEMM, and
its backward) at (B=32, h=8, L=Lk=1024), (32, 8, 256, 256) and (32, 8, 1024, 77): milliseconds per call as
min / median / max over repeated CUDA-event windows, TFLOP/s from true-width FLOPs (forward 4 B h L Lk d; backward
10 B h L Lk d, the FlashAttention count that includes the recomputed logits) and the peak memory each call adds over
its inputs and outputs, next to the size of the (B, h, L, Lk) f32 logits.

usage: python tests/gpu_probe_attn_wide.py [--iters 20] [--rounds 3]"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN  # noqa: E402

dev = torch.device("cuda")
BF16, F32 = torch.bfloat16, torch.float32


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


def peak_extra(fn):
    """bytes the call allocates at its peak beyond what is live before it (the caller keeps outputs alive)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    keep = fn()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    del keep
    return extra


def unfused_fwd(q, k, v, heads, dp, scale):
    """Attention as separate launches: S f32 and P in HBM."""
    Bn, L, HD = q.shape
    Lkp = k.shape[1]
    S = torch.empty((Bn, heads, L, Lkp), dtype=F32, device=dev)
    ops.gemm(GEMM_KK, q, k, S, L, Lkp, dp, HD, HD, Lkp, batch1=heads, batch2=Bn,
             a_s=(dp, L * HD), b_s=(dp, Lkp * HD), d_s=(L * Lkp, heads * L * Lkp), alpha=scale)
    P = ops.softmax_fwd(S, valid=unfused_fwd.valid)
    del S
    o = torch.empty((Bn * L, HD), dtype=BF16, device=dev)
    ops.gemm(GEMM_KMN, P, v, o, L, dp, Lkp, Lkp, HD, HD, batch1=heads, batch2=Bn,
             a_s=(L * Lkp, heads * L * Lkp), b_s=(dp, Lkp * HD), d_s=(dp, L * HD))
    return o, P


def unfused_bwd(q, k, v, P, do, heads, dp, scale, valid):
    """The backward of unfused_fwd: dP f32 and dS in HBM."""
    Bn, L, HD = q.shape
    Lkp = k.shape[1]
    dv = torch.empty((Bn, Lkp, HD), dtype=BF16, device=dev)
    ops.gemm(GEMM_MNMN, P, do, dv, Lkp, dp, L, Lkp, HD, HD, batch1=heads, batch2=Bn,
             a_s=(L * Lkp, heads * L * Lkp), b_s=(dp, L * HD), d_s=(dp, Lkp * HD))
    dP = torch.empty((Bn, heads, L, Lkp), dtype=F32, device=dev)
    ops.gemm(GEMM_KK, do, v, dP, L, Lkp, dp, HD, HD, Lkp, batch1=heads, batch2=Bn,
             a_s=(dp, L * HD), b_s=(dp, Lkp * HD), d_s=(L * Lkp, heads * L * Lkp))
    dS = ops.softmax_bwd(P, dP, scale, valid=valid)
    del dP
    dq = torch.empty((Bn * L, HD), dtype=BF16, device=dev)
    ops.gemm(GEMM_KMN, dS, k, dq, L, dp, Lkp, Lkp, HD, HD, batch1=heads, batch2=Bn,
             a_s=(L * Lkp, heads * L * Lkp), b_s=(dp, Lkp * HD), d_s=(dp, L * HD))
    dk = torch.empty((Bn, Lkp, HD), dtype=BF16, device=dev)
    ops.gemm(GEMM_MNMN, dS, q, dk, Lkp, dp, L, Lkp, HD, HD, batch1=heads, batch2=Bn,
             a_s=(L * Lkp, heads * L * Lkp), b_s=(dp, L * HD), d_s=(dp, Lkp * HD))
    return dq, dk, dv


def kernels(args, info):
    d = 128
    for B, h, L, Lk in ((32, 8, 1024, 1024), (32, 8, 256, 256), (32, 8, 1024, 77)):
        torch.manual_seed(0)
        HD = h * d
        q, k, v, do = (torch.randn(B, n, HD, device=dev).bfloat16() for n in (L, Lk, Lk, L))
        scale = d ** -0.5
        fl_f, fl_b = 4.0 * B * h * L * Lk * d, 10.0 * B * h * L * Lk * d
        logits_gb = B * h * L * Lk * 4 / 1e9
        o, lse = ops.attention_fwd(q, k, v, h, d, scale)
        tf = timed(lambda: ops.attention_fwd(q, k, v, h, d, scale, out=o), args.iters, args.rounds)
        tb = timed(lambda: ops.attention_bwd(q, k, v, o, lse, do, h, d, scale), args.iters, args.rounds)
        mf = peak_extra(lambda: ops.attention_fwd(q, k, v, h, d, scale))
        mb = peak_extra(lambda: ops.attention_bwd(q, k, v, o, lse, do, h, d, scale))
        # unfused: keys zero-padded to a multiple of 32 for the tensor-core tiles
        Lkp = (Lk + 31) // 32 * 32
        kp = torch.zeros(B, Lkp, HD, device=dev, dtype=BF16)
        vp = torch.zeros(B, Lkp, HD, device=dev, dtype=BF16)
        kp[:, :Lk], vp[:, :Lk] = k, v
        unfused_fwd.valid = Lk
        ou, P = unfused_fwd(q, kp, vp, h, d, scale)
        err = ((ou.view(B, L, HD).float() - o.float()).norm() / o.float().norm()).item()
        tuf = timed(lambda: unfused_fwd(q, kp, vp, h, d, scale), args.iters, args.rounds)
        tub = timed(lambda: unfused_bwd(q, kp, vp, P, do, h, d, scale, Lk), args.iters, args.rounds)
        del ou, P
        name = f"B={B} h={h} L={L} Lk={Lk} d=128"
        for what, t, fl, mem in (("fused fwd", tf, fl_f, mf), ("fused bwd", tb, fl_b, mb),
                                 ("unfused fwd", tuf, fl_f, None), ("unfused bwd", tub, fl_b, None)):
            extra = "" if mem is None else f"  peak extra memory {mem / 1e9:.3f} GB (f32 logits: {logits_gb:.2f} GB)"
            print(f"[{info}] {name} {what}: {t[0]:.3f} / {t[1]:.3f} / {t[2]:.3f} ms (min/median/max)  "
                  f"{fl / t[1] / 1e9:.1f} TFLOP/s{extra}", flush=True)
        print(f"[{info}] {name} fused vs unfused output: {err:.2e} relative L2; speed-up fwd {tuf[1] / tf[1]:.2f}x, "
              f"bwd {tub[1] / tb[1]:.2f}x", flush=True)
        del q, k, v, do, o, lse, kp, vp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    print(f"card: {info}", flush=True)
    kernels(args, info)


if __name__ == "__main__":
    main()
