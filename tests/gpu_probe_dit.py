"""SimpleDiT on one H100: graphed training step and Euler step (img/s), the new streaming kernels' times against their
HBM floor, and the same model's training step in torch bf16 (SDPA + autograd) for comparison.

    python tests/gpu_probe_dit.py [--out results.json]

Configs: DiT-B/2 at 64x64 (L = 1024), B = 256, and DiT-B/4 at 256x256 (L = 4096), B = 32.  Times are CUDA events
around warmed-up work; the card's name and power limit are read in the same run."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200._lib import ACT_GELU_TANH  # noqa: E402
from flaxdiff_b200.inputs import DiffusionInputConfig  # noqa: E402
from flaxdiff_b200.models.simple_dit import SimpleDiT  # noqa: E402
from flaxdiff_b200.predictors import KarrasPredictionTransform  # noqa: E402
from flaxdiff_b200.samplers import EulerSampler  # noqa: E402
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler  # noqa: E402
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw  # noqa: E402
from oracle import dit_ref  # noqa: E402

dev = torch.device("cuda")
HBM = 3.35e12          # H100 SXM data sheet, bytes/s
CONFIGS = [("DiT-B/2 64x64", dict(patch_size=2), 64, 256), ("DiT-B/4 256x256", dict(patch_size=4), 256, 32)]
BASE = dict(emb_features=768, num_layers=12, num_heads=12)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def kernels(B, L, F, heads):
    """Each new streaming kernel at the config's shapes: seconds and share of the HBM floor (bytes / 3.35 TB/s)."""
    M, HD, E = B * L, heads * 64, 4 * F
    x = torch.randn(M, F, device=dev).bfloat16()
    y = torch.randn(M, F, device=dev).bfloat16()
    ada = torch.randn(B, 6 * F, device=dev)
    dada = torch.empty_like(ada)
    _, mean, rstd = ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F)
    qkv = torch.randn(M, 3 * HD, device=dev).bfloat16()
    u = torch.randn(M, E, device=dev).bfloat16()
    du = torch.randn(M, E, device=dev).bfloat16()
    t2 = M * F * 2
    cases = {
        "adaln_fwd": (lambda: ops.dit_adaln_fwd(x, L, ada, 3 * F, 4 * F), 2 * t2),
        "adaln_bwd": (lambda: ops.dit_adaln_bwd(x, y, L, mean, rstd, dada[:, :F], dada[:, F:2 * F], ada=ada,
                                                addend=x), 6 * t2),
        "gate_fwd": (lambda: ops.dit_gate_fwd(x, y, L, ada[:, 5 * F:]), 3 * t2),
        "gate_bwd": (lambda: ops.dit_gate_bwd(x, y, L, ada[:, 5 * F:], dada[:, 5 * F:]), 3 * t2),
        "rope": (lambda: ops.dit_rope(qkv, L, heads, 64, 64, nmat=2, mat_off=HD), 2 * 2 * M * HD * 2),
        "gelu_tanh_fwd": (lambda: ops.bias_act(u, None, ACT_GELU_TANH), 2 * M * E * 2),
        "gelu_tanh_bwd": (lambda: ops.bias_act_bwd(u, None, ACT_GELU_TANH, du), 3 * M * E * 2),
    }
    out = {}
    for k, (fn, nbytes) in cases.items():
        s = timed(fn, 20)
        out[k] = {"us": round(s * 1e6, 1), "hbm_floor_share": round(nbytes / HBM / s, 3)}
    return out


def torch_step_fn(P, x, t, freqs, p, heads, eps=1e-5):
    """The same model in torch bf16: the oracle's formulas with F.scaled_dot_product_attention, autograd backward."""
    def rope(z):
        L_, d = z.shape[1], z.shape[3]
        inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float32, device=z.device) / d))
        fr = torch.arange(L_, dtype=torch.float32, device=z.device)[:, None] * inv[None]
        cos = torch.cat([fr.cos(), fr.cos()], -1)[None, :, None, :].to(z.dtype)
        sin = torch.cat([fr.sin(), fr.sin()], -1)[None, :, None, :].to(z.dtype)
        return z * cos + torch.cat([-z[..., d // 2:], z[..., :d // 2]], -1) * sin

    def attention(base, h):
        B_, L_, F_ = h.shape
        q = (torch.einsum("blf,fhd->blhd", h, P[base + "/to_q/kernel"]) + P[base + "/to_q/bias"])
        k = (torch.einsum("blf,fhd->blhd", h, P[base + "/to_k/kernel"]) + P[base + "/to_k/bias"])
        v = (torch.einsum("blf,fhd->blhd", h, P[base + "/to_v/kernel"]) + P[base + "/to_v/bias"])
        q, k = rope(q), rope(k)
        o = Fn.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2)
        return torch.einsum("blhd,hdf->blf", o, P[base + "/to_out_0/kernel"]) + P[base + "/to_out_0/bias"]

    HP0 = x.shape[1] // p
    pos = torch.from_numpy(dit_ref.sincos_2d(P["patch_embed/Conv_0/bias"].shape[0], HP0, x.shape[2] // p)).to(
        x.device, x.dtype)

    def run():
        B_, H_, W_, C_ = x.shape
        HP, WP = H_ // p, W_ // p
        Fd = P["patch_embed/Conv_0/bias"].shape[0]
        tok = x.reshape(B_, HP, p, WP, p, C_).permute(0, 1, 3, 2, 4, 5).reshape(B_, HP * WP, -1)
        tok = tok @ P["patch_embed/Conv_0/kernel"].reshape(-1, Fd) + P["patch_embed/Conv_0/bias"]
        cond = dit_ref.time_embed({k: v.float() for k, v in P.items() if k.startswith("time_embed")}, t,
                                  freqs).to(x.dtype)
        tok = tok + pos
        i = 0
        while f"dit_block_{i}/mlp/layers_0/kernel" in P:
            n = f"dit_block_{i}"
            ada = dit_ref.dense(P, f"{n}/ada_params_module/ada_proj", cond)[:, None, :]
            sc_m, sh_m, g_m, sc_a, sh_a, g_a = ada.chunk(6, -1)
            tok = tok + g_a * attention(f"{n}/attention", Fn.layer_norm(tok, (Fd,), eps=eps) * (1 + sc_a) + sh_a)
            hh = Fn.layer_norm(tok, (Fd,), eps=eps) * (1 + sc_m) + sh_m
            hh = dit_ref.dense(P, f"{n}/mlp/layers_2", Fn.gelu(dit_ref.dense(P, f"{n}/mlp/layers_0", hh),
                                                                 approximate="tanh"))
            tok = tok + g_m * hh
            i += 1
        out = Fn.layer_norm(tok, (Fd,), P["final_norm/scale"], P["final_norm/bias"], eps)
        out = dit_ref.dense(P, "final_proj", out)
        loss = out.float().square().mean()
        loss.backward()
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    res = {"card": card(), "configs": {}}
    print(res["card"], flush=True)
    for name, kw, r, B in CONFIGS:
        row = {}
        model = SimpleDiT(**kw, **BASE)
        L = (r // kw["patch_size"]) ** 2
        try:
            tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                         DiffusionInputConfig("image", (r, r, 3), []), rngs=4,
                                         model_output_transform=KarrasPredictionTransform(0.5), device=dev)
            step = tr._define_train_step()
            batch = {"image": torch.randint(0, 256, (B, r, r, 3), dtype=torch.uint8, device=dev)}
            st = [tr.state, tr.rngstate]

            def train():
                st[0], _, st[1] = step(st[0], st[1], batch)
            s = timed(train, args.iters)
            row["train_step_ms"] = round(s * 1e3, 2)
            row["train_img_per_s"] = round(B / s, 1)
        except torch.cuda.OutOfMemoryError as e:
            row["train_error"] = f"out of memory: {str(e)[:120]}"
        tr = step = st = train = None          # the captured graph's memory pool goes with the trainer
        gc.collect()
        torch.cuda.empty_cache()
        try:
            fp = model.init(0, device=dev)
            smp = EulerSampler(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev),
                               KarrasPredictionTransform(0.5), DiffusionInputConfig("image", (r, r, 3), []))
            s12 = timed(lambda: smp.generate_samples(fp, B, r, diffusion_steps=12, start_step=1000, device=dev), 2,
                        warm=1)
            s2 = timed(lambda: smp.generate_samples(fp, B, r, diffusion_steps=2, start_step=1000, device=dev), 2,
                       warm=1)
            row["euler_step_ms"] = round((s12 - s2) / 10 * 1e3, 2)
            row["euler_img_steps_per_s"] = round(B / ((s12 - s2) / 10), 1)
        except torch.cuda.OutOfMemoryError as e:
            row["euler_error"] = f"out of memory: {str(e)[:120]}"
        smp = fp = None
        gc.collect()
        torch.cuda.empty_cache()
        row["kernels"] = kernels(B, L, 768, 12)
        torch.cuda.empty_cache()
        try:
            fp = model.init(0, device=dev)
            P = {k: v.detach().bfloat16().requires_grad_(True) for k, v in fp.named.items()}
            x = torch.randn(B, r, r, 3, device=dev).bfloat16()
            t = torch.rand(B, device=dev)
            s = timed(torch_step_fn(P, x, t, model._fourier_freqs(dev), kw["patch_size"], 12), args.iters)
            row["torch_bf16_step_ms"] = round(s * 1e3, 2)
        except torch.cuda.OutOfMemoryError as e:
            row["torch_error"] = f"out of memory: {str(e)[:120]}"
        P = fp = x = None
        gc.collect()
        torch.cuda.empty_cache()
        res["configs"][name] = row
        print(name, json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
