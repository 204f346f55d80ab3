"""SimpleMMDiT and HierarchicalMMDiT on one H100: the fdx_mmdit.cu kernels against their HBM floor, one MMDiT block
against one DiTBlock (forward + backward), and graphed training-step and Euler-step throughput.

    python tests/gpu_probe_mmdit.py --which kernels|mmdit|dit|hier|mmdit-euler|dit-euler|hier-euler [--out f.json]

Shapes: SimpleMMDiT-B/2 against SimpleDiT-B/2 at 64x64 (L = 1024), B = 256 for training and B = 64 for the Euler step
(B = 256 runs out of memory in the sampler for both), F = 768, 12 layers, 12 heads; HierarchicalMMDiT at its class
defaults (base patch 8, F (512, 768, 1024), layers (4, 4, 14), heads (8, 12, 16)) at 256x256, B = 32.  The text context
is random bf16 [B, 77, 768] (SimpleDiT is given the same).  Each --which runs in its own process: a training graph and
a sampler in one process exhaust memory.  Times are CUDA events around warmed-up work; the card's name and power limit
are read in the same run."""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200.inputs import ConditionalInputConfig, DiffusionInputConfig, RandomEmbeddingEncoder  # noqa: E402
from flaxdiff_b200.models.mmdit import HierarchicalMMDiT, SimpleMMDiT  # noqa: E402
from flaxdiff_b200.models.simple_dit import SimpleDiT  # noqa: E402
from flaxdiff_b200.predictors import KarrasPredictionTransform  # noqa: E402
from flaxdiff_b200.samplers import EulerSampler  # noqa: E402
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler  # noqa: E402
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw  # noqa: E402
from gpu_probe_dit import HBM, card, timed  # noqa: E402

dev = torch.device("cuda")
P, RES, BATCH, F = 2, 64, 256, 768
EULER_BATCH = 64
BASE = dict(patch_size=P, emb_features=F, num_layers=12, num_heads=12)
HIER_RES, HIER_BATCH = 256, 32


def kernels(B, L, C):
    """Each kernel's time and share of its HBM floor: the bytes it must move at least once (bf16 rows)."""
    M = B * L
    g = torch.Generator(device=dev).manual_seed(0)
    r = lambda: torch.randn(M, C, generator=g, device=dev).bfloat16()  # noqa: E731
    x, a, m, add = r(), r(), r(), r()
    ada = torch.randn(B, 6 * C, generator=g, device=dev) * 0.5
    dada = torch.empty_like(ada)
    _, _, mean, rstd = ops.mmdit_adaln_fwd(x, L, ada)
    cases = (("adaln_fwd", lambda: ops.mmdit_adaln_fwd(x, L, ada), 6 * C * M),          # x in, two rows out
             ("adaln_bwd", lambda: ops.mmdit_adaln_bwd(x, a, m, L, ada, mean, rstd, dada, addend=add), 10 * C * M),
             ("gate_fwd", lambda: ops.mmdit_gate_fwd(x, a, m, L, ada), 8 * C * M),
             ("gate_bwd", lambda: ops.mmdit_gate_bwd(x, a, m, L, ada, dada), 10 * C * M))
    out = {}
    for k, fn, nbytes in cases:
        s = timed(fn, 20)
        out[k] = {"us": round(s * 1e6, 1), "hbm_floor_share": round(nbytes / HBM / s, 3)}
    # fdx_layernorm_rows at HierarchicalMMDiT's finest stage (F0 = 512, a 32 x 32 patch grid at 256^2, B = 32): the
    # floor is one read of the input and one write of y (forward); x and dy in, dx out (backward)
    Bh, G, F0 = HIER_BATCH, HIER_RES // 8, 512
    fine = torch.randn(Bh * G * G, F0, generator=g, device=dev).bfloat16()
    one, zero = torch.ones(4 * F0, device=dev), torch.zeros(4 * F0, device=dev)
    dg, db = torch.zeros(4 * F0, device=dev), torch.zeros(4 * F0, device=dev)
    rows_c = Bh * (G // 2) * (G // 2)
    coarse = torch.randn(rows_c, 4 * F0, generator=g, device=dev).bfloat16()
    ln = ops.layernorm_rows_fwd
    for k, mode, src in (("rows_gather", ops.LN_GATHER, fine), ("rows_scatter", ops.LN_SCATTER, coarse)):
        grid = (G // 2, G // 2)
        y, mu, rs = ln(mode, src, None, rows_c, 4 * F0, one, zero, grid=grid)
        nb = 2 * src.numel() * 2
        s = timed(lambda: ln(mode, src, None, rows_c, 4 * F0, one, zero, grid=grid), 20)
        row = {"fwd_us": round(s * 1e6, 1), "fwd_hbm_floor_share": round(nb / HBM / s, 3)}
        s = timed(lambda: ops.layernorm_rows_bwd(mode, src, None, y, rows_c, 4 * F0, one, mu, rs, dg, db, grid=grid),
                  20)
        row.update(bwd_us=round(s * 1e6, 1), bwd_hbm_floor_share=round(1.5 * nb / HBM / s, 3))
        out[k] = row
    skip = torch.randn(Bh * G * G, F0, generator=g, device=dev).bfloat16()
    one2, zero2 = one[:2 * F0].contiguous(), zero[:2 * F0].contiguous()
    y, mu, rs = ln(ops.LN_CONCAT, fine, skip, Bh * G * G, 2 * F0, one2, zero2)
    nb = 2 * fine.numel() * 2 * 2
    s = timed(lambda: ln(ops.LN_CONCAT, fine, skip, Bh * G * G, 2 * F0, one2, zero2), 20)
    out["rows_concat"] = {"fwd_us": round(s * 1e6, 1), "fwd_hbm_floor_share": round(nb / HBM / s, 3)}
    s = timed(lambda: ops.layernorm_rows_bwd(ops.LN_CONCAT, fine, skip, y, Bh * G * G, 2 * F0, one2, mu, rs,
                                             dg[:2 * F0], db[:2 * F0]), 20)
    out["rows_concat"].update(bwd_us=round(s * 1e6, 1), bwd_hbm_floor_share=round(1.5 * nb / HBM / s, 3))
    return out


def blocks(B, L):
    """One MMDiT block and one DiTBlock, forward + backward, at the same shapes (ms)."""
    out = {}
    for model in (SimpleMMDiT(patch_size=P, emb_features=F, num_layers=1, num_heads=12, context_dim=768),
                  SimpleDiT(patch_size=P, emb_features=F, num_layers=1, num_heads=12)):
        fp = model.init(0, device=dev)
        W32, W16, G = fp.named, fp.shadow(), fp.zeros_like()
        x = torch.randn(B * L, F, device=dev).bfloat16()
        cw = model._cond_width()
        cond16 = torch.randn(B, cw, device=dev).bfloat16()
        dcond = torch.zeros(B, cw, device=dev)
        dx2 = torch.randn_like(x)
        (n, fwd, bwd), = model._blocks()

        def run():
            _, rec = fwd(n, x, cond16, W32, W16, B, L)
            bwd(rec, dx2, cond16, dcond, W32, W16, G.named, B, L)
        out[type(model).__name__ + "_block_fwd_bwd_ms"] = round(timed(run, 5) * 1e3, 2)
        fp = G = None
        gc.collect()
        torch.cuda.empty_cache()
    return out


def throughput(model, r, B, iters, sample):
    row = {}
    enc = RandomEmbeddingEncoder(77, 768, device=dev)
    cfg = DiffusionInputConfig("image", (r, r, 3), [ConditionalInputConfig(enc)])
    ctx = torch.randn(B, 77, 768, device=dev).bfloat16()
    if sample:
        return euler(model, r, B, cfg, ctx)
    try:
        tr = GeneralDiffusionTrainer(model, adamw(1e-4), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                     cfg, rngs=4, model_output_transform=KarrasPredictionTransform(0.5), device=dev)
        step = tr._define_train_step()
        batch = {"image": torch.randint(0, 256, (B, r, r, 3), dtype=torch.uint8, device=dev), "text": ctx}
        st = [tr.state, tr.rngstate]

        def train():
            st[0], _, st[1] = step(st[0], st[1], batch)
        s = timed(train, iters)
        row["train_step_ms"] = round(s * 1e3, 2)
        row["train_img_per_s"] = round(B / s, 1)
        row["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    except torch.cuda.OutOfMemoryError as e:
        row["train_error"] = f"out of memory: {str(e)[:120]}"
    return row


def euler(model, r, B, cfg, ctx):
    row = {}
    try:
        fp = model.init(0, textcontext=ctx, device=dev)
        smp = EulerSampler(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5).to(dev),
                           KarrasPredictionTransform(0.5), cfg)
        gen = lambda n: smp.generate_samples(fp, B, r, diffusion_steps=n, start_step=1000, device=dev,  # noqa: E731
                                             model_conditioning_inputs=(ctx,))
        s12 = timed(lambda: gen(12), 2, warm=1)
        s2 = timed(lambda: gen(2), 2, warm=1)
        row["euler_step_ms"] = round((s12 - s2) / 10 * 1e3, 2)
        row["euler_img_steps_per_s"] = round(B / ((s12 - s2) / 10), 1)
    except torch.cuda.OutOfMemoryError as e:
        row["euler_error"] = f"out of memory: {str(e)[:120]}"
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", choices=("kernels", "mmdit", "dit", "hier", "mmdit-euler", "dit-euler", "hier-euler"),
                    required=True)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    L = (RES // P) ** 2
    res = {"card": card(), "shape": f"B/2 {RES}x{RES}, B = {BATCH}"}
    if args.which == "kernels":
        res["kernels"] = kernels(BATCH, L, F)
        res["blocks"] = blocks(BATCH, L)
    elif args.which.startswith("hier"):
        torch.cuda.reset_peak_memory_stats()
        res["shape"] = f"class defaults {HIER_RES}x{HIER_RES}, B = {HIER_BATCH}"
        res["HierarchicalMMDiT"] = throughput(HierarchicalMMDiT(context_dim=768), HIER_RES, HIER_BATCH, args.iters,
                                              args.which.endswith("euler"))
    else:
        torch.cuda.reset_peak_memory_stats()
        cls = SimpleMMDiT if args.which.startswith("mmdit") else SimpleDiT
        model = cls(context_dim=768, **BASE)
        sample = args.which.endswith("euler")
        if sample:
            res["shape"] = f"B/2 {RES}x{RES}, B = {EULER_BATCH}"
        res[cls.__name__] = throughput(model, RES, EULER_BATCH if sample else BATCH, args.iters, sample)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
