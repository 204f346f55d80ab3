"""GPU probe for the wgmma tap-GEMM engine (run directly on a GPU machine; not a pytest file).

Runs every mode (conv fwd / dgrad / wgrad, stride 1 and 2, GEMM KK / KMN / MNMN, batched)
against a torch fp32 reference on the same bf16-rounded inputs and prints one line per
case, never stopping at the first failure, so one GPU call gives the full picture.
Each case runs in a subprocess-free but exception-guarded block with a device sync.
"""
import sys
import time
import traceback

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from flaxdiff_b200 import ops  # noqa: E402
from flaxdiff_b200._lib import GEMM_KK, GEMM_KMN, GEMM_MNMN  # noqa: E402

dev = torch.device("cuda")
torch.manual_seed(0)
results = []


def rel_err(a, b):
    a = a.float()
    b = b.float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item(), (a - b).abs().max().item()


def ref_conv(x, w, stride):
    # x NHWC, w HWIO ; jax SAME padding: stride 1 -> (1,1); stride 2 even -> (0,1)
    xn = x.float().permute(0, 3, 1, 2)
    wn = w.float().permute(3, 2, 0, 1)
    if stride == 1:
        xn = F.pad(xn, (1, 1, 1, 1))
    else:
        xn = F.pad(xn, (0, 1, 0, 1))
    return F.conv2d(xn, wn, stride=stride).permute(0, 2, 3, 1)


FILTER = sys.argv[1:] 


def case(name, fn):
    if FILTER and not any(name.startswith(f) for f in FILTER):
        return
    t0 = time.time()
    try:
        r, m = fn()
        torch.cuda.synchronize()
        ok = r < 2e-2
        results.append((name, ok, r, m))
        print(f"[{'OK ' if ok else 'BAD'}] {name}: rel={r:.3e} maxabs={m:.3e} ({time.time()-t0:.2f}s)", flush=True)
    except Exception as e:  # noqa: BLE001
        results.append((name, False, float('nan'), float('nan')))
        print(f"[EXC] {name}: {e}", flush=True)
        traceback.print_exc()


def t_conv_fwd(n, h, w, cin, cout, stride=1, extras=False):
    def f():
        x = torch.randn(n, h, w, cin, device=dev).bfloat16()
        wt = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
        bias = torch.randn(cout, device=dev) if extras else None
        rowvec = torch.randn(n, cout, device=dev) if extras else None
        ho, wo = h // stride, w // stride
        res = torch.randn(n, ho, wo, cout, device=dev).bfloat16() if extras else None
        y = ops.conv3x3_fwd(x, wt, bias, rowvec, res, stride=stride)
        ref = ref_conv(x, wt, stride)
        if extras:
            ref = ref + bias + rowvec[:, None, None, :] + res.float()
        return rel_err(y, ref)
    return f


def t_conv_fwd_slot(n, h, w, cin, cout):
    """input is a channel slice of a wider concat buffer; output goes into a slot."""
    def f():
        big = torch.randn(n, h, w, cin + 64, device=dev).bfloat16()
        x = big[..., 64:]
        wt = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
        outbig = torch.zeros(n, h, w, cout + 128, device=dev, dtype=torch.bfloat16)
        y = outbig[..., 128:]
        ops.conv3x3_fwd(x, wt, out=y)
        ref = ref_conv(x, wt, 1)
        r = rel_err(y, ref)
        assert outbig[..., :128].abs().max().item() == 0
        return r
    return f


def t_conv_dgrad(n, h, w, cin, cout, stride=1, accumulate=False):
    def f():
        x = torch.randn(n, h, w, cin, device=dev).bfloat16().float().requires_grad_(True)
        wt = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).bfloat16()
        y = ref_conv(x, wt, stride)
        dy = torch.randn_like(y).bfloat16()
        y.backward(dy.float())
        dx = torch.zeros(n, h, w, cin, device=dev, dtype=torch.bfloat16)
        base = None
        if accumulate:
            base = torch.randn(n, h, w, cin, device=dev).bfloat16()
            dx.copy_(base)
        ops.conv3x3_dgrad(dy.contiguous(), wt, dx, stride=stride, accumulate=accumulate)
        ref = x.grad + (base.float() if accumulate else 0)
        return rel_err(dx, ref)
    return f


def t_conv_wgrad(n, h, w, cin, cout, stride=1):
    def f():
        x = torch.randn(n, h, w, cin, device=dev).bfloat16()
        wt = (torch.randn(3, 3, cin, cout, device=dev) / (3 * cin ** 0.5)).float().requires_grad_(True)
        y = ref_conv(x, wt, stride)
        dy = torch.randn_like(y).bfloat16()
        y.backward(dy.float())
        dw = torch.zeros(3, 3, cin, cout, device=dev, dtype=torch.float32)
        ops.conv3x3_wgrad(x, dy.contiguous(), dw, stride=stride)
        return rel_err(dw, wt.grad)
    return f


def t_gemm_kk(M, N, K):
    def f():
        A = torch.randn(M, K, device=dev).bfloat16()
        B = torch.randn(N, K, device=dev).bfloat16()
        D = torch.empty(M, N, device=dev, dtype=torch.float32)
        ops.gemm(GEMM_KK, A, B, D, M, N, K, K, K, N, alpha=0.5)
        return rel_err(D, 0.5 * A.float() @ B.float().t())
    return f


def t_gemm_kmn(M, N, K, with_bias=True):
    def f():
        A = torch.randn(M, K, device=dev).bfloat16()
        B = torch.randn(K, N, device=dev).bfloat16()
        bias = torch.randn(N, device=dev) if with_bias else None
        D = ops.linear_fwd(A, B, bias=bias)
        ref = A.float() @ B.float()
        if with_bias:
            ref = ref + bias
        return rel_err(D, ref)
    return f


def t_gemm_mnmn(M, N, K):
    def f():
        A = torch.randn(K, M, device=dev).bfloat16()
        B = torch.randn(K, N, device=dev).bfloat16()
        D = torch.zeros(M, N, device=dev, dtype=torch.float32)
        ops.gemm(GEMM_MNMN, A, B, D, M, N, K, M, N, N, atomic=True, reduce_batch=True)
        return rel_err(D, A.float().t() @ B.float())
    return f


def t_attn_qk(Bb, L, h, d):
    """S[b,h,l,lk] = Q[b,l,h,:] . K[b,lk,h,:] (batched KK)"""
    def f():
        Q = torch.randn(Bb, L, h, d, device=dev).bfloat16()
        Kt = torch.randn(Bb, L, h, d, device=dev).bfloat16()
        S = torch.empty(Bb, h, L, L, device=dev, dtype=torch.bfloat16)
        ops.gemm(GEMM_KK, Q, Kt, S, L, L, d, h * d, h * d, L, batch1=h, batch2=Bb,
                 a_s=(d, L * h * d), b_s=(d, L * h * d), d_s=(L * L, h * L * L), alpha=d ** -0.5)
        ref = torch.einsum("blhd,bkhd->bhlk", Q.float(), Kt.float()) * d ** -0.5
        return rel_err(S, ref)
    return f


def t_attn_pv(Bb, L, h, d):
    """O[b,l,h,:] = sum_lk P[b,h,l,lk] V[b,lk,h,:]  (batched KMN)"""
    def f():
        P = torch.softmax(torch.randn(Bb, h, L, L, device=dev), -1).bfloat16()
        V = torch.randn(Bb, L, h, d, device=dev).bfloat16()
        O = torch.empty(Bb, L, h, d, device=dev, dtype=torch.bfloat16)
        ops.gemm(GEMM_KMN, P, V, O, L, d, L, L, h * d, h * d, batch1=h, batch2=Bb,
                 a_s=(L * L, h * L * L), b_s=(d, L * h * d), d_s=(d, L * h * d))
        ref = torch.einsum("bhlk,bkhd->blhd", P.float(), V.float())
        return rel_err(O, ref)
    return f


def t_attn_dv(Bb, L, h, d):
    """dV[b,lk,h,:] = sum_l P[b,h,l,lk] dO[b,l,h,:]  (batched MNMN, no batch reduce)"""
    def f():
        P = torch.softmax(torch.randn(Bb, h, L, L, device=dev), -1).bfloat16()
        dO = torch.randn(Bb, L, h, d, device=dev).bfloat16()
        dV = torch.empty(Bb, L, h, d, device=dev, dtype=torch.bfloat16)
        ops.gemm(GEMM_MNMN, P, dO, dV, L, d, L, L, h * d, h * d, batch1=h, batch2=Bb,
                 a_s=(L * L, h * L * L), b_s=(d, L * h * d), d_s=(d, L * h * d))
        ref = torch.einsum("bhlk,blhd->bkhd", P.float(), dO.float())
        return rel_err(dV, ref)
    return f


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0), flush=True)
    case("gemm_kk 256x128x128", t_gemm_kk(256, 128, 128))
    case("gemm_kk 1000x256x320", t_gemm_kk(1000, 256, 320))
    case("gemm_kmn 256x64x64", t_gemm_kmn(256, 64, 64, False))
    case("gemm_kmn 512x512x256+bias", t_gemm_kmn(512, 512, 256))
    case("gemm_mnmn 128x64x256", t_gemm_mnmn(128, 64, 256))
    case("gemm_mnmn 256x512x4096", t_gemm_mnmn(256, 512, 4096))
    case("conv_fwd 2x16x16 64->64", t_conv_fwd(2, 16, 16, 64, 64))
    case("conv_fwd 2x32x32 128->256 +bias/temb/res", t_conv_fwd(2, 32, 32, 128, 256, extras=True))
    case("conv_fwd 4x8x8 256->512 (multi-image tile)", t_conv_fwd(4, 8, 8, 256, 512))
    case("conv_fwd 1x64x64 320->64", t_conv_fwd(1, 64, 64, 320, 64))
    case("conv_fwd slot views", t_conv_fwd_slot(2, 16, 16, 128, 64))
    case("conv_fwd s2 2x32x32 64->128", t_conv_fwd(2, 32, 32, 64, 128, stride=2))
    case("conv_dgrad 2x16x16 64->128", t_conv_dgrad(2, 16, 16, 64, 128))
    case("conv_dgrad acc 2x32x32 192->64", t_conv_dgrad(2, 32, 32, 192, 64, accumulate=True))
    case("conv_dgrad s2 2x32x32 64->128", t_conv_dgrad(2, 32, 32, 64, 128, stride=2))
    case("conv_wgrad 2x16x16 64->64", t_conv_wgrad(2, 16, 16, 64, 64))
    case("conv_wgrad 4x32x32 192->128", t_conv_wgrad(4, 32, 32, 192, 128))
    case("conv_wgrad s2 2x32x32 64->128", t_conv_wgrad(2, 32, 32, 64, 128, stride=2))
    case("attn_qk B2 L256 h8 d64", t_attn_qk(2, 256, 8, 64))
    case("attn_pv B2 L256 h8 d64", t_attn_pv(2, 256, 8, 64))
    case("attn_dv B2 L256 h8 d64", t_attn_dv(2, 256, 8, 64))
    nbad = sum(1 for r in results if not r[1])
    print(f"SUMMARY: {len(results) - nbad}/{len(results)} ok", flush=True)
