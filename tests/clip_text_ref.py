"""Float64 references of the CLIP text tower's kernels (csrc/fdx_clip.cu and the masked forward of csrc/fdx_attn.cu),
with the first-order error bound `delta` of each kernel's f32 arithmetic, in the tolerance model of
tests/elementwise_ref.py (compare bf16 outputs with its bf16_bound).  Also the seeded CLIPTextConfigs, token batches
and a stand-in tokenizer the tower tests share.  Error constants of the CUDA math functions used here (CUDA C
Programming Guide, Mathematical Functions): expf 2 ulp, erff 2 ulp, correctly rounded division."""
from __future__ import annotations

import math

import torch

from elementwise_ref import EX2, FTZ, RSQRT, TC_ADD, U32, U_BF16, gamma

EXPF = 4 * U32               # expf: 2 ulp, i.e. 4u relative
ERFF = 4 * U32               # erff: 2 ulp of a result in [-1, 1]


# ----------------------------------------------------------------------------------------------- embedding
def token_embed_ref(ids, tok, pos):
    """bf16(tok[ids] + pos[t]) with NaN rows for ids outside [0, vocab): -> (value, delta); one f32 addition."""
    B, T = ids.shape
    vocab, D = tok.shape
    ok = (ids >= 0) & (ids < vocab)
    val = tok[ids.clamp(0, vocab - 1)] + pos[:T].unsqueeze(0)
    val = torch.where(ok.unsqueeze(-1), val, torch.full_like(val, math.nan))
    return val, U32 * val.abs()


# ----------------------------------------------------------------------------------------------- LayerNorm
def layernorm_ref(x, g, b, eps):
    """y = (x - mean) rstd g + b -> (value, delta).  layernorm_fwd_kernel: per lane ceil(C/256) vectors of 8 serial
    additions, then a 5-level warp tree (D1 = 8 ceil(C/256) + 5) for the sum and for the centred squares; mean =
    s / C (1 rounding), d = x - mean (1 rounding), the variance sum relative gamma(D1 + 2) (the mean's error enters
    it only at second order: sum(x - mean) = 0), / C and + eps (2 roundings), rsqrtf; then d rstd (1 rounding) and
    the fma with g, b (1 rounding)."""
    C = x.shape[-1]
    D1 = 8 * math.ceil(C / 256) + 5
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = d * rstd * g + b
    e_mean = gamma(D1 + 1) * x.abs().mean(-1, keepdim=True)
    rho = gamma(D1 + 4) / 2 + RSQRT
    delta = g.abs() * rstd * (d.abs() * (rho + 2 * U32) + e_mean) + U32 * (y.abs() + b.abs())
    return y, delta


# ----------------------------------------------------------------------------------------------- bias + act
def bias_act_ref(x, bias, act: int):
    """act(x + bias): 0 = quick_gelu z / (1 + expf(-1.702 z)), 1 = gelu 0.5 z (1 + erff(z / sqrt 2)) -> (value,
    delta).  z = x + bias rounds once (|act'| <= 1.13 carries it); quick_gelu: fl(1.702) and the product put 2u on
    the exponent, expf 4u, 1 + e and the division 1u each; gelu: the argument's rounding, erff's 2 ulp absolute,
    1 + erf, the two products."""
    z = x if bias is None else x + bias
    if act == 0:
        k = 1.702
        e = torch.exp(-k * z)
        y = z / (1 + e)
        w = e / (1 + e)                                   # d log(1 + e) / d log e
        delta = y.abs() * (w * (2 * U32 * (k * z).abs() + EXPF) + 2 * U32)
    else:
        a = z / math.sqrt(2.0)
        erf = torch.erf(a)
        y = 0.5 * z * (1 + erf)
        derf = ERFF * erf.abs().clamp_min(2.0 ** -24) + U32 * a.abs() * 2 / math.sqrt(math.pi) * torch.exp(-a * a)
        delta = 0.5 * z.abs() * (derf + U32 * (1 + erf)) + 2 * U32 * y.abs()
    return y, delta + 1.13 * U32 * z.abs()


# ----------------------------------------------------------------------------------------------- attention
def attention_masked_ref(q, k, v, heads: int, dh: int, scale: float, causal: bool, key_mask=None):
    """fdx_attention_fwd_masked in float64: o = softmax over the allowed keys (j <= i when causal, key_mask[b][j])
    of q k^T scale, times v; zeros for a row with no allowed key.  -> (o, delta) of shape (B, L, heads dh).  The
    bound is elementwise_ref's forward derivation (_attn_rows) restricted to the allowed keys; the depth of every
    sum over keys stays that of the zero-filled key blocks."""
    B, L, HD = q.shape
    Lk = k.shape[1]
    sc = float(torch.tensor(scale, dtype=torch.float32))
    nblk = math.ceil(Lk / 128)
    Lkp = 128 * nblk
    o = torch.zeros(B, L, HD, dtype=torch.float64, device=q.device)
    d_o = torch.zeros_like(o)
    i = torch.arange(L, device=q.device).view(L, 1)
    j = torch.arange(Lk, device=q.device).view(1, Lk)
    for bi in range(B):
        allowed = torch.ones(L, Lk, dtype=torch.bool, device=q.device)
        if causal:
            allowed &= j <= i
        if key_mask is not None:
            allowed &= (key_mask[bi] != 0).view(1, Lk)
        af = allowed.to(torch.float64)
        any_row = allowed.any(1, keepdim=True)
        for h in range(heads):
            cs = slice(h * dh, (h + 1) * dh)
            qh, kh, vh = q[bi, :, cs], k[bi, :, cs], v[bi, :, cs]
            ka, va = kh.abs(), vh.abs()
            t = sc * (qh @ kh.T)
            tmax = t.masked_fill(~allowed, -math.inf).amax(1, keepdim=True)
            tmax = torch.where(any_row, tmax, torch.zeros_like(tmax))
            e = torch.exp(t - tmax) * af
            lsum = e.sum(1, keepdim=True)
            P = e / lsum.clamp_min(1e-300)
            O = P @ vh
            es = sc * dh * TC_ADD * (qh.abs() @ ka.T)
            eta = (es + 2 * U32 * t.abs() + 2 * U32 * (tmax - t).abs() + nblk * EX2) * af
            Pe = P * eta
            eps_l = gamma(Lkp + nblk + 2)
            spa = P @ va
            err = (Pe @ va + O.abs() * Pe.sum(1, keepdim=True)
                   + (U_BF16 + TC_ADD * Lkp + gamma(nblk) + eps_l + 2 * U32) * spa
                   + FTZ * Lk * va.amax(0))
            o[bi, :, cs] = O
            d_o[bi, :, cs] = torch.where(any_row, err, torch.zeros_like(err))
    return o, d_o


# ----------------------------------------------------------------------------------------------- tower fixtures
def clip_config(kind: str):
    """Seeded CLIPTextConfigs: the tiny one of test_text_encoder_cpu.py with 2 heads of 32 (its 4 heads of 16 are
    narrower than the attention kernels), CLIP ViT-L/14's text tower, and an OpenCLIP-like gelu tower (1024 wide,
    16 heads, a few layers)."""
    from transformers import CLIPTextConfig
    if kind == "tiny":
        return CLIPTextConfig(vocab_size=1000, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                              num_attention_heads=2, max_position_embeddings=77)
    if kind == "clip-l":
        return CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                              num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu")
    if kind == "openclip":
        return CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=3,
                              num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu")
    raise ValueError(kind)


def clip_model(kind: str, seed: int = 0):
    """transformers' CLIPTextModel with random weights (CPU, fp32, eager attention)."""
    from transformers import CLIPTextModel
    torch.manual_seed(seed)
    cfg = clip_config(kind)
    cfg._attn_implementation = "eager"
    return CLIPTextModel(cfg).eval()


def token_batch(vocab: int, lengths, T: int = 77, seed: int = 0):
    """CLIP-tokenizer-shaped batch: BOS, `n` word ids, EOS, then padding (id 0, mask 0); `n` = 75 gives the full
    77-token sequence, 0 the empty prompt.  -> (input_ids, attention_mask) int64 [len(lengths), T]."""
    g = torch.Generator().manual_seed(seed)
    bos, eos = vocab - 2, vocab - 1
    ids = torch.zeros(len(lengths), T, dtype=torch.long)
    mask = torch.zeros(len(lengths), T, dtype=torch.long)
    for r, n in enumerate(lengths):
        n = min(n, T - 2)
        ids[r, 0] = bos
        ids[r, 1:1 + n] = torch.randint(1, vocab - 2, (n,), generator=g)
        ids[r, 1 + n] = eos
        mask[r, :n + 2] = 1
    return ids, mask


class Tok:
    """Stand-in for AutoTokenizer (padding="max_length", 77 tokens): words hash to ids, BOS / EOS around them."""
    model_max_length = 77

    def __init__(self, vocab: int):
        self.vocab = vocab

    def __call__(self, data, padding=None, max_length=None, truncation=None, return_tensors=None):
        import zlib
        assert padding == "max_length" and max_length == 77 and truncation is True and return_tensors == "pt"
        words = [[1 + zlib.crc32(w.encode()) % (self.vocab - 3) for w in str(s).split()][:75] for s in data]
        ids, mask = token_batch(self.vocab, [len(w) for w in words])
        for r, w in enumerate(words):
            ids[r, 1:1 + len(w)] = torch.tensor(w, dtype=torch.long)
        return {"input_ids": ids, "attention_mask": mask}


def rel_l2_per_sequence(got, ref):
    """||got_s - ref_s|| / ||ref_s|| over all T positions of each sequence s, float64."""
    g, r = got.detach().to("cpu", torch.float64), ref.detach().to("cpu", torch.float64)
    return ((g - r).flatten(1).norm(dim=1) / r.flatten(1).norm(dim=1)).tolist()
