"""Kernel launches of one UNet forward plus backward for every attention-block configuration.  Every attention block,
pure or full, runs one program (Unet._tblock_fwd / _tblock_bwd around _mha_fwd / _mha_bwd); the counts below pin
how many libfdx kernels each configuration issues, so a change that adds or drops one shows here.
tests/gpu_probe_op_trace.py prints the calls behind each count."""

import pytest
import torch

from flaxdiff_b200 import _lib
from flaxdiff_b200.models.simple_unet import Unet

pytestmark = pytest.mark.gpu

# (id, attention config without "heads", 77 x 768 text context?)
BLOCKS = [
    ("pure_self", {}, False),
    ("pure_text", {}, True),
    ("pure_proj_self", {"use_projection": True}, False),
    ("pure_proj_text", {"use_projection": True}, True),
] + [
    (f"full{'_both' if both else ''}{'_proj' if proj else ''}_{'text' if text else 'self'}",
     {"only_pure_attention": False, "use_self_and_cross": both, "use_projection": proj}, text)
    for both in (True, False) for proj in (True, False) for text in (False, True)
]
# true head width -> (channels of the attention levels, heads); 16 is stored 32 wide and 80 is stored 128 wide
WIDTHS = {16: (128, 8), 64: (512, 8), 80: (640, 8), 128: (256, 2)}

# launches per forward + backward of `unet_fwd_bwd`: a UNet with feature_depths (C, C) at 16 x 16, B = 2, whose
# three attention blocks (down_1_attention_1, middle_attention_0, up_0_attention_1) run at 8 x 8.  The full blocks'
# counts grow with C: the feed-forward bias gradient sums its 8 C columns in slabs of 2048 (ops.colsum_rows)
LAUNCHES = {
    "pure_self": {16: 315, 64: 315, 80: 315, 128: 315},
    "pure_text": {16: 309, 64: 309, 80: 309, 128: 309},
    "pure_proj_self": {16: 336, 64: 336, 80: 336, 128: 336},
    "pure_proj_text": {16: 327, 64: 327, 80: 327, 128: 327},
    "full_both_proj_self": {16: 435, 64: 438, 80: 441, 128: 435},
    "full_both_proj_text": {16: 426, 64: 429, 80: 432, 128: 426},
    "full_both_self": {16: 423, 64: 426, 80: 429, 128: 423},
    "full_both_text": {16: 414, 64: 417, 80: 420, 128: 414},
    "full_proj_self": {16: 378, 64: 381, 80: 384, 128: 378},
    "full_proj_text": {16: 369, 64: 372, 80: 375, 128: 369},
    "full_self": {16: 366, 64: 369, 80: 372, 128: 366},
    "full_text": {16: 357, 64: 360, 80: 363, 128: 357},
}


def unet_fwd_bwd(block: str, d: int, dev, unet=Unet):
    """One forward plus backward of the UNet above with attention block `block` at head width `d`."""
    _, extra, text = next(b for b in BLOCKS if b[0] == block)
    C, heads = WIDTHS[d]
    cfg = dict(extra, heads=heads)
    model = unet(feature_depths=(C, C), attention_configs=(None, cfg), dtype=torch.bfloat16,
                 context_dim=768 if text else None)
    fp = model.init(4, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    B, res = 2, 16
    x = torch.randn(B, res, res, 3, generator=g, device=dev).bfloat16()
    t = torch.randn(B, generator=g, device=dev)
    ctx = torch.randn(B, 77, 768, generator=g, device=dev).bfloat16() if text else None
    F, saved = model.forward(fp, x, t, ctx, save=True)
    grads = fp.zeros_like()
    model.backward(fp, saved, torch.randn(F.shape, generator=g, device=dev), grads)
    return F, grads


def launch_count() -> int:
    lib = _lib.load()
    return lib.fdx_launch_count()


@pytest.mark.parametrize("d", sorted(WIDTHS))
@pytest.mark.parametrize("block", [b[0] for b in BLOCKS])
def test_attention_block_launch_count(block, d):
    dev = torch.device("cuda")
    before = launch_count()
    F, grads = unet_fwd_bwd(block, d, dev)
    torch.cuda.synchronize()
    assert launch_count() - before == LAUNCHES[block][d]
    assert torch.isfinite(F).all() and torch.isfinite(grads.flat).all()
