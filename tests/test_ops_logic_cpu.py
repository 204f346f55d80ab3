"""Host-side dispatch rules of flaxdiff_b200.ops that decide which kernel arrangement runs (no GPU needed)."""
import torch

import elementwise_ref as R
from flaxdiff_b200 import ops


def _t(*shape):
    return torch.empty(shape, dtype=torch.bfloat16, device="meta")


def test_groupnorm_backward_fusion_follows_the_transposed_engine():
    """The first pass of the GroupNorm backward is fused into the data gradient's epilogue exactly where that
    convolution runs on the transposed engine (DESIGN 3.2): Cin a multiple of 64 but not of 256, <= 512,
    16-aligned images of >= 128 pixels, Cout a multiple of 64."""
    ok = [(64, 64, 64, 64), (32, 32, 128, 128), (64, 64, 320, 64), (16, 16, 192, 256), (16, 16, 384, 256)]
    for h, w, cin, cout in ok:
        assert ops._gn_fuse_default(_t(2, h, w, cin), _t(2, h, w, cout)), (h, w, cin, cout)
    no = [(16, 16, 256, 256),      # Cin multiple of 256: pixels-as-M engine
          (16, 16, 512, 512),
          (8, 8, 128, 128),        # < 128 pixels per image (and not 16-aligned)
          (16, 8, 192, 128),       # width not a multiple of 16
          (32, 32, 576, 128),      # Cin > 512
          (32, 32, 128, 96)]       # Cout not a multiple of 64
    for h, w, cin, cout in no:
        assert not ops._gn_fuse_default(_t(2, h, w, cin), _t(2, h, w, cout)), (h, w, cin, cout)


def test_colstats_constants():
    assert ops.COLSTATS_SLOTS >= 1 and ops.COLSTATS_MIN_PIXELS == 128 and ops.GN_FUSE_MIN_PIXELS == 128


def test_fused_column_sums_take_a_one_image_pixel_box():
    """fdx_tc_launch's pixel box (restated in elementwise_ref.tc_pixel_box) on every output of an input of
    W, H <= 64 at strides 1 and 2.  The packed box of the other launches holds several small images per tile, which
    per-image column sums cannot use; with sums the box is one image deep, so every image of >= 128 pixels is
    served.  Where the packed box already holds one image the two boxes agree, so no launch that ran before
    changes geometry; and every TMA box dimension (the box times the stride) stays within 256."""
    refused = set()
    for s in (1, 2):
        for H in range(1, 65):
            for W in range(1, 65):
                Ho, Wo = -(-H // s), -(-W // s)
                old = R.tc_pixel_box(Wo, Ho)
                new = R.tc_pixel_box(Wo, Ho, colstats=True)
                assert new[2] == 1 and new[0] * new[1] == 128, (W, H, s, new)
                assert new[0] * s <= 256 and new[1] * s <= 256, (W, H, s, new)
                if old[2] == 1:
                    assert new == old, (W, H, s, old, new)
                elif Ho * Wo >= ops.COLSTATS_MIN_PIXELS:
                    refused.add((Wo, Ho))
    # the images of >= 128 pixels the packed box could not serve: every square of 12 to 15 pixels a side
    assert {w for w, h in refused if w == h} == {12, 13, 14, 15}
    assert (6, 24) in refused and (26, 5) in refused
