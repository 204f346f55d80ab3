"""Compile-time guard for the CLIP metric kernels (no GPU needed): fdx_clip.cu's image preparation, vision embedding,
pooling and similarity kernels have no stack frame and no spills under `-Xptxas -v`."""
import os
import re

import pytest

from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def test_clip_metric_kernels_have_no_frame_and_no_spills():
    frames, _ = _report("fdx_clip.cu")
    names = {k: v for k, v in frames.items()
             if re.search(r"clip_(image_prep|vision_embed|pool|similarity)_kernel", k)}
    assert len(names) == 4, sorted(frames)
    assert all(v == (0, 0, 0) for v in names.values()), names
