"""Compile-time guard for fdx_dit.cu (no GPU needed).  SimpleDiT adds no tensor-core instantiation (its dense layers and
attention reuse fdx_gemm and the fused attention kernels), so what is held here is the streaming kernels: none spills,
and none but RoPE and the Fourier features - whose sincosf / sinf keep the slow-path argument reduction's 32-byte local
array - has a stack frame."""
import os
import re

import pytest

from test_clip_text_ptxas_cpu import _report
from test_ptxas_cpu import NVCC

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def test_dit_kernels_have_no_spills_and_no_frames():
    frames, notes = _report("fdx_dit.cu")
    dit = {k: v for k, v in frames.items() if "dit_" in k}
    assert len(dit) == 14, sorted(dit)
    for name, (frame, stores, loads) in dit.items():
        assert stores == loads == 0, (name, frame, stores, loads)
        if not re.search(r"dit_(rope|fourier)_kernel", name):
            assert frame == 0, (name, frame)
    assert not any("dit_" in k for k in notes), notes
