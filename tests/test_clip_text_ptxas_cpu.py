"""Compile-time guard for the CLIP text tower's kernels (no GPU needed): fdx_clip.cu's streaming kernels have no stack
frame and no spills, and every masked attention forward (fdx_attn_fwd_kernel<DH, SHORT, true>) is no worse under
`-Xptxas -v` than its unmasked twin (<DH, SHORT, false>): no spills, no larger stack frame, and no ptxas performance
note (C7507 / C7514 / C7517 - C7520) the twin does not have."""
import os
import re
import subprocess
import tempfile

import pytest

from test_ptxas_cpu import CSRC, NVCC

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _report(src):
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler",
               "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", os.path.join(tmp, "a.o")]
        p = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, f"{src} failed to compile:\n{p.stdout[-4000:]}"
    frames, notes, current = {}, {}, None
    for line in p.stdout.splitlines():
        note = re.search(r"\((C75(?:07|14|17|18|19|20))\).*'(\w+)'", line)
        if note:
            notes.setdefault(note.group(2), set()).add(note.group(1))
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            frames[current] = tuple(int(g) for g in m.groups())
            current = None
    return frames, notes


def test_clip_kernels_have_no_frame_and_no_spills():
    frames, _ = _report("fdx_clip.cu")
    names = {k: v for k, v in frames.items() if re.search(r"(token_embed|layernorm_fwd|bias_act)_kernel", k)}
    assert len(names) == 4, sorted(frames)               # embedding, LayerNorm, two activations
    assert all(v == (0, 0, 0) for v in names.values()), names


def test_masked_attention_is_no_worse_than_its_unmasked_twin():
    frames, notes = _report("fdx_attn.cu")
    pairs = 0
    for name, (frame, stores, loads) in frames.items():
        m = re.search(r"fdx_attn_fwd_kernelILi(\d+)ELb([01])ELb1E", name)
        if not m:
            continue
        twin = name.replace(m.group(0), m.group(0)[:-len("ELb1E")] + "ELb0E")
        assert twin in frames, twin
        tf, ts, tl = frames[twin]
        assert stores == loads == 0 and ts == tl == 0, (name, frames[name], frames[twin])
        assert frame <= tf, (name, frame, tf)
        assert notes.get(name, set()) <= notes.get(twin, set()), (name, notes.get(name), notes.get(twin))
        pairs += 1
    assert pairs == 4                                    # dh 32 / 64, single-stage / ring
