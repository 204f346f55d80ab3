"""Compile-time guard for the head-width-128 attention kernels (no GPU needed): compiles fdx_attn.cu for sm_90a with
`-Xptxas -v` and fails when ptxas serialised the wgmma of fdx_attn_fwd128_kernel / fdx_attn_bwd128_kernel, had to
inject warpgroup synchronisation into them, or ignored their setmaxnreg (C7507 / C7514 / C7517 - C7520), or when
one of them has a stack frame or spills.  Only these kernels are checked: the 32 / 64-wide attention kernels in
the same file still carry such notes (DESIGN section 8)."""
import os
import re
import subprocess
import tempfile

import pytest

from test_ptxas_cpu import CSRC, NVCC

KERNELS = ("fdx_attn_fwd128_kernel", "fdx_attn_bwd128_kernel")

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _short(name):
    m = re.search(r"fdx_attn_(?:fwd|bwd)128_kernelILb[01]E", name)
    return m.group(0) if m else name


def test_wide_attention_kernels_keep_their_accumulators_in_registers():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler",
               "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "fdx_attn.cu"), "-o", os.path.join(tmp, "a.o")]
        p = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, f"fdx_attn.cu failed to compile:\n{p.stdout[-4000:]}"
    problems, seen, current = [], set(), None
    for line in p.stdout.splitlines():
        note = re.search(r"\((C75(?:07|14|17|18|19|20))\).*'(\w+)'", line)
        if note and any(k in note.group(2) for k in KERNELS):
            problems.append(f"{_short(note.group(2))}: ptxas {note.group(1)}")
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if current:
                seen.add(_short(current))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            if any(int(g) for g in m.groups()):
                problems.append(f"{_short(current)}: {m.group(0)}")
            current = None
    # forward: single-stage and ring; backward: dQ and dK / dV
    assert len(seen) == 4, sorted(seen)
    assert not problems, "\n".join(problems)
