"""Compile-time guard for the warp-specialised wgmma kernels (no GPU needed): compiles fdx_tc.cu, fdx_tct.cu and
fdx_wgrad9.cu for sm_90a with `-Xptxas -v` and fails when ptxas reports that it serialised a kernel's wgmma or
ignored its setmaxnreg (C7507 / C7514 / C7518 / C7520), or when a kernel has a stack frame or spills.  Either one
means the accumulator goes through local memory, which has cost these kernels up to half their time."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "flaxdiff_b200", "csrc")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
SOURCES = ["fdx_tc.cu", "fdx_tct.cu", "fdx_wgrad9.cu"]
KERNELS = ("fdx_tc_kernel", "fdx_tct_kernel", "fdx_wgrad9_kernel")
# the halo variant of the transposed engine with the fused GroupNorm backward keeps one 4-byte value in local memory
ALLOWED = {"fdx_tct_kernelILb0ELb1ELb1E": (8, 4)}   # mangled template arguments -> (stack frame, spill stores)

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _ptxas_report(src, tmp):
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
           "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", os.path.join(tmp, src + ".o")]
    return subprocess.Popen(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


def _short(name):
    m = re.search(r"(fdx_[a-z0-9]+_kernel\w*?E)(?:E?v|14CUtensorMap)", name)
    return m.group(1) if m else name


def test_wgmma_kernels_keep_their_accumulators_in_registers():
    with tempfile.TemporaryDirectory() as tmp:
        procs = [(src, _ptxas_report(src, tmp)) for src in SOURCES]
        logs = {}
        for src, p in procs:
            out, _ = p.communicate(timeout=900)
            assert p.returncode == 0, f"{src} failed to compile:\n{out[-4000:]}"
            logs[src] = out
    problems, seen = [], set()
    for src, log in logs.items():
        current = None
        for line in log.splitlines():
            note = re.search(r"\((C75(?:07|14|18|20))\).*'(\w+)'", line)
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
                frame, stores, loads = (int(g) for g in m.groups())
                allowed = next((v for k, v in ALLOWED.items() if k in current), (0, 0))
                if frame > allowed[0] or stores > allowed[1] or (loads and not allowed[1]):
                    problems.append(f"{_short(current)}: {frame} B stack frame, {stores} B spill stores, "
                                    f"{loads} B spill loads")
                current = None
    assert sum(1 for s in seen if "fdx_tc_kernel" in s) == 15, sorted(seen)
    assert any("fdx_tct_kernel" in s for s in seen) and any("fdx_wgrad9_kernel" in s for s in seen), sorted(seen)
    assert not problems, "\n".join(problems)
