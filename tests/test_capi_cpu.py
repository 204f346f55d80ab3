"""The C-ABI shared library loads without a GPU / libcuda and exports every symbol that
include/fdx.h declares.  No compute entry point is called here."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from flaxdiff_b200 import _lib
    if not os.path.exists(_lib.lib_path()):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


def test_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "fdx.h")).read()
    names = sorted(set(re.findall(r"^(?:int|const char\*|unsigned long long)\s+(fdx_[a-z0-9_]+)\s*\(", hdr, re.M)))
    assert len(names) >= 30
    for n in names:
        assert getattr(lib, n) is not None, n


def test_version_and_error_string(lib):
    assert lib.fdx_version() >= 100
    lib.fdx_last_error.restype = ctypes.c_char_p
    assert isinstance(lib.fdx_last_error(), bytes)


def test_no_libcuda_link_dependency():
    """libfdx must load on a box without the driver: TMA descriptors are encoded through
    cudaGetDriverEntryPoint at run time, cudart is linked statically."""
    import subprocess
    from flaxdiff_b200 import _lib
    out = subprocess.run(["ldd", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out and "libtorch" not in out


def test_ops_refuse_cpu_tensors(lib):
    import torch
    from flaxdiff_b200 import ops
    from flaxdiff_b200._lib import FdxError
    x = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16)
    with pytest.raises(FdxError):
        ops.groupnorm_stats(x, 8)


_ATTN_CHILD = r"""
import ctypes, json, sys
from flaxdiff_b200 import _lib
lib = _lib.load()
base = 1 << 40                                   # fake, 16-byte aligned addresses: nothing is ever dereferenced
B, heads, dh, L, Lk = 2, 8, 64, 100, 77
HD = heads * dh


def desc():
    a = _lib.fdx_attn_desc()
    a.B, a.heads, a.L, a.Lk, a.dh, a.scale = B, heads, L, Lk, dh, 0.125
    for i, (t, rows) in enumerate((("q", L), ("k", Lk), ("v", Lk), ("o", L), ("do", L), ("dq", L), ("dk", Lk),
                                   ("dv", Lk))):
        setattr(a, "d_o" if t == "do" else t, base + i * (1 << 30))
        setattr(a, t + "_ld", HD)
        setattr(a, t + "_bs", rows * HD)
    a.lse, a.dvec_ws = base + (9 << 30), base + (10 << 30)
    return a


out = []
for entry, field, value in json.loads(sys.argv[1]):
    a = desc()
    setattr(a, field, (base + value) if value < 16 else value)
    fn = lib.fdx_attention_fwd if entry == "fwd" else lib.fdx_attention_bwd
    st = fn(ctypes.byref(a), None)
    out.append([st, lib.fdx_last_error().decode()])
print(json.dumps(out))
"""


def test_attention_rejects_misaligned_strides_and_pointers(lib):
    """fdx_attention_fwd / _bwd refuse, naming the field, every row / batch stride that is not a multiple of
    8 elements and every tensor pointer off a 16-byte boundary: the kernels access o, d_o, dq, dk, dv with
    16-byte (and 4-byte) vector loads and stores, and TMA reads q, k, v, d_o in 16-byte units.  The calls run in
    a child process that sees no GPU, on fake addresses: a check that let one through could launch nothing."""
    import json
    import subprocess
    import sys
    cases = []
    for entry, tensors in (("fwd", ("q", "k", "v", "o")), ("bwd", ("q", "k", "v", "o", "do", "dq", "dk", "dv"))):
        for t in tensors:
            cases += [(entry, t + "_ld", 8 * 64 + 4), (entry, t + "_bs", 100 * 8 * 64 + 2)]
            cases.append((entry, "d_o" if t == "do" else t, 8))          # base + 8 bytes: 8- but not 16-aligned
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _ATTN_CHILD, json.dumps(cases)], capture_output=True, text=True,
                       env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for (entry, field, _), (status, msg) in zip(cases, res):
        who = "attention_fwd" if entry == "fwd" else "attention_bwd"
        assert status == -1 and msg.startswith(f"{who}: {field} must be"), (entry, field, status, msg)


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under flaxdiff_b200/ may reference it."""
    for dp, _, fs in os.walk(os.path.join(ROOT, "flaxdiff_b200")):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, f)
