"""The C-ABI shared library loads without a GPU / libcuda and exports every symbol that
include/fdx.h declares, and the ctypes binding mirrors the header type for type.  No compute
entry point is called here."""
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
    assert isinstance(lib.fdx_last_error(), bytes)


# ------------------------------------------------------------------- the ctypes mirror of include/fdx.h
# _lib.SIGNATURES' mapping rule: the C type of every parameter, struct field and return value -> its ctypes type.
DESCRIPTORS = ("fdx_act", "fdx_colstats", "fdx_gemm_desc", "fdx_opt_desc", "fdx_attn_desc")
SCALARS = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float, "uint32_t": ctypes.c_uint32}
RETURNS = {"int": ctypes.c_int, "unsigned long long": ctypes.c_ulonglong, "const char*": ctypes.c_char_p}


def _ctype(c: str):
    from flaxdiff_b200 import _lib
    if c in SCALARS:
        return SCALARS[c]
    m = re.fullmatch(r"(?:const )?(\w+)\*", c)
    if m and m.group(1) in DESCRIPTORS:
        return ctypes.POINTER(getattr(_lib, m.group(1)))
    assert c.endswith("*"), f"fdx.h: no ctypes type for the C type {c!r}"
    return ctypes.c_void_p


def _norm(c: str) -> str:
    """C type with single spaces and none around '*': 'const float * const *' -> 'const float*const*'."""
    return re.sub(r"\s*\*\s*", "*", " ".join(c.split()))


def _header():
    """-> ([(name, return type, [parameter types])] of the fdx_* prototypes, {typedef name: [(field, type)]} of the
    structs), in declaration order.  Every statement must be a prototype, a struct typedef or an opaque typedef."""
    src = open(os.path.join(ROOT, "include", "fdx.h")).read()
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", src, flags=re.S)
    src = re.sub(r"#ifdef __cplusplus.*?#endif", " ", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", " ", src, flags=re.M)
    structs = {}

    def struct(m):
        fields = []
        for decl in filter(str.strip, m.group(1).split(";")):
            # one base type, then declarators: 'long long a_ld, a_s1, a_s2', 'const void* A'
            base, decls = re.fullmatch(r"\s*(.*?)\s*(\**\s*\w+(?:\s*,\s*\**\s*\w+)*)\s*", decl, re.S).groups()
            for d in decls.split(","):
                stars, field = re.fullmatch(r"(\**)\s*(\w+)", d.strip()).groups()
                fields.append((field, _norm(base + stars)))
        structs[m.group(2)] = fields
        return " "
    src = re.sub(r"typedef\s+struct\s*\w*\s*\{(.*?)\}\s*(\w+)\s*;", struct, src, flags=re.S)
    protos = []
    for stmt in src.split(";"):
        stmt = " ".join(stmt.split())
        if not stmt or re.fullmatch(r"typedef struct (\w+) \1", stmt):
            continue
        m = re.fullmatch(r"(.+?) ?\b(fdx_\w+) ?\((.*)\)", stmt)
        assert m, f"fdx.h: cannot parse {stmt!r}"
        params = []
        for p in ([] if m.group(3) == "void" else m.group(3).split(",")):
            pm = re.fullmatch(r"(.*[\s*])(\w+)", p.strip())
            assert pm, f"fdx.h: {m.group(2)}: unnamed or unparsed parameter {p!r}"
            params.append(_norm(pm.group(1)))
        protos.append((m.group(2), _norm(m.group(1)), params))
    return protos, structs


def test_signature_table_names_every_header_function():
    """_lib.SIGNATURES declares exactly the functions of include/fdx.h, in the header's order."""
    from flaxdiff_b200 import _lib
    names = [name for name, _, _ in _header()[0]]
    missing = [n for n in names if n not in _lib.SIGNATURES]
    extra = [n for n in _lib.SIGNATURES if n not in names]
    assert not missing and not extra, f"missing from _lib.SIGNATURES: {missing}; not declared in fdx.h: {extra}"
    assert list(_lib.SIGNATURES) == names, "_lib.SIGNATURES is not in fdx.h's order"


def test_signature_table_matches_header_types():
    """Each entry's restype and argtypes are the header's return and parameter types, position by position."""
    from flaxdiff_b200 import _lib
    for name, ret, params in _header()[0]:
        restype, argtypes = _lib.SIGNATURES[name]
        assert ret in RETURNS, f"{name}: no ctypes type for the return type {ret!r}"
        assert restype is RETURNS[ret], f"{name} returns {ret}: the table has {restype.__name__}"
        assert len(argtypes) == len(params), f"{name}: {len(params)} parameters in fdx.h, {len(argtypes)} in the table"
        for k, (c, t) in enumerate(zip(params, argtypes)):
            assert t is _ctype(c), f"{name}: parameter {k} is {c} ({_ctype(c).__name__}), the table has {t.__name__}"


def test_descriptor_structs_match_header():
    """fdx_act, fdx_colstats, fdx_gemm_desc, fdx_opt_desc and fdx_attn_desc: the ctypes _fields_ are the header's
    fields, with the same names and types in the same order."""
    from flaxdiff_b200 import _lib
    structs = _header()[1]
    assert sorted(structs) == sorted(DESCRIPTORS)
    for name in DESCRIPTORS:
        want = [(f, _ctype(c)) for f, c in structs[name]]
        have = list(getattr(_lib, name)._fields_)
        for k in range(max(len(want), len(have))):
            w, h = (want[k] if k < len(want) else None), (have[k] if k < len(have) else None)
            assert w == h, (f"{name} field {k}: fdx.h has {w and (w[0], w[1].__name__)}, "
                            f"_lib has {h and (h[0], h[1].__name__)}")


def test_load_declares_every_entry_point(lib):
    """After load(), every function of the header carries the table's restype and argtypes."""
    from flaxdiff_b200 import _lib
    raw = lib._lib if isinstance(lib, _lib._TracingLib) else lib
    for name, _, _ in _header()[0]:
        restype, argtypes = _lib.SIGNATURES[name]
        fn = getattr(raw, name)
        assert fn.restype is restype and tuple(fn.argtypes) == tuple(argtypes), name


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


_COLSTATS_CHILD = r"""
import ctypes, json, sys
from flaxdiff_b200 import _lib
lib = _lib.load()
base = 1 << 40                                   # fake, 16-byte aligned addresses: nothing is ever dereferenced
vp = ctypes.c_void_p


def act(i, hw, c):
    return ctypes.byref(_lib.fdx_act(base + (i << 30), 2, hw, hw, c, c))


out = []
for entry, ws_off, ld, hw in json.loads(sys.argv[1]):
    cs = ctypes.byref(_lib.fdx_colstats(base + (3 << 30) + ws_off, 4, ld))
    if entry == "conv":
        st = lib.fdx_conv3x3_fwd_stats(act(0, hw, 64), vp(base + (1 << 30)), None, None, None, act(2, hw, 64),
                                       ctypes.c_int(1), cs, None)
    else:
        st = lib.fdx_upconv3x3_fwd_stats(act(0, hw // 2, 64), vp(base + (1 << 30)), None, act(2, hw, 64), cs, None)
    out.append([st, lib.fdx_last_error().decode()])
print(json.dumps(out))
"""


def test_colstats_rejects_misaligned_workspace_and_small_images(lib):
    """fdx_conv3x3_fwd_stats / fdx_upconv3x3_fwd_stats refuse a workspace off a 16-byte boundary or with a row
    length (ld) that is not a multiple of 4 floats - the pixels-as-M epilogue adds its sums with 16-byte vector
    reductions - and, as include/fdx.h documents, outputs of fewer than 128 pixels per image.  The calls run in a
    child process that sees no GPU, on fake addresses: a check that let one through could launch nothing."""
    import json
    import subprocess
    import sys
    cases, want = [], []
    for entry, who in (("conv", "conv3x3_fwd_stats"), ("upconv", "upconv3x3_fwd_stats")):
        for ws_off, ld, hw in ((8, 320, 16), (4, 320, 16), (0, 322, 16), (0, 318, 16)):
            cases.append((entry, ws_off, ld, hw))
            want.append((-1, f"{who}: the workspace must be 16-byte aligned"))
        for hw in (8, 10) if entry == "upconv" else (8, 11):    # 64, 100 / 121 pixels
            cases.append((entry, 0, 320, hw))
            want.append((-2, f"{who}: fewer than 128 pixels per image"))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _COLSTATS_CHILD, json.dumps(cases)], capture_output=True, text=True,
                       env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for case, (status, msg), (st, prefix) in zip(cases, res, want):
        assert status == st and msg.startswith(prefix), (case, status, msg)


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under flaxdiff_b200/ may reference it."""
    for dp, _, fs in os.walk(os.path.join(ROOT, "flaxdiff_b200")):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, os.path.join(dp, f)
