"""jax.random's streams, host side: the key type that selects them, and the NumPy restatements
(`utils.uniform / normal_f32 / randint / bernoulli`) that csrc/fdx_random.cu is held to bit for bit by
tests/test_prng_streams_gpu.py.  A plain tuple key keeps drawing today's torch.Generator numbers."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
from scipy.special import erfinv

from flaxdiff_b200 import utils as u
from flaxdiff_b200.trainer import rank_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

# float32 erf_inv polynomial against float64 scipy.special.erfinv, in ulps of the float32 result: what
# test_erfinv_polynomial_against_float64 observes is 3.8 for |u| <= 0.9 and 65 overall (at |u| ~ 0.9998).  The tail
# error is not the polynomial's: log1p(-u*u) sees u*u rounded to float32, which near |u| = 1 costs 1 - u*u several
# bits.  It is part of XLA's formulation, hence of JAX's draws.  The GPU test uses the same bounds.
ERFINV_ULP_CENTRAL, ERFINV_ULP_ALL = 4.0, 96.0


def erfinv_ulp_error(u32: np.ndarray, got: np.ndarray) -> np.ndarray:
    ref = erfinv(u32.astype(np.float64))
    return np.abs(got.astype(np.float64) - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)


def test_jax_key_has_the_words_of_prngkey_and_its_type_is_preserved():
    for seed in (0, 42, 2 ** 32 + 5, 2 ** 64 - 1):
        k, p = u.jax_key(seed), u.PRNGKey(seed)
        assert isinstance(k, u.ThreefryKey) and tuple(k) == p and k == p
        assert type(p) is tuple
        for a, b in zip(u.split(k, 3), u.split(p, 3)):
            assert type(a) is u.ThreefryKey and type(b) is tuple and a == b
        assert type(u.fold_in(k, 7)) is u.ThreefryKey and type(u.fold_in(p, 7)) is tuple
        assert u.fold_in(k, 7) == u.fold_in(p, 7)
        assert type(rank_key(k, 1)) is u.ThreefryKey and type(rank_key(p, 1)) is tuple and rank_key(k, 1) == rank_key(p, 1)
        sk, kk = u.RandomMarkovState(k).get_random_key()
        sp, kp = u.RandomMarkovState(p).get_random_key()
        assert type(sk.rng) is u.ThreefryKey and type(kk) is u.ThreefryKey
        assert type(sp.rng) is tuple and type(kp) is tuple and sk.rng == sp.rng and kk == kp
    assert u.key_like(u.jax_key(1), np.array([3, 4], np.uint32)) == u.ThreefryKey((3, 4))
    assert type(u.key_like((0, 1), np.array([3, 4], np.uint32))) is tuple


def test_normal_f32_reproduces_the_jax_quickstart_vector():
    # jax.random.normal(jax.random.PRNGKey(0), (10,)) printed in the JAX quick-start (as tests/test_prng.py)
    want = np.array([-0.3721109, 0.26423115, -0.18252768, -0.7368197, -0.44030377, -0.1521442,
                     -0.67135346, -0.5908641, 0.73168886, 0.5673026], dtype=np.float32)
    got = u.normal_f32(u.PRNGKey(0), 10)
    assert got.dtype == np.float32
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-7)
    np.testing.assert_allclose(got, u.normal(u.PRNGKey(0), 10), rtol=0, atol=2e-7)


def test_erfinv_polynomial_against_float64():
    rng = np.random.default_rng(0)
    lo = [np.nextafter(np.float32(-1), np.float32(0))]
    hi = [np.nextafter(np.float32(1), np.float32(0))]
    for _ in range(1023):                                   # the 2^10 float32 values nearest each end
        lo.append(np.nextafter(lo[-1], np.float32(0)))
        hi.append(np.nextafter(hi[-1], np.float32(0)))
    dist = np.exp(rng.uniform(np.log(2.0 ** -24), 0.0, 500_000)).astype(np.float32)     # log-spaced towards the ends
    x = np.concatenate([rng.uniform(-1, 1, 1_000_000).astype(np.float32), np.float32(1) - dist, dist - np.float32(1),
                        np.asarray(lo, np.float32), np.asarray(hi, np.float32)])
    x = x[np.abs(x) < 1]
    got = u.erfinv_f32(x)
    assert got.dtype == np.float32 and np.isfinite(got).all()
    err = erfinv_ulp_error(x, got)
    assert err[np.abs(x) <= 0.9].max() <= ERFINV_ULP_CENTRAL, err[np.abs(x) <= 0.9].max()
    assert err.max() <= ERFINV_ULP_ALL, (err.max(), x[err.argmax()])
    # a wrong digit in a coefficient shows as >= 1e-4 relative error
    rel = np.abs(got.astype(np.float64) - erfinv(x.astype(np.float64))) / np.abs(erfinv(x.astype(np.float64)) + 1e-300)
    assert rel[x != 0].max() < 1e-5
    z = u.normal_f32(u.PRNGKey(3), 200_001)                  # odd n: the last word of the second half is dropped
    assert np.isfinite(z).all() and abs(z.mean()) < 0.02 and abs(z.var() - 1) < 0.02


def test_uniform_range_and_bits_construction():
    key = u.PRNGKey(11)
    for lo, hi in ((0.0, 1.0), (-1.0, 1.0), (float(np.nextafter(np.float32(-1), np.float32(0))), 1.0), (3.0, 3.5)):
        x = u.uniform(key, 100_003, lo, hi)
        assert x.dtype == np.float32 and x.min() >= np.float32(lo) and x.max() < np.float32(hi)
    bits = u._random_bits32(key, 9)
    f = ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1)
    assert np.array_equal(u.uniform(key, 9), f) and np.array_equal(u.uniform(key, 9), u.uniform01(key, 9))


@pytest.mark.parametrize("span", [1, 2, 1000, 65536, 65537, 2 ** 31 - 1])
def test_randint_range(span):
    key = u.PRNGKey(5)
    lo = 0 if span == 2 ** 31 - 1 else -3
    r = u.randint(key, 20_001, lo, lo + span)
    assert r.dtype == np.int32 and r.min() >= lo and r.max() < lo + span
    if span == 1:
        assert (r == lo).all()
    if 2 < span < 2 ** 20:
        assert r.min() < lo + span // 10 and r.max() > lo + span - 1 - span // 10       # it does reach both ends
    k1, k2 = u.split(key)
    hi_bits, lo_bits = u._random_bits32(k1, 20_001).astype(np.uint64), u._random_bits32(k2, 20_001).astype(np.uint64)
    # the same in unbounded integers, every product and sum reduced mod 2^32 as uint32 arithmetic does
    mult = (65536 % span) ** 2 % 2 ** 32 % span
    want = ((hi_bits % span) * mult % 2 ** 32 + (lo_bits % span)) % 2 ** 32 % span
    assert np.array_equal(r.astype(np.int64) - lo, want.astype(np.int64))


def test_randint_power_of_two_span_is_the_low_bits_and_bernoulli_is_uniform_below_p():
    key = u.PRNGKey(9)
    _, k2 = u.split(key)
    for k in (1, 10, 16, 20):
        assert np.array_equal(u.randint(key, 1001, 0, 2 ** k), (u._random_bits32(k2, 1001) % np.uint32(2 ** k)).view(np.int32))
    for p in (0.0, 0.12, 0.5, 1.0):
        assert np.array_equal(u.bernoulli(key, p, 4097), u.uniform(key, 4097) < np.float32(p))
    assert abs(u.bernoulli(key, 0.12, 100_000).mean() - 0.12) < 0.005
    with pytest.raises(ValueError):
        u.randint(key, 4, 5, 5)


def test_plain_tuple_keys_draw_what_they_drew_before():
    key = u.split(u.PRNGKey(42))[1]
    assert type(key) is tuple

    def gen():
        return torch.Generator(device="cpu").manual_seed(u.key_to_seed(key))

    assert torch.equal(u.device_normal(key, (3, 5), "cpu"), torch.randn((3, 5), generator=gen()))
    assert torch.equal(u.device_uniform(key, (7,), "cpu"), torch.rand((7,), generator=gen()))
    assert torch.equal(u.device_randint(key, (9,), 0, 1000, "cpu"),
                       torch.randint(0, 1000, (9,), generator=gen(), dtype=torch.int32))
    assert torch.equal(u.device_bernoulli(key, 0.12, (64,), "cpu"), torch.rand((64,), generator=gen()) < 0.12)


def test_threefry_keys_have_no_cpu_path():
    from flaxdiff_b200._lib import FdxError
    with pytest.raises(FdxError):
        u.device_normal(u.jax_key(0), (4,), "cpu")
    with pytest.raises(FdxError):
        u.device_normal(u.jax_key(0), (4,), "cuda", dtype=torch.bfloat16)


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_random_kernels_have_no_spills_and_no_stack_frame():
    csrc = os.path.join(ROOT, "flaxdiff_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
                            "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c", os.path.join(csrc, "fdx_random.cu"),
                            "-o", os.path.join(tmp, "fdx_random.o")], cwd=csrc, capture_output=True, text=True,
                           timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    log = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\w*fdx_random_kernel\w*)'", log)
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(kernels) == 4 and len(frames) >= 4, log[-2000:]
    assert all(f == ("0", "0", "0") for f in frames), frames
