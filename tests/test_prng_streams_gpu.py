"""csrc/fdx_random.cu against the host restatements of jax.random's draws in flaxdiff_b200/utils.py, through
`ops` (the C ABI): bits, uniform and randint bit for bit; normal bit for bit up to CUDA's log1pf / sqrtf and in any
case inside the float64 bound of tests/test_prng_streams_cpu.py."""
import numpy as np
import pytest
import torch
from scipy.special import erfinv

from flaxdiff_b200 import ops
from flaxdiff_b200 import utils as u
from flaxdiff_b200._lib import FdxError

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

SIZES = [1, 2, 3, 7, 8, 9, 1023, 1024, 1025, 2 ** 20 + 1, 3_145_728, 6_291_456]
KEYS = [(0, 0), (2 ** 32 - 1, 2 ** 32 - 1), u.PRNGKey(42), u.split(u.PRNGKey(42))[1]]
SENTINEL = 0x5A5A5A5A
PAD = 8
# the bounds tests/test_prng_streams_cpu.py establishes for the float32 erf_inv polynomial against float64 (ulps of
# the result), plus 2 ulp for CUDA's log1pf (1 ulp) and the final multiplication by sqrt(2)
ERFINV_ULP_CENTRAL, ERFINV_ULP_ALL = 4.0 + 2, 96.0 + 2


def _draw(fn, key, n, dtype, offset_words=0, **kw):
    """fn(key, (n,), out=...) into the middle of a sentinel-filled buffer; returns the n words as uint32 after
    checking that nothing around them was written."""
    buf = torch.full((PAD + offset_words + n + PAD,), SENTINEL, dtype=torch.int32, device=dev)
    out = buf[PAD + offset_words: PAD + offset_words + n].view(dtype)
    assert out.data_ptr() % 16 == (4 * offset_words) % 16
    fn(key, (n,), out=out, **kw)
    host = buf.cpu().numpy().view(np.uint32)
    assert (host[:PAD + offset_words] == SENTINEL).all() and (host[PAD + offset_words + n:] == SENTINEL).all()
    return host[PAD + offset_words: PAD + offset_words + n]


@pytest.mark.parametrize("key", KEYS, ids=["zero", "ones", "key42", "child"])
def test_random_bits_bit_for_bit(key):
    for n in SIZES:
        assert np.array_equal(_draw(ops.random_bits, key, n, torch.int32), u._random_bits32(key, n)), n


@pytest.mark.parametrize("offset_words", [1, 2, 3])
def test_random_bits_at_unaligned_outputs(offset_words):
    """Output pointers 4, 8 and 12 bytes past a 16-byte boundary, even and odd n: the ragged edges of the two
    halves' vector stores."""
    key = u.PRNGKey(42)
    for n in (1, 2, 3, 7, 8, 9, 1023, 1024, 1025, 2049, 4101, 2 ** 20 + 1):
        assert np.array_equal(_draw(ops.random_bits, key, n, torch.int32, offset_words), u._random_bits32(key, n)), n


def test_random_uniform_and_randint_bit_for_bit():
    key = u.split(u.PRNGKey(42))[0]
    lo = float(np.nextafter(np.float32(-1), np.float32(0)))
    for n in SIZES:
        for a, b in ((lo, 1.0), (0.0, 1.0)):
            got = _draw(ops.random_uniform, key, n, torch.float32, n % 4, minval=a, maxval=b).view(np.float32)
            assert np.array_equal(got, u.uniform(key, n, a, b)), (n, a, b)
        for lo_i, hi_i in ((0, 1000), (-5, 65532)):                  # spans 1000 (the DDPM timesteps) and 65 537
            got = _draw(ops.random_randint, key, n, torch.int32, n % 4, minval=lo_i, maxval=hi_i).view(np.int32)
            assert np.array_equal(got, u.randint(key, n, lo_i, hi_i)), (n, lo_i, hi_i)
    for span in (1, 2, 65536, 2 ** 31 - 1):
        got = _draw(ops.random_randint, key, 4099, torch.int32, minval=0, maxval=span).view(np.int32)
        assert np.array_equal(got, u.randint(key, 4099, 0, span)), span


def _normal_ulp_error(key, z):
    """Error of z = the kernel's normal draw against float64 sqrt(2) * erfinv of the SAME float32 uniform, in ulps."""
    x = u.uniform(key, z.size, u._NORMAL_LO, 1.0)
    ref = float(np.float32(np.sqrt(2.0))) * erfinv(x.astype(np.float64))
    return x, np.abs(z.astype(np.float64) - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)


def test_random_normal_against_host_polynomial_and_float64():
    want = np.array([-0.3721109, 0.26423115, -0.18252768, -0.7368197, -0.44030377, -0.1521442,
                     -0.67135346, -0.5908641, 0.73168886, 0.5673026], dtype=np.float32)     # the JAX quick-start
    got = ops.random_normal(u.PRNGKey(0), (10,), device=dev).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-7)
    key = u.split(u.PRNGKey(42))[1]
    for n in (1, 3, 1025, 2 ** 20 + 1, 6_291_456):
        z = _draw(ops.random_normal, key, n, torch.float32, n % 4).view(np.float32)
        assert np.isfinite(z).all()
        host = u.normal_f32(key, n)
        same = z == host
        # where they differ, CUDA's log1pf / sqrtf rounded w differently from NumPy's: a last-bits effect
        np.testing.assert_allclose(z[~same], host[~same], rtol=2e-5, atol=0)
        x, err = _normal_ulp_error(key, z)
        central = np.abs(x) <= 0.9
        assert not central.any() or err[central].max() <= ERFINV_ULP_CENTRAL, err[central].max()
        assert err.max() <= ERFINV_ULP_ALL, err.max()
    # moments of the 6 291 456 draws inside 5 sigma of their sampling error
    zz = z.astype(np.float64)
    n = zz.size
    assert abs(zz.mean()) < 5 / np.sqrt(n)
    assert abs(zz.var() - 1) < 5 * np.sqrt(2 / n)
    assert abs(((zz - zz.mean()) ** 4).mean() / zz.var() ** 2 - 3) < 5 * np.sqrt(24 / n)


def _words(key):
    return torch.from_numpy(np.asarray(key, dtype=np.uint32).view(np.int32)).to(dev)


def test_key_from_device_memory_equals_key_by_value():
    key = u.split(u.PRNGKey(7))[0]
    kd = _words(key)
    n = 100_003
    assert torch.equal(ops.random_bits(kd, (n,)), ops.random_bits(key, (n,), device=dev))
    assert torch.equal(ops.random_uniform(kd, (n,), -1.0, 1.0), ops.random_uniform(key, (n,), -1.0, 1.0, device=dev))
    assert torch.equal(ops.random_randint(kd, (n,), 0, 1000), ops.random_randint(key, (n,), 0, 1000, device=dev))
    a, b = ops.random_normal(kd, (n,)), ops.random_normal(key, (n,), device=dev)
    assert torch.equal(a, b) and torch.equal(b, ops.random_normal(key, (n,), device=dev))     # and repeatable


def test_graph_replay_draws_from_the_key_the_device_words_hold():
    k1, k2 = u.split(u.PRNGKey(11))
    kd = _words(k1)
    out = torch.empty(50_001, dtype=torch.float32, device=dev)
    ops.random_normal(kd, out.shape, out=out)                       # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.random_normal(kd, out.shape, out=out)
    out.zero_()
    g.replay()
    assert torch.equal(out, ops.random_normal(k1, out.shape, device=dev))
    kd.copy_(_words(k2))                                            # overwrite the 8 key bytes
    g.replay()
    assert torch.equal(out, ops.random_normal(k2, out.shape, device=dev))
    assert not torch.equal(out, ops.random_normal(k1, out.shape, device=dev))


def test_shaped_draw_is_the_flat_draw_reshaped_and_device_dispatch():
    key = u.jax_key(3)
    flat = ops.random_normal(key, (3072,), device=dev)
    assert torch.equal(u.device_normal(key, (4, 16, 16, 3), dev), flat.view(4, 16, 16, 3))
    assert torch.equal(u.device_normal(u.DeviceKey(_words(key)), (4, 16, 16, 3), dev), flat.view(4, 16, 16, 3))
    assert np.array_equal(u.device_uniform(key, (5, 7), dev).cpu().numpy().reshape(-1), u.uniform(key, 35))
    assert np.array_equal(u.device_randint(key, (33,), 0, 1000, dev).cpu().numpy(), u.randint(key, 33, 0, 1000))
    assert np.array_equal(u.device_bernoulli(key, 0.12, (4097,), dev).cpu().numpy(), u.bernoulli(key, 0.12, 4097))
    assert ops.random_normal(key, (0,), device=dev).numel() == 0
    # a plain tuple with the same words keeps torch's generator
    g = torch.Generator(device=dev).manual_seed(u.key_to_seed(tuple(key)))
    assert torch.equal(u.device_normal(tuple(key), (64,), dev), torch.randn((64,), generator=g, device=dev))


def test_ops_refuse_bad_arguments_without_launching():
    from flaxdiff_b200 import _lib
    lib = _lib.load()
    before = lib.fdx_launch_count()
    key = u.PRNGKey(1)
    with pytest.raises(FdxError):
        ops.random_normal(key, (8,), out=torch.empty(8))                         # CPU output
    with pytest.raises(FdxError):
        ops.random_bits(torch.zeros(2, dtype=torch.int32), (8,), device=dev)     # CPU key words
    with pytest.raises(FdxError):
        ops.random_normal(key, (-1,), device=dev)
    with pytest.raises(FdxError):
        ops.random_normal(key, (8,), device="cpu")
    with pytest.raises(FdxError):
        ops.random_uniform(key, (8,), 1.0, 1.0, device=dev)
    with pytest.raises(FdxError):
        ops.random_randint(key, (8,), 5, 5, device=dev)
    with pytest.raises(FdxError):
        ops.random_normal(key, (8,), out=torch.empty(9, device=dev))
    import ctypes
    st = lib.fdx_random_normal(ctypes.c_uint32(0), ctypes.c_uint32(0), None, ctypes.c_longlong(-1), None, None)
    assert st == -1 and b"random_normal" in lib.fdx_last_error()
    assert lib.fdx_launch_count() == before
