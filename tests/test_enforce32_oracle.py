"""The 32-bit engine's oracle and the ABI of the _x32 exports, without a GPU.

* oracle/_ref/libk4ref32.so (upstream's engine with LZ4_hashPosition's hash5 branch off) equals the C
  restatement's LZ4Codec.Encode with enforce32, which was written from LL32's text, on inputs of 65 547 bytes to
  4 MiB at full and limited capacities; below 65 547 bytes it equals the unpatched build; and its chained blocks
  differ from the unpatched build's, so the patch takes effect where the GPU tests rely on it.
* Every _x32 export returns its twin's code for every bad argument, with or without a GPU.
"""
import numpy as np
import pytest

from tests import enforce32_ref as E
from tests import inputs


@pytest.fixture(scope="module")
def up32():
    if not E.have_ref32():
        pytest.skip("oracle/_ref/libk4ref32.so missing: run __graft_entry__.build() where the reference is present")
    return E.EncUpstream32()


@pytest.fixture(scope="module")
def ref():
    import oracle
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libk4ref.so missing")
    return oracle.Ref()


def _data(port, n: int, k: int, seed: int) -> bytes:
    """Input k % 4: datagen 0.63, datagen 0.55, text, high entropy."""
    if k % 4 < 2:
        return port.datagen(n, (0.63, 0.55)[k % 4], 0.0, seed)[:n].tobytes()
    return inputs.gen(("lorem", "random")[k % 4 - 2], n, seed)


def test_patched_upstream_equals_restatement(port, up32):
    """>= 200 inputs of 65 547 bytes .. 4 MiB (log-uniform), at full capacity and at limited ones."""
    rng = np.random.default_rng(32)
    sizes = [E.LIMIT_64K, E.LIMIT_64K + 1, 4 << 20] + [int(np.exp(x)) for x in
                                                         rng.uniform(np.log(E.LIMIT_64K), np.log(4 << 20), 200)]
    fails = 0
    for i, n in enumerate(sizes):
        src = _data(port, n, i, 1000 + i)
        bound = n + n // 255 + 16
        r, b = up32.compress_fast(src, bound)
        assert r > 0 and (r, b) == port.encode(src, bound, 0, enforce32=True), (i, n)
        for cap in (r - 1, r, r // 2, int(rng.integers(1, r + 1))):
            rl, bl = up32.compress_fast(src, cap)
            want = port.encode(src, cap, 0, enforce32=True)
            assert (rl if rl > 0 else -1) == want[0], (i, n, cap)
            assert rl <= 0 or bl == want[1], (i, n, cap)
            fails += rl <= 0
    assert fails > 0


def test_patched_upstream_below_limit_is_unchanged(port, up32, ref):
    """Below 65 547 bytes the u16 table decides, whose hash was always hash4: both builds agree."""
    rng = np.random.default_rng(33)
    for i, n in enumerate([1, 12, 13, 100, 4096, 65535, 65536, E.LIMIT_64K - 1] +
                          [int(x) for x in rng.integers(1, E.LIMIT_64K, 40)]):
        src = _data(port, n, i, 2000 + i)
        r, b = up32.compress_fast(src, n + n // 255 + 16)
        assert (r, b) == ref.encode(src), (i, n)


def test_patched_upstream_chains_differently(port, up32):
    """Chained blocks of any size hash the u32 table, so the two builds' linked blocks differ; so do one-shot
    encodes of 65 547 bytes or more."""
    from tests import chain_enc_ref as ER
    up = ER.EncUpstream()
    data = _data(port, 8 * 65536, 0, 7)
    a = up.encode_chain(data)
    st = up32.lib.LZ4_createStream()
    try:
        src = np.frombuffer(data, dtype=np.uint8)
        b = [up32.compress(st, src.ctypes.data + o, 65536, 65809)[1] for o in range(0, len(data), 65536)]
    finally:
        up32.lib.LZ4_freeStream(st)
    assert sum(x != y for x, y in zip(a, b)) >= 6
    big = data[:300000]
    assert up32.compress_fast(big, 400000) != port.encode(big, 400000)     # LL64's bytes differ too


# ---- the _x32 exports: their twins' argument checks, in the same order ------------------------------------------

def _batch_calls(L):
    """name -> (plain, x32, call(f, ptrs, n, level, memKind, device, blockSize, flags))."""
    return {
        "encode_chain_batch": (L.k4lz4_encode_chain_batch, L.k4lz4_encode_chain_batch_x32,
                               lambda f, p, n, lv, mk, d, bs, fl: f(*p(10), n, lv, mk, None, d)),
        "pickle_batch": (L.k4lz4_pickle_batch, L.k4lz4_pickle_batch_x32,
                         lambda f, p, n, lv, mk, d, bs, fl: f(*p(6), n, lv, mk, None, d)),
        "pickle_writer_batch": (L.k4lz4_pickle_writer_batch, L.k4lz4_pickle_writer_batch_x32,
                                lambda f, p, n, lv, mk, d, bs, fl: f(*p(6), n, lv, mk, None, d)),
        "frame_encode_batch": (L.k4lz4_frame_encode_batch, L.k4lz4_frame_encode_batch_x32,
                               lambda f, p, n, lv, mk, d, bs, fl: f(*p(7), n, bs, fl, lv, mk, None, d)),
    }


# (pointers, count, level, device, blockSize, flags); "real" pointers are zeroed host arrays, "neg" arrays of -1
_CASES = {
    "negative_count": ("null", -1, 0, 0, 65536, 0),
    "null_pointer": ("null", 1, 0, 0, 65536, 0),
    "empty_nulls": ("null", 0, 0, 0, 65536, 0),
    "device_out_of_range": ("real", 1, 0, "ndev", 65536, 0),
    "level_256": ("real", 1, 256, 0, 65536, 0),
    "level_negative": ("real", 1, -1, 0, 65536, 0),
    "frame_flag_8": ("real", 1, 0, 0, 65536, 8),
    "frame_block_size_0": ("real", 1, 0, 0, 0, 0),
    "frame_block_size_5m": ("real", 1, 0, 0, 5 << 20, 0),
    "negative_prefix": ("neg", 1, 0, 0, 65536, 0),
}
# the rows that would run a kernel on a GPU are left out: the pickler checks no level, the chained batch no frame
# arguments, and only the chained batch reads prefix lengths on the host
_SKIP = {("pickle_batch", c) for c in ("level_256", "level_negative", "frame_flag_8", "frame_block_size_0",
                                       "frame_block_size_5m", "negative_prefix")}
_SKIP |= {("pickle_writer_batch", c) for _, c in _SKIP}
_SKIP |= {("encode_chain_batch", c) for c in ("frame_flag_8", "frame_block_size_0", "frame_block_size_5m")}
_SKIP |= {("frame_encode_batch", "negative_prefix")}


@pytest.mark.parametrize("case", sorted(_CASES))
@pytest.mark.parametrize("mem", ["host", "device", "unknown"])
@pytest.mark.parametrize("export", ["encode_chain_batch", "frame_encode_batch", "pickle_batch", "pickle_writer_batch"])
def test_x32_batch_exports_return_their_twins_codes(native, export, mem, case):
    from tests.conftest import has_gpu
    from k4os.compression.lz4_b200 import _native as N
    if (export, case) in _SKIP or (has_gpu() and mem == "device" and _CASES[case][0] == "neg"):
        pytest.skip("would reach the device")     # device memory: prefix lengths are the kernel's to judge
    kind, n, level, dev, bs, fl = _CASES[case]
    keep = [np.zeros(64, dtype=np.int64) if kind != "neg" else np.full(64, -1, dtype=np.int64) for _ in range(10)]
    ptrs = (lambda k: [None] * k) if kind == "null" else (lambda k: [a.ctypes.data for a in keep[:k]])
    mk = {"host": N.MEM_HOST, "device": N.MEM_DEVICE, "unknown": 7}[mem]
    dev = native.k4lz4_device_count() if dev == "ndev" else dev
    plain, x32, call = _batch_calls(native)[export]
    want = call(plain, ptrs, n, level, mk, dev, bs, fl)
    got = call(x32, ptrs, n, level, mk, dev, bs, fl)
    assert got == want, (export, mem, case, got, want, native.k4lz4_last_error())
    if kind == "null" and n != 0 or mem == "unknown":
        assert want == N.E_ARG


@pytest.mark.parametrize("mem", [0, 1, 7])
@pytest.mark.parametrize("n", [-1, 0, 1])
def test_x32_group_exports_return_their_twins_codes_for_a_null_group(native, mem, n):
    from k4os.compression.lz4_b200 import _native as N
    keep = [np.zeros(64, dtype=np.int64) for _ in range(9)]
    p = [a.ctypes.data for a in keep]
    L = native
    pairs = [
        (lambda f: f(None, *p[:8], n, 0, mem, None), L.k4lz4_chain_group_encode, L.k4lz4_chain_group_encode_x32),
        (lambda f: f(None, *p[:8], n, mem, None), L.k4lz4_frame_writer_group_write,
         L.k4lz4_frame_writer_group_write_x32),
        (lambda f: f(None, *p[:5], n, mem, None), L.k4lz4_frame_writer_group_close,
         L.k4lz4_frame_writer_group_close_x32),
    ]
    for call, plain, x32 in pairs:
        assert call(x32) == call(plain) == N.E_ARG
