"""Chained block encoding without a GPU: the reference's encoder ring (LZ4EncoderBase + LZ4FastChainEncoder)
restated over upstream, the prefix-length rule of k4lz4_encode_chain_batch, and the new export's argument checks.

The ring tests need upstream's engine (oracle/_ref/, built by __graft_entry__.build() where the reference is
present); without it they are skipped."""

import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests.conftest import has_gpu

# LZ4EncoderTests.cs:31-36,46-53,63-64 (block size, total, extraBlocks), plus 1 MiB and 4 MiB blocks
ROWS = [(1024, 50, 0), (1024, 1024, 0), (1024, 1026, 0), (1024, 1100, 0), (1024, 0x10000, 0), (1024, 0x20000, 100),
        (0x10000, 50, 0), (0x10000, 0x10000, 0), (0x10000, 0x20000, 0), (0x10000, 0x20000, 5),
        (0x10000, 0x20000, 1), (0x10000, 0x20000, 10), (0x10000, 0x50000, 0), (0x10000, 0x50000, 5),
        (0x20000, 0x50000, 1), (0x20000, 0x100000, 1), (1 << 20, 3 << 20, 0), (4 << 20, 9 << 20, 1)]


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.skip("upstream's engine is not built (oracle/_ref/)")
    return ER.EncUpstream()


def _content(n: int, seed: int = 1) -> bytes:
    import oracle
    return oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n].tobytes()


@pytest.mark.parametrize("bs,total,extra", ROWS)
def test_ring_model_equals_contiguous_and_prefix_rule(up, bs, total, extra):
    """The ring (saveDict relocating the history) gives the bytes of one contiguous stream, and before every call
    the prefix the GPU would be given (the ring's _inputIndex) is upstream's dictSize, so that
    min(dictSize, prefixLen) + n is upstream's dictSize after the call."""
    total = (total + bs - 1) // bs * bs                     # FastStreamEncoder rounds the length up
    data = _content(total, bs + total)
    want = up.encode_chain(data, bs)
    ring = ER.RingModel(up, bs, extra)
    cap = ring.block + ring.block // 255 + 16
    got, o = [], 0
    try:
        while o < len(data):
            o += ring.topup(data[o:o + ring.block])
            r, out, P, before, after = ring.encode(cap, False)
            after = after.view(np.uint32)
            b32 = before.view(np.uint32)
            got.append(out)
            assert P == b32[4097]
            n = int(after[4096] - b32[4096])                # currentOffset advances by n
            assert n > 0 and after[4097] == min(int(b32[4097]), P) + n
    finally:
        ring.close()
    assert got == want


def test_fresh_first_block_equals_prefix_p0(up):
    """A fresh LZ4_stream_t (dictionary NULL) takes upstream's external-dictionary branch with dictSize 0; it gives
    the same bytes, result and state as the prefix mode with no history that the GPU implements."""
    for i, n in enumerate([1, 4, 12, 13, 100, 65535, 65536, 65547, 300000]):
        src = _content(n, 10 + i)
        st = up.lib.LZ4_createStream()
        a = np.frombuffer(src, dtype=np.uint8)
        try:
            for cap in (n + n // 255 + 16, max(n // 3, 1)):
                up.lib.LZ4_freeStream(st)
                st = up.lib.LZ4_createStream()
                assert up.view(st).dictionary is None
                r, out = up.compress(st, a.ctypes.data, n, cap)
                want = (r, out, up.state_of(st))
                got = up.step(ER.make_state(), b"", src, cap)
                assert got[:2] == want[:2] and np.array_equal(got[2], want[2]), (n, cap)
        finally:
            up.lib.LZ4_freeStream(st)


def test_step_clamps_history_like_save_dict(up):
    """step() with a long history and dictSize D equals upstream after LZ4_saveDict(min(P, 64 KiB)) on a real
    contiguous stream: the prefix rule is saveDict's clamp."""
    data = _content(300000, 3)
    a = np.frombuffer(data, dtype=np.uint8)
    for P in (0, 1, 3, 4, 65534, 65535, 65536, 70000):
        st = up.lib.LZ4_createStream()
        try:
            up.compress(st, a.ctypes.data, 200000, 1 << 20)
            before = up.state_of(st)
            safe = np.zeros(65536 + 100000 + 16, dtype=np.uint8)
            k = int(up.lib.LZ4_saveDict(st, safe.ctypes.data, P))
            assert k == min(P, 65536)
            safe[k:k + 100000] = a[200000:300000]
            want = up.compress(st, safe.ctypes.data + k, 100000, 1 << 20), up.state_of(st)
        finally:
            up.lib.LZ4_freeStream(st)
        r, out, after = up.step(before, data[200000 - P:200000], data[200000:], 1 << 20)
        if P > 65536:       # saveDict keeps at most 64 KiB; the prefix rule keeps dictSize = P, which no match can tell
            w = want[1].view(np.uint32).copy()
            w[4097] = P + 100000
            want = want[0], w.view(np.uint8)
        assert (r, out) == want[0] and np.array_equal(after, want[1]), P


# ---- argument errors of k4lz4_encode_chain_batch ----------------------------------------------------------------

def _args(n=1, prefix=0, state_off=0, level=0):
    keep = dict(src=np.zeros(64, np.uint8), so=np.zeros(n, np.int64), sl=np.full(n, 16, np.int32),
                pl=np.full(n, prefix, np.int32), dst=np.zeros(256, np.uint8), do=np.zeros(n, np.int64),
                dc=np.full(n, 64, np.int32), st=np.zeros(ER.STATE_BYTES + 32, np.uint8),
                sto=np.full(n, state_off, np.int64), out=np.zeros(n, np.int32))
    ptrs = [keep[k].ctypes.data for k in ("src", "so", "sl", "pl", "dst", "do", "dc", "st", "sto", "out")]
    return keep, ptrs, level


def _call(native, ptrs, n, level, mem):
    return native.k4lz4_encode_chain_batch(*ptrs, n, level, mem, None, 0)


def test_argument_error_matrix(native):
    """Unknown memKind, negative count, each required pointer NULL (three memKinds), host-memory contents
    (negative prefixLen, a state offset that is not a multiple of 16, a bad level), in check()'s order; then the
    machine."""
    from k4os.compression.lz4_b200 import _native as N
    gpu = has_gpu()
    err = lambda: native.k4lz4_last_error().decode()
    for mem in (N.MEM_HOST, N.MEM_DEVICE, 7):
        keep, ptrs, lv = _args()
        if mem == 7:
            assert _call(native, ptrs, 1, 0, mem) == N.E_ARG and "memKind" in err()
            p = list(ptrs); p[0] = None
            assert _call(native, p, 1, 0, mem) == N.E_ARG and "memKind" in err()     # memKind before pointers
            continue
        assert _call(native, ptrs, -1, 0, mem) == N.E_ARG and "count" in err()
        for i in range(10):
            p = list(ptrs); p[i] = None
            assert _call(native, p, 1, 0, mem) == N.E_ARG and "null" in err(), (mem, i)
        p = list(ptrs); p[7] = None
        assert _call(native, p, 0, 0, mem) in (N.OK, N.E_NODEVICE)                    # nothing is read when n == 0
    # host-memory contents, after the pointers
    for kw, word in ((dict(prefix=-1), "prefix"), (dict(state_off=8), "multiple of 16"), (dict(level=256), "level"),
                     (dict(level=-1), "level")):
        keep, ptrs, lv = _args(**kw)
        assert _call(native, ptrs, 1, lv, N.MEM_HOST) == N.E_ARG and word in err(), kw
        p = list(ptrs); p[4] = None
        assert _call(native, p, 1, lv, N.MEM_HOST) == N.E_ARG and "null" in err(), kw
    keep, ptrs, lv = _args(prefix=-1)
    assert _call(native, ptrs, 1, 0, 7) == N.E_ARG and "memKind" in err()
    # then the machine: valid arguments
    keep, ptrs, lv = _args(n=0)
    assert _call(native, ptrs, 0, 0, N.MEM_HOST) == (N.OK if gpu else N.E_NODEVICE)
    if not gpu:
        keep, ptrs, lv = _args()
        assert _call(native, ptrs, 1, 0, N.MEM_HOST) == N.E_NODEVICE
        assert native.k4lz4_encode_chain_batch(*ptrs, 1, 0, N.MEM_HOST, None, 99) == N.E_NODEVICE
    else:
        keep, ptrs, lv = _args()
        ndev = native.k4lz4_device_count()
        assert native.k4lz4_encode_chain_batch(*ptrs, 1, 0, N.MEM_HOST, None, ndev) == N.E_ARG


def test_encoder_factory_and_hc():
    from k4os.compression.lz4_b200 import LZ4Encoder, LZ4FastChainEncoder, LZ4BlockEncoder, LZ4Level
    e = LZ4Encoder.Create(True, LZ4Level.L00_FAST, 1000, 2)
    assert isinstance(e, LZ4FastChainEncoder) and e.BlockSize == 1024
    assert e._in_len == 65536 + 3 * 1024 + 32
    assert isinstance(LZ4Encoder.Create(False, LZ4Level.L00_FAST, 4096), LZ4BlockEncoder)
    with pytest.raises(NotImplementedError):
        LZ4Encoder.Create(True, LZ4Level.L03_HC, 65536)
    assert e.Topup(b"x" * 5000) == 1024 and e.Topup(b"y") == 0 and e.BytesReady == 1024
