"""Frame writer groups without a GPU: the incremental LZ4FrameWriter model (tests/frame_writer_ref.py) against the
whole-content frame writers, its emission schedule, streaming XXH32, the bound arithmetic, and the argument checks
of the k4lz4_frame_writer_* exports.  The engine comparisons need upstream's engine (oracle/_ref/)."""
import ctypes as C
import struct

import numpy as np
import pytest

from tests import frame_writer_ref as FW
from tests.conftest import has_gpu

E_ARG, E_NODEVICE, R_DELEGATE = -102, -100, -2


def _content(n: int, seed: int) -> bytes:
    import oracle
    rng = np.random.default_rng(seed)
    a = oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n].copy()
    if n > 3000:                                           # an incompressible stretch: raw blocks
        at = int(rng.integers(0, n // 2))
        k = min(n - at, 70000)
        a[at:at + k] = rng.integers(0, 256, k, dtype=np.uint8)
    return a.tobytes()


def chunkings(n: int, B: int, rng) -> list:
    """Cuts of n bytes into writes: the edge sizes around 16 and B, then random ones, each with 0-byte writes."""
    edge = [0, 1, 15, 16, 17, B - 1, B, B + 1, 3 * B + 17]
    out = []
    for pick in (lambda: edge[int(rng.integers(0, len(edge)))], lambda: int(rng.integers(0, 2 * B)),
                 lambda: int(rng.integers(0, 40))):
        cuts, at = [], 0
        while at < n:
            k = min(pick(), n - at)
            cuts.append(k)
            at += k
        out.append(cuts or [0])
    out.append([n])
    out.append([0, n, 0])
    return out


def _split(data: bytes, cuts) -> list:
    out, at = [], 0
    for k in cuts:
        out.append(data[at:at + k])
        at += k
    return out


@pytest.fixture(scope="module")
def engines():
    import oracle
    if not oracle.have_ref():
        pytest.skip("upstream's engine (oracle/_ref/) is not built")
    from tests import chain_enc_ref as ER
    return ER.EncUpstream(), oracle.Ref()


@pytest.mark.parametrize("chaining", [True, False])
@pytest.mark.parametrize("bs", [1024, 4096, 65536])
def test_model_concatenation_equals_whole_frame(engines, chaining, bs):
    """For every chunking, the writes' and the close's bytes concatenated equal the reference writer over the
    whole content; each write ends exactly after the last block its cumulative content completes."""
    from tests import chain_enc_ref as ER
    from tests.test_gpu_frames import indep_ref
    up, ref = engines
    rng = np.random.default_rng(bs + chaining)
    B = FW.rounded_block(bs)
    for n in (0, 1, 15, 16, 17, B - 1, B, B + 1, 3 * B + 17, 70000 + 5 * B):
        data = _content(n, n + bs)
        for bc, cc in ((False, False), (True, True), (bool(n & 1), not n & 1)):
            if bs == 65536:
                want = (ER.frame_linked_ref(up, data, bs, bc, cc) if chaining else indep_ref(ref, data, bs, bc, cc))
            else:
                want = b"".join(FW.emit(FW.Writer(bs, chaining, bc, cc, FW.UpstreamEngine(up, ref, chaining)), [data]))
            for cuts in chunkings(n, B, rng):
                w = FW.Writer(bs, chaining, bc, cc, FW.UpstreamEngine(up, ref, chaining))
                parts = FW.emit(w, _split(data, cuts))
                assert b"".join(parts) == want, (n, cuts[:8])
                # each write emits the blocks its cumulative content completes, nothing more
                done, at = 0, 0
                for i, k in enumerate(cuts):
                    done += k
                    nb = done // B
                    end = 7 + sum(len(x) for x in _blocks(want, bc)[:nb])
                    at += len(parts[i])
                    assert at == end, (n, i)


def _blocks(frame: bytes, bc: bool) -> list:
    """The stored blocks of a frame (length code, body, checksum) as byte strings."""
    out, p = [], 7
    while True:
        code = struct.unpack_from("<I", frame, p)[0]
        if code == 0:
            return out
        k = 4 + (code & 0x7FFFFFFF) + 4 * bc
        out.append(frame[p:p + k])
        p += k


def test_model_empty_write_and_close(engines):
    up, ref = engines
    for chaining in (True, False):
        for bc in (False, True):
            for cc in (False, True):
                w = FW.Writer(65536, chaining, bc, cc, FW.UpstreamEngine(up, ref, chaining))
                assert w.close() == b""                                   # never written: nothing
                h = w.write(b"")
                assert h == FW.header(65536, chaining, bc, cc) and len(h) == 7
                tail = w.close()
                assert tail == struct.pack("<I", 0) + (struct.pack("<I", ref.xxh32(b"")) if cc else b"")
                assert w.close() == b""                                   # closed: new again
                assert w.write(b"abc")[:7] == h                           # a new frame


def test_header_equals_reference_writer(engines):
    _, ref = engines
    for bs, code in ((1, 4), (65536, 4), (65537, 5), (100000, 5), (1 << 18, 5), (1 << 20, 6), (4 << 20, 7)):
        for fl in range(8):
            h = FW.header(bs, not fl & 1, bool(fl & 2), bool(fl & 4))
            assert h[:4] == b"\x04\x22\x4d\x18" and h[5] == code << 4
            assert h[6] == (ref.xxh32(h[4:6]) >> 8) & 0xFF


def test_streaming_xxh32_equals_whole_buffer(native):
    rng = np.random.default_rng(7)
    for n in (0, 1, 15, 16, 17, 31, 32, 33, 100, 1000, 70001):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        buf = np.frombuffer(data + b"\0", dtype=np.uint8)
        want = int(native.k4lz4_xxh32(buf.ctypes.data, n, 0))
        assert FW.xxh32(data) == want
        for _ in range(6):
            s = FW.XXH32Stream()
            at = 0
            while at < n:
                k = int(rng.choice([0, 1, 3, 15, 16, 17, int(rng.integers(0, 64))]))
                s.update(data[at:at + k])
                at += k
            assert s.digest() == want, n


@pytest.mark.parametrize("bs", [1, 1000, 1024, 65536, 65537, 100000, 1 << 20, 4 << 20])
def test_bounds(bs):
    B = FW.rounded_block(bs)
    assert B == max(1024, -(-bs // 1024) * 1024)
    for bc in (False, True):
        for L in (0, 1, B - 1, B, B + 1, 5 * B + 3):
            want = 7 + (B - 1 + L) // B * (4 + B + 4 * bc)
            assert FW.write_bound(L, bs, bc) == want
        for cc in (False, True):
            assert FW.close_bound(bs, bc, cc) == 4 + B + 4 * bc + 4 + 4 * cc


def test_argument_errors_without_device(native):
    """K4LZ4_E_ARG for bad arguments whether or not a device exists; good ones reach the device check."""
    if has_gpu():
        pytest.skip("this matrix is for a machine without a GPU")
    L = native
    g = C.c_void_p()
    for args in ((0, 65536, 0, 0), (-1, 65536, 0, 0), (4, 0, 0, 0), (4, (4 << 20) + 1, 0, 0), (4, 65536, 8, 0),
                 (4, 65536, 0, -1), (4, 65536, 0, 256)):
        assert L.k4lz4_frame_writer_group_create(*args, 0, C.byref(g)) == E_ARG, args
        assert g.value is None
    assert L.k4lz4_frame_writer_group_create(4, 65536, 0, 0, 0, None) == E_ARG
    assert L.k4lz4_frame_writer_group_create(4, 65536, 0, 3, 0, C.byref(g)) == R_DELEGATE and g.value is None
    assert L.k4lz4_frame_writer_group_create(4, 65536, 7, 0, 0, C.byref(g)) == E_NODEVICE and g.value is None
    s = np.zeros(4, np.int32)
    o = np.zeros(4, np.int64)
    n = np.zeros(4, np.int32)
    b = np.zeros(16, np.uint8)
    p = [s.ctypes.data, b.ctypes.data, o.ctypes.data, n.ctypes.data, b.ctypes.data, o.ctypes.data, n.ctypes.data,
         n.ctypes.data]
    assert L.k4lz4_frame_writer_group_write(None, *p, 1, 0, None) == E_ARG
    assert L.k4lz4_frame_writer_group_close(None, s.ctypes.data, b.ctypes.data, o.ctypes.data, n.ctypes.data,
                                            n.ctypes.data, 1, 0, None) == E_ARG
    assert L.k4lz4_frame_writer_group_reset(None, s.ctypes.data, 1, 0, None) == E_ARG
    assert L.k4lz4_frame_writer_group_destroy(None) == 0
    assert L.k4lz4_frame_writer_bound(None, 10) == E_ARG
    assert L.k4lz4_frame_writer_close_bound(None) == E_ARG


def test_python_mirror_delegates_hc_levels(native):
    from k4os.compression.lz4_b200 import FrameWriterGroup, _native
    with pytest.raises(NotImplementedError):
        FrameWriterGroup(4, 65536, level=3)
    with pytest.raises(_native.K4Error) as e:
        FrameWriterGroup(4, 0)
    assert e.value.code == E_ARG
