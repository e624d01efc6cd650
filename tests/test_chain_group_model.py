"""Chain groups without a GPU: the group's history rule (tests/chain_group_ref.py) against the reference's ring
buffers, and the argument checks of the k4lz4_chain_group_* exports.

The rule: a stream's history is its last min(total, 65 536) bytes, and the last 64 KiB slide to the front of its
ring when the next block might not fit.  It must give the reference's bytes for every blockSize / extraBlocks of
LZ4FastChainEncoder and LZ4ChainDecoder.  With upstream's engine built (oracle/_ref/) the encoder is compared with
the reference ring over upstream (bytes and state after every block) and the decoder with LZ4ChainDecoder over
upstream's LZ4_streamDecode_t.  Without it, the history bookkeeping of both directions still runs against the
reference's rings restated in Python, and digests of the results are compared with those recorded from upstream
in tests/golden/chain_group_digests.json (regenerate with ``python -m tests.test_chain_group_model``)."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

from tests import chain_enc_ref as ER
from tests import chain_group_ref as GR
from tests import chain_ref as CR
from tests.conftest import ROOT, has_gpu

K64 = 65536
DIGESTS = os.path.join(ROOT, "tests", "golden", "chain_group_digests.json")
ENC_CASES = [(bs, extra) for bs in (1024, 4096, 65536, 1 << 20) for extra in (0, 1, 3)]
DEC_CASES = [(bs, extra) for bs in (1024, 4096, 65536) for extra in (0, 1, 3)]


def _have_ref() -> bool:
    import oracle
    return oracle.have_ref()


def _enc_lengths(bs: int, seed: int) -> list:
    """Block lengths of one stream: full, short and 1-byte blocks, enough to wrap the largest ring (extraBlocks 3)
    and the group's ring at least twice."""
    rng = np.random.default_rng(seed)
    need = 2 * (K64 + 4 * bs + 32) + 3 * K64
    out, tot = [], 0
    while tot < need:
        k = int(rng.choice([bs, bs, bs, 1, int(rng.integers(1, bs + 1))]))
        out.append(k)
        tot += k
    return out


def _content(n: int, seed: int) -> bytes:
    import oracle
    return oracle.Port().datagen(max(n, 1), 0.63, 0.0, seed)[:n].tobytes()


class _RefEncRing:
    """LZ4EncoderBase.cs:27-97 + LZ4FastChainEncoder.cs bookkeeping without an engine: the ring, _inputIndex and
    LZ4_saveDict's length, with dictSize advanced by the kernel's rule min(dictSize, prefix) + n."""

    def __init__(self, bs: int, extra: int):
        self.block = bs
        self.in_len = K64 + (1 + extra) * bs + 32
        self.buf = np.zeros(self.in_len + 8, dtype=np.uint8)
        self.index = 0
        self.dict_size = 0

    def encode(self, src: bytes):
        """-> (prefix, the dictionary the engine sees) of the block, then commits it."""
        P = self.index
        d = min(self.dict_size, P)
        window = self.buf[P - min(d, 65535):P].tobytes()
        n = len(src)
        self.buf[P:P + n] = np.frombuffer(src, dtype=np.uint8)
        self.dict_size = d + n
        self.index = P + n
        if self.index + self.block > self.in_len:                    # Commit -> CopyDict = LZ4_saveDict
            size = min(self.index, K64, self.dict_size)
            self.buf[:size] = self.buf[self.index - size:self.index].copy()
            self.index = self.dict_size = size
        return P, d, window


def _equivalent_dict(d_group: int, d_ref: int) -> bool:
    """Two dictionary lengths the engine cannot tell apart: equal, or both a full window (no offset exceeds 65 535,
    no catch-up reaches below -65 535, dictSmall needs < 65 536)."""
    return d_group == d_ref or (d_group >= K64 and d_ref >= K64)


def _dict_size_ok(group_state: np.ndarray, ref_state: np.ndarray) -> bool:
    g, r = group_state.view(np.uint32), ref_state.view(np.uint32)
    return (np.array_equal(g[:4097], r[:4097]) and _equivalent_dict(int(g[4097]), int(r[4097]))
            and np.array_equal(g[4098:], r[4098:]))


@pytest.mark.parametrize("bs,extra", ENC_CASES)
def test_encoder_history_rule_bookkeeping(bs, extra):
    """Before every block: the group's history is the stream's last min(total, 64 KiB) bytes, and the dictionary
    the kernel sees through it (min(dictSize, prefix)) is equivalent to the reference ring's and ends in the same
    bytes.  No engine is needed."""
    lengths = _enc_lengths(bs, bs + extra)
    data = np.random.default_rng(bs * 7 + extra).integers(0, 256, sum(lengths), dtype=np.uint8).tobytes()
    ref, ring = _RefEncRing(bs, extra), GR.GroupRing(bs)
    dsz, o, h = 0, 0, hashlib.sha256()
    for n in lengths:
        src = data[o:o + n]
        P_ref, d_ref, w_ref = ref.encode(src)
        hist = ring.history()
        assert hist == data[max(o - K64, 0):o]
        d = min(dsz, ring.prefix)
        assert _equivalent_dict(d, d_ref), (o, d, d_ref)
        k = min(d, 65535)
        assert hist[len(hist) - k:] == w_ref[len(w_ref) - k:]
        h.update(f"{ring.prefix}:{d}:".encode())
        dsz = d + n
        ring.append(src)
        o += n
    assert ring.slides >= 2
    _check_digest(f"enc-rule-{bs}-{extra}", h.hexdigest())


@pytest.mark.parametrize("bs,extra", ENC_CASES)
def test_encoder_group_equals_reference_ring(bs, extra):
    """The group's rule over upstream gives the bytes and (up to a dictSize beyond 64 KiB, which no block can tell)
    the state of LZ4FastChainEncoder's ring over upstream after every block: full, short and 1-byte blocks."""
    if not _have_ref():
        pytest.skip("upstream's engine is not built (oracle/_ref/); the bookkeeping test covers the rule")
    up = ER.EncUpstream()
    lengths = _enc_lengths(bs, bs + extra)
    data = _content(sum(lengths), bs + extra)
    ring, grp = ER.RingModel(up, bs, extra), GR.GroupEncoder(up, bs)
    cap = bs + bs // 255 + 16
    h = hashlib.sha256()
    try:
        o = 0
        for n in lengths:
            assert ring.topup(data[o:o + n]) == n
            r, out, _, _, after = ring.encode(cap, False)
            g = grp.encode(data[o:o + n], cap)
            assert g == (r, out), o
            assert _dict_size_ok(grp.state, after), o
            h.update(out)
            o += n
    finally:
        ring.close()
    assert grp.ring.slides >= 2
    _check_digest(f"enc-bytes-{bs}-{extra}", h.hexdigest(), record_only=True)


def _run_decoder(bs: int, extra: int, decode, ref):
    """Drives a GroupDecoder and a reference LZ4ChainDecoder model through one script; returns the digest."""
    grp = GR.GroupDecoder(bs, decode)
    h = hashlib.sha256()
    fails = 0
    for op in GR.decode_script(bs + extra, bs, 60 if bs >= K64 else 300):
        if op[0] == "inj":
            ref.inject(op[1])
            grp.inject(op[1])
            h.update(b"i")
        else:
            _, src, cap = op
            try:
                r_ref = ref.decode(src, cap)
                want = (r_ref, ref.peek(-r_ref) if r_ref else b"")
            except RuntimeError:
                want = (-1, b"")
            got = grp.decode(src, cap)
            assert got == want
            fails += got[0] < 0
            h.update(f"{got[0]}:".encode() + got[1])
        hist = grp.ring.history()
        assert ref.peek(-len(hist)) == hist
    assert fails > 0 and grp.ring.slides >= 2
    return h.hexdigest()


@pytest.mark.parametrize("bs,extra", DEC_CASES)
def test_decoder_group_equals_reference_ring(bs, extra):
    """Random Decode / Inject sequences that wrap both rings, with malformed blocks mid-stream: the group's rule
    gives LZ4ChainDecoder's results and bytes, and its history equals Peek.  Over upstream's streaming decoder
    where it is built; always over the prefix-mode restatement, whose results are pinned by a digest of
    upstream's."""
    dig = _run_decoder(bs, extra, CR.decompress_prefix, GR.RefDecoder(bs, extra, CR.decompress_prefix))
    if _have_ref():
        up = CR.Upstream()
        rm = CR.RingModel(up, bs, extra)
        try:
            assert _run_decoder(bs, extra, up.decode_prefix, rm) == dig
        finally:
            rm.close()
    _check_digest(f"dec-{bs}-{extra}", dig)


def _check_digest(key: str, value: str, record_only: bool = False) -> None:
    rec = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
    if os.environ.get("K4LZ4_RECORD_DIGESTS"):
        rec[key] = value
        with open(DIGESTS, "w") as f:
            json.dump(rec, f, indent=1, sort_keys=True)
            f.write("\n")
        return
    if not record_only or key in rec:
        assert rec.get(key) == value, key


# ---- argument errors of the k4lz4_chain_group_* exports -------------------------------------------------------

def test_group_argument_errors_without_group(native):
    """A null group or a bad create argument is E_ARG with or without a device; create leaves *out null; a valid
    create without a device is E_NODEVICE."""
    from k4os.compression.lz4_b200 import _native as N
    L = native
    a = [np.zeros(64, np.uint8) for _ in range(4)]
    p = [x.ctypes.data for x in a]
    h = C.c_void_p(12345)
    for kind, S, B in ((2, 4, 1024), (-1, 4, 1024), (0, 0, 1024), (1, -3, 1024), (0, 4, 0), (1, 4, -1)):
        h.value = 12345
        assert L.k4lz4_chain_group_create(kind, S, B, 0, C.byref(h)) == N.E_ARG and h.value is None, (kind, S, B)
    assert L.k4lz4_chain_group_create(0, 4, 1024, 0, None) == N.E_ARG
    for mem in (N.MEM_HOST, N.MEM_DEVICE, 7):
        assert L.k4lz4_chain_group_encode(None, *p[:1], *p[:1] * 7, 1, 0, mem, None) == N.E_ARG
        assert L.k4lz4_chain_group_decode(None, *p[:1], *p[:1] * 7, 1, mem, None) == N.E_ARG
        assert L.k4lz4_chain_group_inject(None, *p[:4], 1, mem, None) == N.E_ARG
        assert L.k4lz4_chain_group_reset(None, p[0], 1, mem, None) == N.E_ARG
    assert L.k4lz4_chain_group_state(None, 0, p[0]) == N.E_ARG
    assert L.k4lz4_chain_group_history(None, 0, p[0], 64) == N.E_ARG
    assert L.k4lz4_chain_group_destroy(None) == N.OK
    h.value = 12345
    rc = L.k4lz4_chain_group_create(0, 4, 1024, 0, C.byref(h))
    if has_gpu():
        assert rc == N.OK and h.value
        L.k4lz4_chain_group_destroy(h)
        assert L.k4lz4_chain_group_create(0, 4, 1024, L.k4lz4_device_count(), C.byref(h)) == N.E_ARG
    else:
        assert rc == N.E_NODEVICE and h.value is None
        with pytest.raises(N.K4Error) as e:
            from k4os.compression.lz4_b200 import ChainDecoderGroup
            ChainDecoderGroup(4, 1024)
        assert e.value.code == N.E_NODEVICE


if __name__ == "__main__":
    os.environ["K4LZ4_RECORD_DIGESTS"] = "1"
    raise SystemExit(pytest.main([__file__, "-q", "-k", "not argument"]))
