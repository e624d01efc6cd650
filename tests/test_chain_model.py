"""Chained blocks without a GPU: the prefix-mode restatement (tests/chain_ref.py) against upstream's
LZ4_decompress_safe_continue, the routing model with a history, the new C export's argument checks and
LZ4ChainDecoder's ring bookkeeping against upstream's LZ4_streamDecode_t.

Where upstream's engine is not built, the restatement is compared with a digest of upstream's results
recorded in tests/golden/chain_digests.json (regenerate with ``python -m tests.test_chain_model``)."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import chain_ref as CR
from tests import inputs
from tests import lz4_blocks as LB
from tests.conftest import ROOT, has_gpu

PREFIXES = [0, 1, 4, 12, 15, 16, 65534, 65535, 65536, 70000]
DIGESTS = os.path.join(ROOT, "tests", "golden", "chain_digests.json")


def _have_ref() -> bool:
    import oracle
    return oracle.have_ref()


def _history(P: int) -> bytes:
    return np.random.default_rng(P + 1).integers(0, 256, P, dtype=np.uint8).tobytes()


def prefix_cases():
    """(name, src, cap, history): valid blocks whose matches reach into histories of every length in PREFIXES,
    the two offset boundaries, and byte mutations of them."""
    rng = np.random.default_rng(7)
    out = []
    for P in PREFIXES:
        h = _history(P)
        Pe = min(P, 65535)
        body = rng.integers(0, 256, 40, dtype=np.uint8).tobytes()
        for off in sorted({1, 4, 8, 15, 16, 17, Pe, Pe + 1, 65535} - {0}):
            if off > 65535:
                continue
            for ml in (4, 12, 19, 40):
                lits = body[:3]
                if off > Pe + 3:                             # beyond the history: the block is built by hand
                    s, _ = LB.build_block([(lits, 3, 4)], body[:10])
                    s = bytearray(s)
                    s[4:6] = bytes([off & 0xFF, off >> 8])   # first sequence's offset
                    out.append((f"P{P}-off{off}-ml{ml}-beyond", bytes(s), 64, h))
                    continue
                s, d = CR.build_prefix_block(h, [(lits, off, ml), (body[:5], 7, 6)], body[:12])
                for cap in (len(d), len(d) + 1, len(d) - 1, len(d) + 40):
                    out.append((f"P{P}-off{off}-ml{ml}-cap{cap}", s, cap, h))
        # datagen through upstream's chained encoder cannot run without upstream: mutations of a mid-size block
        seqs = [(body[:2], min(Pe, 1000) or 1, 24)] if Pe else [(body[:8], 4, 24)]
        seqs += [(body[:int(rng.integers(0, 20))], int(rng.integers(1, 30)), int(rng.integers(4, 40))) for _ in range(30)]
        s, d = CR.build_prefix_block(h, seqs, body[:16])
        for k in range(24):
            m = bytearray(s)
            m[int(rng.integers(0, len(m)))] ^= 1 << int(rng.integers(0, 8))
            out.append((f"P{P}-mut{k}", bytes(m), len(d), h))
    return out


def _comparable(src: bytes, res):
    """(r, bytes), bytes dropped where an offset-0 match leaves the content unspecified"""
    r, b = res
    return (r, b"" if r <= 0 or inputs.uses_zero_offset(src) else b)


def _digest(cases, results) -> str:
    h = hashlib.sha256()
    for (name, s, _, _), res in zip(cases, results):
        r, b = _comparable(s, res)
        h.update(f"{name}:{r}:".encode() + b)
    return h.hexdigest()


def test_restatement_matches_builder():
    for P in PREFIXES:
        h = _history(P)
        Pe = min(P, 65535)
        s, d = CR.build_prefix_block(h, [(b"abc", min(Pe + 3, 65535) if Pe else 2, 30), (b"", 9, 5)], b"0123456789ab")
        assert CR.decompress_prefix(s, len(d), h) == (len(d), d)


def test_restatement_against_upstream():
    """Return codes and bytes of the restatement equal upstream's prefix mode on every case, or the recorded
    digest of upstream's results."""
    cases = prefix_cases()
    mine = [CR.decompress_prefix(s, c, h) for _, s, c, h in cases]
    assert any(r < 0 for r, _ in mine) and any(r > 0 for r, _ in mine)
    if _have_ref():
        up = CR.Upstream()
        for (n, s, c, h), got in zip(cases, mine):
            assert _comparable(s, got) == _comparable(s, up.decode_prefix(s, c, h)), n
        # upstream's streaming call gives the same as its usingDict dispatch (what the oracle uses)
        rm = CR.RingModel(up, 65536)
        try:
            h = _history(300)
            rm.inject(h)
            s, d = CR.build_prefix_block(h, [(b"xy", 290, 20)], b"0123456789ab")
            assert rm.decode(s, 4096) == len(d) and rm.peek(-len(d)) == d
        finally:
            rm.close()
    else:
        rec = json.load(open(DIGESTS))
        assert rec["prefix_cases"] == len(cases)
        assert _digest(cases, mine) == rec["prefix_digest"]


def test_routing_model_with_history():
    """The model's offset test moves by P: offset P is on the tile path, P + 1 goes to the exact engine."""
    for P in (1, 16, 1000, 65534):
        h = _history(P)
        body = bytes(range(40))
        L = min(5, 65535 - P)
        s, d = CR.build_prefix_block(h, [(body[:L], P + L, 8)], body[:16])
        assert CR.tile_route_p(s, len(d), P) == "tile"
        assert CR.tile_route_p(s, len(d), P - 1) == "generic"
        assert CR.tile_route_p(s, len(d), 0) == "generic" == LB.expected_engine(s, len(d))
    s, d = CR.build_prefix_block(_history(65535), [(b"a", 65535, 8)], bytes(16))
    assert CR.tile_route_p(s, len(d), 65535) == CR.tile_route_p(s, len(d), 70000) == "tile"


def test_chain_export_arguments(native):
    """k4lz4_decode_chain_batch: a negative prefix is an argument error (checked before anything else with
    host memory); without a device a valid call fails with E_NODEVICE -- there is no CPU fallback."""
    from k4os.compression.lz4_b200 import _native as N
    from k4os.compression.lz4_b200 import batch as B
    src = np.frombuffer(b"\x10a", dtype=np.uint8).copy()
    dst = np.zeros(64, dtype=np.uint8)
    args = (src, [0], [2], dst, [32], [16])
    with pytest.raises(N.K4Error) as e:
        B.decode_chain_batch_host(*args, [-1])
    assert e.value.code == N.E_ARG
    rc = native.k4lz4_decode_chain_batch(None, None, None, None, None, None, None, None, 1, N.MEM_HOST, None, 0)
    assert rc == N.E_ARG
    assert native.k4lz4_decode_chain_batch(None, None, None, None, None, None, None, None, 0, 7, None, 0) == N.E_ARG
    if not has_gpu():
        with pytest.raises(N.K4Error) as e:
            B.decode_chain_batch_host(*args, [4])
        assert e.value.code == N.E_NODEVICE


def _inject_script(rng, n_ops: int, block: int):
    ops = []
    for _ in range(n_ops):
        k = int(rng.integers(0, 5))
        size = [1, 17, 4096, 65535, 65536][k] if rng.random() < 0.3 else int(rng.integers(1, max(block, 65536) + 1))
        ops.append(rng.integers(0, 256, size, dtype=np.uint8).tobytes())
    return ops


@pytest.mark.parametrize("block,extra", [(1024, 0), (65536, 0), (65536, 2), (300000, 1)])
def test_chain_decoder_inject_bookkeeping(block, extra):
    """Inject's three paths (LZ4ChainDecoder.cs:64-93), Peek and Drain: the write position, the prefix size and
    the ring's bytes equal the reference's class run over upstream's LZ4_streamDecode_t."""
    from k4os.compression.lz4_b200 import LZ4ChainDecoder, LZ4Decoder, LZ4BlockDecoder
    if not _have_ref():
        pytest.skip("upstream's LZ4_streamDecode_t is needed for the reference bookkeeping")
    assert isinstance(LZ4Decoder.Create(False, block), LZ4BlockDecoder)
    dec = LZ4Decoder.Create(True, block, extra)
    assert isinstance(dec, LZ4ChainDecoder)
    rm = CR.RingModel(CR.Upstream(), block, extra)
    try:
        assert dec.BlockSize == rm.block and dec._out_len == rm.out_len
        rng = np.random.default_rng(block + extra)
        for src in _inject_script(rng, 60, dec.BlockSize):
            if len(src) > max(dec.BlockSize, 65536):
                with pytest.raises(RuntimeError):
                    dec.Inject(src)
                continue
            assert dec.Inject(src) == rm.inject(src)
            assert dec.BytesReady == rm.index and dec.PrefixSize == rm.prefix_size
            assert np.array_equal(dec._out[:dec.BytesReady], rm.buf[:rm.index])
            k = int(rng.integers(0, dec.BytesReady + 1))
            assert dec.Peek(-k).tobytes() == rm.peek(-k)
            t = bytearray(k)
            dec.Drain(t, -k, k)
            assert bytes(t) == rm.peek(-k)
        with pytest.raises(RuntimeError):
            dec.Peek(-dec.BytesReady - 1)
        with pytest.raises(RuntimeError):
            dec.Drain(bytearray(8), -4, 8)
        assert dec.Inject(b"") == 0
        dec.Dispose()
        with pytest.raises(RuntimeError):
            dec.Inject(b"x")
    finally:
        rm.close()


def _record():
    cases = prefix_cases()
    up = CR.Upstream()
    res = [up.decode_prefix(s, c, h) for _, s, c, h in cases]
    rec = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
    rec.update({"prefix_cases": len(cases), "prefix_digest": _digest(cases, res)})
    with open(DIGESTS, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    _record()
