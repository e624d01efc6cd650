"""GPU tests of k4lz4_decode_chain_streams: whole chained streams in one call.

Every stream's lengths and bytes must equal both upstream's LZ4_decompress_safe_continue stepped block by block
(tests/chain_stream_ref.step_reference) and k4lz4_decode_chain_batch stepped block by block across the same
streams; bytes outside the streams' regions (0xCD sentinels) and the histories stay untouched."""
import functools

import numpy as np
import pytest

from tests import chain_ref as CR
from tests import chain_stream_ref as SR

pytestmark = pytest.mark.gpu
K64 = 65536


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@functools.lru_cache(maxsize=None)
def _up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return CR.Upstream()


@functools.lru_cache(maxsize=None)
def datagen(size: int, seed: int, proba: float = 0.63) -> bytes:
    import oracle
    return oracle.Port().datagen(size, proba, 0.0, seed).tobytes()


@functools.lru_cache(maxsize=None)
def chain(kind: str, block: int, nblocks: int, seed: int = 1):
    """(data, upstream's linked blocks) of one input"""
    size = block * nblocks
    if kind == "datagen":
        data = datagen(size, seed)
    elif kind == "random":
        data = np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8).tobytes()
    else:                                                     # repetitive: every block copies from the one before
        unit = np.random.default_rng(seed).integers(0, 256, 40000 + seed, dtype=np.uint8).tobytes()
        data = (unit * (size // len(unit) + 1))[:size]
    return data, _up().encode_chain(data, block)


def stream_of(kind, block, nblocks, P=0, seed=1, raw_every=0):
    """(history, entries): upstream's blocks j .. j + nblocks - 1 behind the P bytes in front of block j (the first
    block boundary at or after P: with P = 0 the whole stream); with raw_every, every raw_every-th entry stored as its plain content."""
    j = -(-P // block)
    data, blocks = chain(kind, block, nblocks + j, seed)
    hist = data[j * block - P:j * block]
    entries = []
    for k in range(j, nblocks + j):
        raw = raw_every > 0 and k % raw_every == 0
        entries.append((data[k * block:(k + 1) * block] if raw else blocks[k], block, raw))
    return hist, entries


def run_streams(k4, streams, mem: str):
    """streams: [(history, [(src, cap, raw)])] -> [(outLen list, produced bytes)]; checks the sentinels."""
    from k4os.compression.lz4_b200 import batch
    srcs = [s for _, es in streams for s, _, _ in es]
    lens = np.array([len(s) for s in srcs], dtype=np.int32)
    soff = np.zeros(len(srcs), dtype=np.int64)
    soff[1:] = np.cumsum(lens[:-1], dtype=np.int64)
    src = np.frombuffer(b"".join(srcs) or b"\0", dtype=np.uint8).copy()
    caps = np.array([c for _, es in streams for _, c, _ in es], dtype=np.int32)
    raw = np.array([r for _, es in streams for _, _, r in es], dtype=np.uint8)
    es = np.zeros(len(streams) + 1, dtype=np.int32)
    es[1:] = np.cumsum([len(e) for _, e in streams])
    doff, pos, region = [], 48, []
    for h, e in streams:
        pos = (pos + len(h) + 15) // 16 * 16 + 3
        doff.append(pos)
        room = sum(max(c, 0) for _, c, _ in e)
        region.append(room)
        pos += room + 48
    dst = np.full(pos + 48, 0xCD, dtype=np.uint8)
    for o, (h, _) in zip(doff, streams):
        dst[o - len(h):o] = np.frombuffer(h, dtype=np.uint8)
    before = dst.copy()
    pre = np.array([len(h) for h, _ in streams], dtype=np.int32)
    doff = np.array(doff, dtype=np.int64)
    if mem == "host":
        out = batch.decode_chain_streams_host(src, soff, lens, caps, es, dst, doff, pre, raw=raw)
    else:
        import torch
        dev = torch.device("cuda", 0)
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev)
             for k, v in dict(src=src, soff=soff, lens=lens, raw=raw, caps=caps, es=es, dst=dst, doff=doff,
                              pre=pre).items()}
        t_out = torch.full((len(srcs),), -7, dtype=torch.int32, device=dev)
        batch.decode_chain_streams_device(t["src"].data_ptr(), t["soff"].data_ptr(), t["lens"].data_ptr(),
                                          t["raw"].data_ptr(), t["caps"].data_ptr(), t_out.data_ptr(), len(srcs),
                                          t["es"].data_ptr(), t["dst"].data_ptr(), t["doff"].data_ptr(),
                                          t["pre"].data_ptr(), len(streams))
        torch.cuda.synchronize()
        out, dst = t_out.cpu().numpy(), t["dst"].cpu().numpy()
    res = []
    mask = np.ones(len(dst), dtype=bool)
    for s, (h, e) in enumerate(streams):
        mask[doff[s]:doff[s] + region[s]] = False
        ol = [int(x) for x in out[es[s]:es[s + 1]]]
        got = sum(x for x in ol if x > 0)
        res.append((ol, dst[doff[s]:doff[s] + got].tobytes()))
    assert np.array_equal(dst[mask], before[mask]), "a byte outside the streams' regions changed"
    return res


def step_chain_batch(k4, streams):
    """k4lz4_decode_chain_batch stepped: call k decodes block k of every stream still alive."""
    from k4os.compression.lz4_b200 import batch
    seen = [bytearray(h) for h, _ in streams]
    lens = [[] for _ in streams]
    dead = [False] * len(streams)
    for k in range(max((len(e) for _, e in streams), default=0)):
        idx = [s for s, (_, e) in enumerate(streams) if k < len(e)]
        live = [s for s in idx if not dead[s] and not streams[s][1][k][2]]
        for s in idx:
            src, cap, raw = streams[s][1][k]
            if dead[s]:
                lens[s].append(-1)
            elif raw:
                ok = len(src) <= cap
                lens[s].append(len(src) if ok else -1)
                dead[s] = not ok
                if ok:
                    seen[s] += src
        if live:
            out, data = batch.decode_chain_blocks_host([streams[s][1][k][0] for s in live],
                                                       [bytes(seen[s][-K64:]) for s in live],
                                                       [streams[s][1][k][1] for s in live])
            for s, r, d in zip(live, out, data):
                lens[s].append(int(r))
                if r < 0:
                    dead[s] = True
                else:
                    seen[s] += d
    return [(lens[s], bytes(seen[s][len(h):])) for s, (h, _) in enumerate(streams)]


def check(k4, streams, mem):
    got = run_streams(k4, streams, mem)
    stepped = step_chain_batch(k4, streams)
    for s, (h, e) in enumerate(streams):
        want = SR.step_reference(_up(), h, len(h), e)
        assert got[s][0] == want[0], f"stream {s}: lengths"
        assert got[s][1] == want[1], f"stream {s}: bytes"
        assert stepped[s][0] == want[0] and stepped[s][1] == want[1], f"stream {s}: stepped chain batch"
    return got


@pytest.mark.parametrize("mem", ["device", "host"])
@pytest.mark.parametrize("block", [4096, K64, 4 << 20])
def test_seven_streams(k4, block, mem):
    """1 and 7 streams: datagen at every prefixLen edge, stored entries interleaved, random and repetitive input
    (nothing deferred / every block copying from the one before), an empty stream."""
    nb = {4096: 40, K64: 12, 4 << 20: 3}[block]
    streams = [stream_of("datagen", block, nb, P=0, seed=2), (b"", []),
               stream_of("datagen", block, nb, P=1, seed=3, raw_every=3),
               stream_of("datagen", block, nb, P=65534, seed=4), stream_of("datagen", block, nb, P=65535, seed=5),
               stream_of("random", block, nb, P=65536, seed=9), stream_of("repetitive", block, nb, seed=10)]
    got = check(k4, streams[:1], mem)
    assert got[0][0] == [block] * nb
    got = check(k4, streams, mem)
    assert [ol for ol, _ in got][-3:] == [[block] * nb] * 3


@pytest.mark.parametrize("mem", ["device", "host"])
def test_300_streams(k4, mem):
    rng = np.random.default_rng(5)
    streams = []
    for s in range(300):
        n = int(rng.integers(0, 6))
        kind = ("datagen", "random", "repetitive")[s % 3]
        streams.append(stream_of(kind, 4096, n, P=int(rng.choice([0, 1, 4096])), seed=100 + s) if n else (b"", []))
    check(k4, streams, mem)


def test_one_stream_of_20000_blocks(k4):
    """4 KiB blocks: a block's history spans 16 blocks."""
    streams = [stream_of("datagen", 4096, 20000, seed=7)]
    got = check(k4, streams, "device")
    assert min(got[0][0]) == 4096


def test_block_over_the_deferred_budget(k4):
    """A 64 KiB block of thousands of short matches into the block before it: more deferred copies than the budget,
    so it is decoded whole in the replay."""
    rng = np.random.default_rng(8)
    data, blocks = chain("random", K64, 1, 8)
    seqs, op = [], 0
    while op < 40000:
        off = op + 1 + int(rng.integers(0, 65535 - op - 1))   # every match reads the block before
        seqs.append((bytes([int(rng.integers(0, 256))]), off, 4))
        op += 5
    blk, _ = CR.build_prefix_block(data, seqs, b"z" * 16)
    entries = [(blocks[0], K64, False), (blk, K64, False)]
    st = SR.Stats()
    SR.decode_streams([(b"", 0, entries)], stats=st)
    assert st.whole_blocks == 1
    for mem in ("device", "host"):
        got = check(k4, [(b"", entries)], mem)
        assert got[0][0] == [K64, op + 16]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_mutated_block(k4, where):
    """A chain-breaking mutant at block k: -1 from k on, exact bytes before it."""
    h, entries = stream_of("datagen", K64, 9, seed=12)
    k = {"first": 0, "middle": 4, "last": 8}[where]
    s = entries[k][0]
    for m in (b"\xf0", s[:1] + b"\xff" * 40, s + b"\x00\x01"):
        es = list(entries)
        es[k] = (m, K64, False)
        got = check(k4, [(h, es)], "device")
        ol = got[0][0]
        assert ol[:k] == [K64] * k and set(ol[k:]) == {-1}


def test_host_stream_larger_than_a_staging_chunk(k4):
    """64 blocks of 4 MiB: the host path splits the stream into pieces, each behind the last 64 KiB of the one
    before."""
    streams = [stream_of("datagen", 4 << 20, 64, seed=13)]
    got = check(k4, streams, "host")
    assert got[0][0] == [4 << 20] * 64
    assert run_streams(k4, streams, "device") == got


def test_chain_decoder_decode_blocks(k4):
    """LZ4ChainDecoder.DecodeBlocks leaves the decoder as the same Decode / Inject calls do: ring, PrefixSize,
    BytesReady, across ring wraps."""
    from k4os.compression.lz4_b200.encoders import LZ4ChainDecoder
    data, blocks = chain("datagen", K64, 12, 14)
    raw = [k % 5 == 3 for k in range(12)]
    items = [data[k * K64:(k + 1) * K64] if raw[k] else blocks[k] for k in range(12)]
    a, b = LZ4ChainDecoder(K64, 0), LZ4ChainDecoder(K64, 0)
    a.Decode(items[0])
    b.Decode(items[0])
    want = bytearray()
    for k in range(1, 12):
        if raw[k]:
            a.Inject(items[k])
            want += items[k]
        else:
            r = a.Decode(items[k])
            want += a.Peek(-r).tobytes()
    got = b.DecodeBlocks(items[1:], raw=raw[1:])
    assert got == bytes(want) == data[K64:]
    assert (a.BytesReady, a.PrefixSize) == (b.BytesReady, b.PrefixSize)
    assert np.array_equal(a._out[:a.BytesReady], b._out[:b.BytesReady])
    bad = b"\xf0"                                             # a literal run without its length
    c, d = LZ4ChainDecoder(K64, 0), LZ4ChainDecoder(K64, 0)
    with pytest.raises(RuntimeError):
        c.DecodeBlocks([blocks[0], blocks[1], blocks[2], bad, blocks[4]])
    for k in range(3):                                         # the blocks before the bad one are applied
        d.Decode(blocks[k])
    assert (c.BytesReady, c.PrefixSize) == (d.BytesReady, d.PrefixSize)
    assert np.array_equal(c._out[:c.BytesReady], d._out[:d.BytesReady])
