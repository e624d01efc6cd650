"""GPU tests of k4lz4_decode_chain_streams on the adversarial families of tests/stream_cases.py, and on the call's
edges that tests/test_gpu_chain_stream.py does not reach: more streams than the replay has resident warps, the
device-memory stream table's -1 contract, a failing or whole block around a host staging-piece boundary, and
LZ4ChainDecoder.DecodeBlocks across a whole block.

Every output equals upstream stepped block by block, k4lz4_decode_chain_batch stepped, and the model
(tests/chain_stream_ref.py); offset-0 streams, whose content upstream leaves unspecified, are held to the model.
Destinations are filled with 0xCD (stream_cases.FILL, a byte no family decodes to), so a match whose source pass 2
wrongly took for final reads it every time."""
import numpy as np
import pytest

from tests import chain_ref as CR
from tests import chain_stream_ref as SR
from tests import stream_cases as SC
from tests.test_gpu_chain_stream import _up, chain, run_streams, step_chain_batch, stream_of

pytestmark = pytest.mark.gpu
K4, K64 = 4096, 65536
STAGE_BYTES = 256 << 20                 # k4lz4_api.cu: bytes per host staging chunk
DS_WORK = 2048 * 12                     # device workspace per entry: K4_DS_BUDGET records of 12 bytes


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


def check_all(k4, streams, mem, zero_offset=False):
    """GPU == model, upstream stepped and the chain batch stepped (bytes with the model only where offset 0)"""
    got = run_streams(k4, streams, mem)
    model = SR.decode_streams([(h, len(h), e) for h, e in streams])
    stepped = step_chain_batch(k4, streams)
    for s, (h, e) in enumerate(streams):
        want = SR.step_reference(_up(), h, len(h), e)
        assert got[s] == model[s], f"stream {s}: model"
        assert got[s][0] == want[0] == stepped[s][0], f"stream {s}: lengths"
        if not zero_offset:
            assert got[s][1] == want[1] == stepped[s][1], f"stream {s}: bytes"
    return got


@pytest.mark.parametrize("mem", ["device", "host"])
@pytest.mark.parametrize("name", ["history", "depth", "own-intervals", "phase-a", "phase-b-runs", "periodic",
                                  "zero-offset", "budget", "mutants"])
def test_family(k4, name, mem):
    f = SC.families()[name]
    check_all(k4, f.streams, mem, f.zero_offset)


def test_more_streams_than_resident_replay_warps(k4):
    """32 x SMs + 1 000 streams of 0 .. 3 small blocks, shuffled, with whole and failing streams among them: the
    replay's warps take second streams from the ticket."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(31)
    chains = [chain("datagen", 1024, 12, 300 + c) for c in range(8)]
    whole = SC.families()["budget"].streams[-40:]
    streams = []
    for s in range(32 * sms + 1000):
        c, j, n = int(rng.integers(0, 8)), int(rng.integers(0, 8)), int(rng.integers(0, 4))
        data, blocks = chains[c]
        es = [(blocks[k], 1024, False) for k in range(j, j + n)]
        if n and s % 97 == 5:
            es[-1] = (b"\xf0", 1024, False)                   # a literal run without its length: fails
        streams.append((data[:j * 1024], es))
    for w in whole:
        streams.insert(int(rng.integers(0, len(streams))), w)
    got = run_streams(k4, streams, "device")
    for s, (h, e) in enumerate(streams):
        assert got[s] == SR.step_reference(_up(), h, len(h), e), f"stream {s}"
    assert sum(-1 in ol for ol, _ in got) >= 20


def test_device_table_contract(k4):
    """entryStart[0] > 0, entryStart[m] < n and a stream with prefixLen -1: the entries no stream holds and the
    negative stream's entries get -1, every other stream is exact and no byte outside their regions changes."""
    import torch
    from k4os.compression.lz4_b200 import batch
    fam = SC.families()
    good = [fam["phase-b-runs"].streams[0], fam["budget"].streams[3], fam["own-intervals"].streams[1],
            stream_of("datagen", K4, 6, P=4096, seed=41)]
    lost = [(b, K4, False) for b in chain("datagen", K4, 3, 42)[1]]
    # entries: 2 held by no stream | good[0] | good[1] | the negative stream | good[2] | good[3] | 3 lost at the end
    layout = [(None, lost[:2]), (0, good[0][1]), (1, good[1][1]), (-1, good[2][1]), (2, good[2][1]),
              (3, good[3][1]), (None, lost)]
    hists = {0: good[0][0], 1: good[1][0], -1: good[2][0], 2: good[2][0], 3: good[3][0]}
    srcs = [e for _, es in layout for e in es]
    lens = np.array([len(s) for s, _, _ in srcs], dtype=np.int32)
    soff = np.zeros(len(srcs), dtype=np.int64)
    soff[1:] = np.cumsum(lens[:-1])
    src = np.frombuffer(b"".join(s for s, _, _ in srcs), dtype=np.uint8).copy()
    caps = np.array([c for _, c, _ in srcs], dtype=np.int32)
    raw = np.array([r for _, _, r in srcs], dtype=np.uint8)
    held = layout[1:-1]
    es = np.cumsum([len(layout[0][1])] + [len(e) for _, e in held]).astype(np.int32)
    doff, pos, regions = [], 64, []
    for key, e in held:
        pos = (pos + len(hists[key]) + 15) // 16 * 16 + 5
        doff.append(pos)
        room = sum(c for _, c, _ in e)
        regions.append((pos, room))
        pos += room + 64
    dst = np.full(pos + 64, SC.FILL, dtype=np.uint8)
    for o, (key, _) in zip(doff, held):
        h = hists[key]
        dst[o - len(h):o] = np.frombuffer(h, dtype=np.uint8)
    before = dst.copy()
    pre = np.array([-1 if key == -1 else len(hists[key]) for key, _ in held], dtype=np.int32)
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev)
         for k, v in dict(src=src, soff=soff, lens=lens, raw=raw, caps=caps, es=es, dst=dst,
                          doff=np.array(doff, dtype=np.int64), pre=pre).items()}
    out = torch.full((len(srcs),), -7, dtype=torch.int32, device=dev)
    batch.decode_chain_streams_device(t["src"].data_ptr(), t["soff"].data_ptr(), t["lens"].data_ptr(),
                                      t["raw"].data_ptr(), t["caps"].data_ptr(), out.data_ptr(), len(srcs),
                                      t["es"].data_ptr(), t["dst"].data_ptr(), t["doff"].data_ptr(),
                                      t["pre"].data_ptr(), len(held))
    torch.cuda.synchronize()
    ol, d = out.cpu().numpy(), t["dst"].cpu().numpy()
    assert list(ol[:2]) == [-1, -1] and list(ol[es[-1]:]) == [-1] * 3, "entries no stream holds"
    mask = np.ones(len(d), dtype=bool)
    for s, ((key, e), (o, room)) in enumerate(zip(held, regions)):
        r = [int(x) for x in ol[es[s]:es[s + 1]]]
        if key == -1:
            assert r == [-1] * len(e), "a stream with a negative prefix length"
            continue
        mask[o:o + room] = False
        want = SR.step_reference(_up(), hists[key], len(hists[key]), e)
        assert (r, d[o:o + sum(x for x in r if x > 0)].tobytes()) == want, f"stream {s}"
    assert np.array_equal(d[mask], before[mask]), "a byte outside the valid streams' regions changed"


def _first_piece_end(entries, prefix: int = 0) -> int:
    """run_streams_staged's cut of one stream: the first entry of the second piece"""
    total = 0
    for e, (src, cap, raw) in enumerate(entries):
        add = len(src) + max(cap, 0) + 32 + (min(prefix, 65535) + 16 if e == 0 else 0) + DS_WORK
        if e and total + add > STAGE_BYTES:
            return e
        total += add
    raise AssertionError("one piece")


def _place(entries, make, rel: int):
    """entries with entry b + rel replaced by make(index), b the first entry of the second piece after the
    replacement (the replacement's own size moves the cut)"""
    idx = _first_piece_end(entries) + rel
    for _ in range(8):
        es = list(entries)
        es[idx] = make(idx)
        b = _first_piece_end(es)
        if b + rel == idx:
            return es, b
        idx = b + rel
    raise AssertionError("the piece boundary does not settle")


def _whole_block(data: bytes, k: int):
    """2 049 deferred 4-byte matches into block k - 1 of `data` (4 KiB blocks): over the budget"""
    seqs = [(b"", 4 + (i * 7919) % (K4 - 8), 4) for i in range(2049)]
    src, dec = CR.build_prefix_block(data[(k - 16) * K4:k * K4], seqs, b"w" * 16)
    return (src, len(dec), False)


@pytest.mark.parametrize("kind", ["fail", "whole"])
def test_host_staging_pieces(k4, kind):
    """One stream of 20 000 4 KiB blocks, cut by the host path into pieces: a failing or a whole block at the
    entry before, at and after the first piece boundary.  After a failure every later entry (later pieces
    included) is -1 and the bytes before it are exact."""
    h, entries = stream_of("datagen", K4, 20000, seed=7)
    data = chain("datagen", K4, 20000, 7)[0]
    make = (lambda i: (b"\xf0", K4, False)) if kind == "fail" else (lambda i: _whole_block(data, i))
    for rel in (-1, 0, 1):
        es, b = _place(entries, make, rel)
        got = run_streams(k4, [(h, es)], "host")
        want = SR.step_reference(_up(), h, len(h), es)
        assert got[0] == want, (kind, rel)
        if kind == "fail":
            assert got[0][0][b + rel:] == [-1] * (len(es) - b - rel) and min(got[0][0][:b + rel]) == K4
        else:
            assert min(got[0][0]) > 0


def test_chain_decoder_decode_blocks_across_a_whole_block(k4):
    """LZ4ChainDecoder.DecodeBlocks over a whole block and a later block whose records read it leaves the decoder
    as the same Decode calls do."""
    from k4os.compression.lz4_b200.encoders import LZ4ChainDecoder
    s = SC.families()["budget"].streams[3][1]             # stored, whole, reader, whole after writes, readers
    items = [e[0] for e in s]
    raw = [e[2] for e in s]
    a, b = LZ4ChainDecoder(K64, 0), LZ4ChainDecoder(K64, 0)
    want = bytearray()
    for item, r in zip(items, raw):
        if r:
            a.Inject(item)
            want += item
        else:
            n = a.Decode(item)
            want += a.Peek(-n).tobytes()
    got = b.DecodeBlocks(items, raw=raw)
    assert got == bytes(want)
    assert (a.BytesReady, a.PrefixSize) == (b.BytesReady, b.PrefixSize)
    assert np.array_equal(a._out[:a.BytesReady], b._out[:b.BytesReady])
    st = SR.Stats()
    SR.decode_streams([(b"", 0, s)], stats=st)
    assert st.whole_blocks == 2 and st.phase_a > 0 and st.runs > 0
