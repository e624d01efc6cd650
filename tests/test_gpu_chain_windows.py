"""The chained and dictionary encoders' batched match search (chain_search_warp) on inputs built for its batches
(tests/chain_windows.py), against upstream alone: LZ4_compress_fast_continue on a planted state for
k4lz4_encode_chain_batch and _x32 (result, bytes, the whole 16 400-byte state record and the 0xCD sentinels around
every slot and record), LZ4_loadDict + LZ4_compress_fast_continue for k4lz4_encode_dict_batch, and LZ4F_compressFrame
and upstream's CDict frames for the linked frame calls.  A wrong store in the search often leaves a block's bytes
intact and changes only its state, so the families also run as linked streams, where the next block shows it."""
import numpy as np
import pytest

from tests import chain_enc_ref as CE
from tests import chain_search_ref as SR
from tests import chain_windows as CW
from tests import test_gpu_chain_encode as GE
from tests.test_gpu_enforce32 import run_x32

pytestmark = pytest.mark.gpu
SB = CE.STATE_BYTES


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def engines():
    import oracle
    from tests import dict_enc_ref as DR
    from tests import enforce32_ref as E32
    if not oracle.have_ref() or not E32.have_ref32():
        pytest.fail("oracle/_ref missing: run __graft_entry__.build() where the reference is present")
    return DR.DictUpstream(), E32.EncUpstream32()


@pytest.fixture(scope="module")
def cases(engines):
    """(family cases, tight cases, upstream's (result, bytes, state) by name)."""
    up, up32 = engines
    fam = CW.family_cases(up, up32)
    want = {c.name: SR.upstream_case(up, up32, c) for c in fam}
    tight = CW.tight_cases(fam, {k: v[1] for k, v in want.items()})
    want.update({c.name: SR.upstream_case(up, up32, c) for c in tight})
    return fam, tight, want


def _filler(up, n_items: int, seed: int):
    """Fresh and continued streams of 4 KiB datagen blocks, so that one call holds more than 4 224 items."""
    raw = GE._datagen(8192 * n_items, seed).tobytes()
    items, want = [], []
    for i in range(n_items):
        a, b = raw[8192 * i:8192 * i + 4096], raw[8192 * i + 4096:8192 * (i + 1)]
        if i % 2:
            s = GE._after_block(up, a)
            items.append((a, b, CW.bound(4096), s))
        else:
            s = CE.make_state()
            items.append((b"", b, CW.bound(4096), s))
        want.append(up.step(s, items[-1][0], b, CW.bound(4096)))
    return items, want


# ---- 1. one call of every prefix-mode case, more items than resident chain warps --------------------------------

@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("x32", [False, True])
def test_cases_in_one_call(k4, engines, cases, host, x32):
    up, _ = engines
    fam, tight, want = cases
    sel = [c for c in fam + tight if not c.ext and c.h4 == x32]
    items = [(c.before, c.src, c.cap, c.state) for c in sel]
    w = [want[c.name] for c in sel]
    fill_items, fill_want = _filler(up, 4400 - len(items), 77 + int(x32))
    if x32:
        fill_want = [engines[1].step(s, h, src, cap) for h, src, cap, s in fill_items]
    # the cases spread among the filler, so that they land on different warps and in their later rounds
    order = np.random.default_rng(5 + int(host)).permutation(len(items) + len(fill_items))
    all_items, all_want = items + fill_items, w + fill_want
    all_items = [all_items[i] for i in order]
    all_want = [all_want[i] for i in order]
    assert len(all_items) > 4224
    k4.batch.encode_stats(0, reset=True)
    got = run_x32(k4, all_items, host, x32=x32)
    GE.check(all_items, all_want, got)
    assert k4.batch.encode_stats(0, reset=True)["chain"] == sum(1 for it in all_items if it[1])
    assert sum(x[0] == 0 for x in w) == len([c for c in sel if c.family == "tight"]) > 100


# ---- 2. the families as linked streams, one call per step ---------------------------------------------------------

def _streams(fam, x32: bool):
    """Streams of 3 or 4 blocks: each a family case's source, the first behind the case's own history and state;
    every third stream fails its second block at a tight capacity and goes on."""
    sel = [c for c in fam if not c.ext and c.h4 == x32]
    out = []
    for i in range(0, len(sel) - 4, 4):
        k = 3 + (i // 4) % 2
        blocks = [sel[i + j].src for j in range(k)]
        caps = [CW.bound(len(b)) for b in blocks]
        out.append((sel[i].before, sel[i].state, blocks, caps, (i // 4) % 3 == 0))
    return out


@pytest.mark.parametrize("x32", [False, True])
def test_family_streams(k4, engines, cases, x32):
    up = engines[1] if x32 else engines[0]
    streams = _streams(cases[0], x32)
    # upstream over each stream's contiguous buffer, from a planted state
    want = []
    for hist, state, blocks, caps, tight in streams:
        st = up.lib.LZ4_createStream()
        rows = []
        try:
            buf = np.frombuffer(hist + b"".join(blocks) + bytes(16), dtype=np.uint8)
            v = up.view(st)
            s32 = state.view(np.uint32)
            np.ctypeslib.as_array(v.hashTable)[:] = s32[:4096]
            v.currentOffset, v.tableType = int(s32[4096]), 2
            v.dictSize = min(int(s32[4097]), len(hist))
            v.dictionary = buf.ctypes.data + len(hist) - v.dictSize
            at = len(hist)
            for j, b in enumerate(blocks):
                cap = caps[j]
                if tight and j == 1:                    # the first match check of the block fails
                    full = up.step(rows[-1][2], hist + blocks[0], b, caps[j])[1]
                    cap = (CW.tight_caps(full)["match"] or [len(full) - 1])[0]
                r, out = up.compress(st, buf.ctypes.data + at, len(b), cap)
                after = up.state_of(st)
                after.view(np.uint32)[4098:] = 0
                rows.append((r, out, after, cap))
                at += len(b)
        finally:
            up.lib.LZ4_freeStream(st)
        want.append(rows)
    states = [s for _, s, _, _, _ in streams]
    for j in range(4):
        idx = [i for i, s in enumerate(streams) if j < len(s[2])]
        items = [(streams[i][0] + b"".join(streams[i][2][:j]), streams[i][2][j], want[i][j][3], states[i]) for i in idx]
        got = run_x32(k4, items, host=False, x32=x32)
        GE.check(items, [want[i][j][:3] for i in idx], got)
        out, dst, do, st, sto = got
        for k, i in enumerate(idx):
            states[i] = st[sto[k]:sto[k] + SB].copy()
    assert any(want[i][1][0] == 0 for i in range(len(streams)))


# ---- 3. the dictionary encoder: extDict cases at every buffer phase -------------------------------------------------

def test_dict_cases_at_every_phase(k4, engines, cases):
    import torch
    from k4os.compression.lz4_b200 import batch
    up = engines[0]
    fam, tight, want = cases
    sel = [c for c in fam + tight if c.ext]
    dicts = sorted({c.before for c in sel}, key=len)
    # every dictionary at 16 phases in one buffer, every source at 16 phases
    d_at, parts, at = {}, [], 0
    for d in dicts:
        for ph in range(16):
            start = (at + 15) // 16 * 16 + ph
            parts.append((start, d))
            d_at[(d, ph)] = start
            at = start + len(d) + 1
    dic = np.full(at + 16, 0xA5, dtype=np.uint8)
    for start, d in parts:
        dic[start:start + len(d)] = np.frombuffer(d, dtype=np.uint8)
    # the family cases at all 16 x 16 phases, the tight ones at 16
    rows = [(c, sp, dp) for c in sel for sp in range(16) for dp in range(16)
            if c.family != "tight" or sp == dp]
    so = np.zeros(len(rows), dtype=np.int64)
    at = 0
    for k, (c, sp, _) in enumerate(rows):
        so[k] = (at + 15) // 16 * 16 + sp
        at = int(so[k]) + c.n
    src = np.zeros(at + 16, dtype=np.uint8)
    for k, (c, _, _) in enumerate(rows):
        src[so[k]:so[k] + c.n] = np.frombuffer(c.src, dtype=np.uint8)
    sl = np.array([c.n for c, _, _ in rows], dtype=np.int32)
    doff = np.array([d_at[(c.before, dp)] for c, _, dp in rows], dtype=np.int64)
    dl = np.array([len(c.before) for c, _, _ in rows], dtype=np.int32)
    caps = [c.cap for c, _, _ in rows]
    dst, do, dc = batch._slots(caps)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    g = [t(src), t(so), t(sl), t(dst), t(do), t(dc), t(dic), t(doff), t(dl),
         torch.full((len(rows),), -7, dtype=torch.int32, device="cuda")]
    before = batch.encode_stats(0)["chain"]
    batch.encode_dict_batch_device(*[x.data_ptr() for x in g], len(rows), stream=0, device=0)
    torch.cuda.synchronize()
    assert batch.encode_stats(0)["chain"] - before == len(rows)
    out, got = g[9].cpu().numpy(), g[3].cpu().numpy()
    bad = []
    for k, (c, sp, dp) in enumerate(rows):
        r, b, _ = want[c.name]
        slot = got[do[k]:do[k] + c.cap]
        # a block that does not fit may have written anything below its capacity, as upstream's engine does
        if out[k] != (r if r > 0 else -1) or (r > 0 and (slot[:r].tobytes() != b or (slot[r:] != 0xCD).any())):
            bad.append((c.name, sp, dp, int(out[k]), r))
    assert not bad, f"{len(bad)} blocks differ from upstream, first {bad[:5]}"
    assert (got[-1:] == 0xCD).all()
    # round trip of the phase-(0, 0) blocks through the dictionary decoder
    ok = [(c, want[c.name][1]) for c in sel if want[c.name][0] > 0]
    dec, dout = batch.decode_dict_batch_host([b for _, b in ok], [c.n for c, _ in ok], [c.before for c, _ in ok])
    assert list(dout) == [c.n for c, _ in ok] and dec == [c.src for c, _ in ok]
    assert sum(c.family == "tight" for c in sel) > 50 and sum(c.family == "straddle" for c in sel) >= 14


# ---- 4. the frame layer over family content ----------------------------------------------------------------------------

def _contents(fam, seed: int):
    """~200-300 KiB contents of family sources: as they come, behind a raw (incompressible) 64 KiB block 0, and
    with an incompressible 64 KiB block mid-stream."""
    rng = np.random.default_rng(seed)
    srcs = [c.src for c in fam if not c.ext and not c.h4]
    body = b"".join(srcs)
    noise = lambda: rng.integers(0, 256, 65536, dtype=np.uint8).tobytes()
    out = []
    for k in range(6):
        a = int(rng.integers(0, len(body) - 300000))
        x = body[a:a + 200000 + 20000 * k]
        if k % 3 == 1:
            x = noise() + x
        elif k % 3 == 2:
            x = x[:131072] + noise() + x[131072:]
        out.append(x)
    return out


def test_lz4f_linked_frames(k4, cases):
    from k4os.compression.lz4_b200 import LZ4F
    from tests import lz4f_ref as R
    up = R.Lz4fUpstream()
    items = _contents(cases[0], 3)
    for bc, cc in ((False, False), (True, True)):
        frames, out = LZ4F.compress_many(items, 65536, True, bc, cc, True)
        assert (out > 0).all()
        for f, x in zip(frames, items):
            assert f == up.frame(x, 65536, R.flags_of(True, bc, cc, True)), (len(x), bc, cc)


def test_cdict_linked_frames(k4, cases):
    from k4os.compression.lz4_b200 import LZ4Frame
    from tests import frame_dict_ref as FR
    up = FR.FrameDictUpstream()
    items = _contents(cases[0], 4)
    dic_cases = [c for c in cases[0] if c.ext and len(c.before) >= 8]
    dicts = [dic_cases[7 * k % len(dic_cases)].before for k in range(len(items))]
    # a dictionary that the first block refers to: block 0 of a linked CDict frame searches it
    items[0] = dicts[0][-3000:] + items[0]
    frames, out = LZ4Frame.EncodeManyWithDictionary(items, dicts, [k + 1 for k in range(len(items))], 65536, True)
    assert (out > 0).all()
    for k, (f, x, d) in enumerate(zip(frames, items, dicts)):
        assert f == up.cdict_frame(x, d, 65536, True, False, False, k + 1), (k, len(x), len(d))
