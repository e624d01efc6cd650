"""The facts the dictionary frame calls rest on, checked on the CPU against upstream lz4 (oracle/_ref/libk4ref.so,
which __graft_entry__.build() compiles where the reference is present):

* upstream's CDict frames are LZ4_loadDict + LZ4_compress_fast_continue per block (capacity n - 1, raw when that
  fails), so the GPU's extDict search reproduces them (frame_dict_ref.assemble);
* LZ4_attach_dictionary (the dictCtx mode upstream's CDict frames use for blocks of <= 4 KiB) gives the same bytes
  as LZ4_loadDict's extDict mode, so no dictCtx engine is needed;
* frame.py's _Frame restatement reads the dictID field as LZ4F_getFrameInfo does, and its verdict order holds on
  dictionary frames.
"""
import struct

import numpy as np
import pytest

from tests import frame_dict_ref as FD


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return FD.FrameDictUpstream()


def test_cdict_frames_are_per_block_extdict_assembly(up):
    from k4os.compression.lz4_b200.frame import _Frame
    chained, raw_first = set(), set()
    for data, dic, bs, linked, bc, cc, did in FD.grid():
        want = up.cdict_frame(data, dic, bs, linked, bc, cc, did)
        assert up.assemble(data, dic, bs, linked, bc, cc, did) == want, (len(data), len(dic), bs, linked)
        assert up.decode_frame(want, dic, len(data)) == data
        raws = _Frame(want, dictionary=True).raws
        if linked and len(raws) > 1:
            chained.add((len(dic), bs))
            if raws[0] and not all(raws[1:]):
                raw_first.add(bs)
    # the grid reaches what it is for: block 0's state handed on to the chained steps for every dictionary and block
    # size, also after a block 0 that did not fit
    assert chained == {(d, bs) for d in FD.DICT_SIZES for bs in FD.BLOCK_SIZES}
    assert raw_first == set(FD.BLOCK_SIZES)


def test_cdict_small_messages(up):
    rng = np.random.default_rng(3)
    dic = FD.dictionary(rng, 65536)
    for i in range(200):
        n = int(rng.integers(0, 5000))
        data = FD.content(rng, n, dic)
        for linked in (True, False):
            assert up.assemble(data, dic, 1 << 16, linked, False, i % 2 == 0, i) == \
                up.cdict_frame(data, dic, 1 << 16, linked, False, i % 2 == 0, i)


@pytest.mark.parametrize("reuse", [False, True])
def test_attach_dictionary_equals_load_dict(up, reuse):
    rng = np.random.default_rng(17 + reuse)
    dics = [FD.dictionary(rng, dl) for dl in (0, 1, 7, 8, 100, 4096, 65535, 65536, 69000) for _ in range(3)]
    ws = up.lib.LZ4_createStream() if reuse else None
    try:
        for i in range(10000):
            dic = dics[int(rng.integers(len(dics)))]
            dl = len(dic)
            n = int(rng.integers(1, 4097))
            src = FD.content(rng, n, dic, noise=int(i % 5 == 0))
            for cap in (n - 1, n + n // 255 + 16):
                assert up.attach_encode(src, dic, cap, ws) == up.encode(src, dic, cap), (dl, n, cap)
    finally:
        if ws is not None:
            up.lib.LZ4_freeStream(ws)


def test_restatement_reads_dict_id(up):
    from k4os.compression.lz4_b200.frame import _Frame, InvalidDataException
    rng = np.random.default_rng(5)
    dic = FD.dictionary(rng, 3000)
    for did, size in [(0, False), (1, False), (0xFFFFFFFF, True), (12345, True)]:
        data = FD.content(rng, 70000, dic)
        f = up.cdict_frame(data, dic, 1 << 16, True, False, True, did, content_size=size)
        info = up.frame_info(f)
        assert info == (did, len(data) if size else 0)
        p = _Frame(f, dictionary=True)
        assert p.dict_id == (did if did else None)
        if did:
            with pytest.raises(NotImplementedError):
                _Frame(f)
        # the ID bytes are covered by HC: flipping one is a header checksum error, for both readers
        if did:
            at = 6 + (8 if size else 0)
            g = bytearray(f)
            g[at] ^= 0x40
            assert up.frame_info(bytes(g)) is None
            with pytest.raises(InvalidDataException, match="header checksum"):
                _Frame(bytes(g), dictionary=True)


def test_restatement_verdict_order_on_dict_frames(up):
    from k4os.compression.lz4_b200.frame import _Frame, InvalidDataException
    rng = np.random.default_rng(9)
    dic = FD.dictionary(rng, 2000)
    f = up.cdict_frame(FD.content(rng, 5000, dic), dic, 1 << 16, False, True, True, 99)
    # magic before everything else
    with pytest.raises(InvalidDataException, match="magic"):
        _Frame(b"\0" + f[1:], dictionary=True)
    # version before the header checksum
    with pytest.raises(InvalidDataException, match="version"):
        _Frame(f[:4] + bytes([f[4] & 0x3F]) + f[5:], dictionary=True)
    # a header cut inside the ID field is a header checksum error (the field is read before HC)
    with pytest.raises(InvalidDataException, match="header checksum"):
        _Frame(f[:9], dictionary=True)
    # a truncated block after a good header
    with pytest.raises(InvalidDataException, match="Unexpected end"):
        _Frame(f[:-9], dictionary=True)
    # the same frame without the ID: the restatement reads it, and so does upstream
    g = up.cdict_frame(FD.content(rng, 5000, dic), dic, 1 << 16, False, True, True, 0)
    assert _Frame(g, dictionary=True).dict_id is None and up.frame_info(g)[0] == 0
    assert struct.unpack_from("<I", f, 6)[0] == 99
