"""GPU parity tests: the CUDA path, called through the C ABI, against the oracle.

Bit-exact for everything (integer/byte work): identical compressed bytes and return codes
for Encode at L00_FAST, identical bytes and return codes for Decode (well-formed and
malformed), identical pickles.  Mirrors the reference's BlockRoundtripTests / SpanTests /
PicklingTests on the accelerated path."""
import json
import os
import zlib

import numpy as np
import pytest

from tests import inputs

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def chk():
    import oracle
    return oracle.best()


def test_loaded_library_is_in_tree(k4):
    from k4os.compression.lz4_b200 import _native
    assert os.path.dirname(_native.SO_PATH).endswith(os.path.join("k4os", "compression", "lz4_b200"))


def test_issue64_golden_decode_gpu(k4):
    comp = open(os.path.join(G, "issue64_block0.lz4"), "rb").read()
    expect = open(os.path.join(G, "issue64_block0.bin"), "rb").read()
    out = bytearray(65536)
    assert k4.LZ4Codec.Decode(comp, out) == 65536 and bytes(out) == expect
    big = bytearray(b"\xCD" * 131072)
    assert k4.LZ4Codec.Decode(comp, big) == 65536
    assert bytes(big[:65536]) == expect and bytes(big[65536:]) == b"\xCD" * 65536   # untouched tail
    assert k4.LZ4Codec.Decode(comp, bytearray(65535)) == -1


def test_golden_encode_rows_gpu(k4):
    """Every committed known-answer row, as one batch per capacity class."""
    rows = json.load(open(os.path.join(G, "encode_rows.json")))["rows"]
    datas = [inputs.gen(r["kind"], r["size"], r["seed"]) for r in rows]
    enc, lens = k4.batch.encode_batch_host(datas)
    for r, c, n in zip(rows, enc, lens):
        assert n == r["len"], (r["kind"], r["size"], n, r["len"])
        assert zlib.adler32(c) & 0xFFFFFFFF == r["adler32"], (r["kind"], r["size"])
    # limited-output capacities: same return codes as the reference engine
    lim_data, lim_caps, lim_expect = [], [], []
    for r, d in zip(rows, datas):
        for cap, e in r["limited"]:
            lim_data.append(d); lim_caps.append(cap); lim_expect.append(e)
    _, got = k4.batch.encode_batch_host(lim_data, lim_caps)
    assert got.tolist() == lim_expect
    # decode them back, exact and oversized capacity
    dec, dl = k4.batch.decode_batch_host(enc, [len(d) for d in datas])
    assert dl.tolist() == [len(d) for d in datas] and dec == datas
    dec2, dl2 = k4.batch.decode_batch_host(enc, [len(d) + 77 for d in datas])
    assert dl2.tolist() == [len(d) for d in datas] and dec2 == datas


def test_encode_matches_oracle_on_corpus(k4, chk):
    items = list(inputs.corpus(sizes=inputs.THRESHOLD_SIZES + inputs.BIG_SIZES))
    datas = [d for _, d in items]
    enc, lens = k4.batch.encode_batch_host(datas)
    for (name, d), c, n in zip(items, enc, lens):
        r, ref = chk.encode(d)
        assert (int(n), c) == (r, ref), name


def test_encode_never_writes_past_returned_length(k4):
    """PartialDecompressionTests.cs:33-35 / SpanTests.cs:36-37: 0xCD sentinels stay intact."""
    d = inputs.gen("text2", 20000, 5)
    tgt = bytearray(b"\xCD" * 30000)
    n = k4.LZ4Codec.Encode(d, 0, len(d), tgt, 100, 25000)
    assert n > 0 and bytes(tgt[:100]) == b"\xCD" * 100 and bytes(tgt[100 + n:]) == b"\xCD" * (30000 - 100 - n)


def test_decode_malformed_matches_oracle(k4):
    import oracle
    port = oracle.Port()     # the restatement of LL64.dec.cs is the authority for malformed input
    rng = np.random.default_rng(11)
    streams, caps = [], []
    for it in range(4000):
        n = int(rng.choice([20, 50, 100, 300, 1000, 5000, 70000]))
        kind = ["text2", "lowent", "runs", "random", "lorem"][it % 5]
        c = inputs.mutate(port.encode(inputs.gen(kind, n, it))[1], rng)
        streams.append(c)
        caps.append(int(rng.choice([n, n, n + 5, n - 1, 2 * n, n + 64, 1])))
    dec, got = k4.batch.decode_batch_host(streams, caps)
    for i, (c, cap) in enumerate(zip(streams, caps)):
        r, ref = port.decode(c, cap)
        assert int(got[i]) == r, (i, cap, int(got[i]), r)
        if r > 0 and not inputs.uses_zero_offset(c):      # offset-0 content is unspecified
            assert dec[i] == ref, i


def test_codec_edge_semantics_gpu(k4):
    C = k4.LZ4Codec
    assert C.Encode(b"", bytearray(10)) == 0 and C.Decode(b"", bytearray(10)) == 0
    assert C.Decode(b"\x00", bytearray(10)) == -1
    assert C.Encode(b"abc", bytearray(1)) == -1
    with pytest.raises(k4.DelegateToManagedEngine):
        C.Encode(b"a" * 100, bytearray(200), k4.LZ4Level.L09_HC)
    # QuickFox (BlockRoundtripTests.cs:44-61): decode into a 2x buffer returns the true size
    t = b"The quick brown fox jumps over the lazy dog"
    e = bytearray(C.MaximumOutputSize(len(t)))
    n = C.Encode(t, 0, len(t), e, 0, len(e))
    d = bytearray(2 * len(t))
    assert C.Decode(e, 0, n, d, 0, len(d)) == len(t) and bytes(d[:len(t)]) == t


def test_border_line_compression_gpu(k4):
    for kind in ("random", "text2", "synth525"):
        d = inputs.gen(kind, 65536, 11)
        tgt = bytearray(k4.LZ4Codec.MaximumOutputSize(len(d)))
        req = k4.LZ4Codec.Encode(d, tgt)
        tgt2 = bytearray(req)
        assert k4.LZ4Codec.Encode(d, tgt2) == req and tgt2 == tgt[:req]


def test_pickler_matches_oracle(k4):
    import oracle
    port = oracle.Port()
    rng = np.random.default_rng(3)
    msgs = [b"x", inputs.gen("random", 300, 1), b"a" * 200, b"a" * 5000, b"a" * 100000]
    for i in range(300):
        n = int(rng.integers(1, 4097)) if i % 3 else int(rng.choice([255, 256, 257, 1023, 1024, 1025, 4096]))
        msgs.append(inputs.gen(["text2", "synth435", "lorem", "random", "lowent"][i % 5], n, i))
    pk, lens = k4.batch.pickle_batch_host(msgs)
    for m, p in zip(msgs, pk):
        assert p == port.pickle(m), len(m)
    sizes = k4.batch.unpickled_size_batch_host(pk)
    assert sizes.tolist() == [len(m) for m in msgs]
    un, ul = k4.batch.unpickle_batch_host(pk)
    assert un == msgs and ul.tolist() == [len(m) for m in msgs]
    # single-message mirror + corruption -> InvalidDataException (PicklingTests.cs:149-172)
    P = k4.LZ4Pickler
    assert P.Pickle(b"") == b"" and P.Unpickle(b"") == b""
    good = P.Pickle(b"a" * 200)
    assert P.Unpickle(good) == b"a" * 200 and P.UnpickledSize(good) == 200
    for bad in (bytes([good[0] | 1]) + good[1:], good[:-1], b"\xC0\x01"):
        with pytest.raises(k4.InvalidDataException):
            P.Unpickle(bad)


def test_device_path_batch_roundtrip_and_host_generator(k4):
    """cfg-2/3 shape at reduced count: synth on device == synth on host; encode on device ==
    oracle; decode(encode(x)) == x; property: checksum over all blocks."""
    import torch
    import oracle
    chk = oracle.best()
    B = k4.batch
    nb, bs = 512, 65536
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    raw = torch.empty(nb * bs, dtype=torch.uint8, device=dev)
    B.synth_device(raw.data_ptr(), nb, bs, 435, 77, 5, st)
    host = B.synth_host(nb, bs, 435, 77, 5)
    assert np.array_equal(raw.cpu().numpy(), host)
    bound = k4.LZ4Codec.MaximumOutputSize(bs)
    idx = torch.arange(nb, dtype=torch.int64, device=dev)
    roff, coff = idx * bs, idx * bound
    rlen = torch.full((nb,), bs, dtype=torch.int32, device=dev)
    ccap = torch.full((nb,), bound, dtype=torch.int32, device=dev)
    comp = torch.full((nb * bound,), 0xCD, dtype=torch.uint8, device=dev)
    clen = torch.zeros(nb, dtype=torch.int32, device=dev)
    B.encode_batch_device(raw.data_ptr(), roff.data_ptr(), rlen.data_ptr(), comp.data_ptr(),
                          coff.data_ptr(), ccap.data_ptr(), clen.data_ptr(), nb, 0, st)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device=dev)
    olen = torch.zeros(nb, dtype=torch.int32, device=dev)
    B.decode_batch_device(comp.data_ptr(), coff.data_ptr(), clen.data_ptr(), out.data_ptr(),
                          roff.data_ptr(), rlen.data_ptr(), olen.data_ptr(), nb, st)
    torch.cuda.synchronize()
    assert torch.equal(out, raw) and bool((olen == bs).all())
    c, l = comp.cpu().numpy(), clen.cpu().numpy()
    for i in range(nb):                                      # every block, not a sample
        r, ref = chk.encode(host[i * bs:(i + 1) * bs])
        assert r == int(l[i]) and c[i * bound:i * bound + r].tobytes() == ref
        assert (c[i * bound + r:(i + 1) * bound] == 0xCD).all()      # slot tail untouched
    # tight packing through copy_blocks, then decode from unaligned starts
    poff = torch.cumsum(clen.to(torch.int64), 0) - clen.to(torch.int64)
    packed = torch.empty(int(clen.sum()) + 64, dtype=torch.uint8, device=dev)
    B.copy_blocks_device(comp.data_ptr(), coff.data_ptr(), packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), nb, st)
    out.zero_()
    B.decode_batch_device(packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), out.data_ptr(),
                          roff.data_ptr(), rlen.data_ptr(), olen.data_ptr(), nb, st)
    torch.cuda.synchronize()
    assert torch.equal(out, raw) and bool((olen == bs).all())


def test_full_size_roundtrip_property(k4):
    """BASELINE configs[1]/[2] at FULL size (65 536 x 64 KiB = 4 GiB): size-independent
    properties -- decode(encode(x)) == x for every block, every length == 64 KiB, and the
    compressed size total lands on the expected ratio."""
    import torch
    B = k4.batch
    nb, bs = 65536, 65536
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    raw = torch.empty(nb * bs, dtype=torch.uint8, device=dev)
    B.synth_device(raw.data_ptr(), nb, bs, 525, 1234, 0, st)
    bound = k4.LZ4Codec.MaximumOutputSize(bs)
    idx = torch.arange(nb, dtype=torch.int64, device=dev)
    roff, coff = idx * bs, idx * bound
    rlen = torch.full((nb,), bs, dtype=torch.int32, device=dev)
    ccap = torch.full((nb,), bound, dtype=torch.int32, device=dev)
    comp = torch.empty(nb * bound, dtype=torch.uint8, device=dev)
    clen = torch.zeros(nb, dtype=torch.int32, device=dev)
    B.encode_batch_device(raw.data_ptr(), roff.data_ptr(), rlen.data_ptr(), comp.data_ptr(),
                          coff.data_ptr(), ccap.data_ptr(), clen.data_ptr(), nb, 0, st)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device=dev)
    olen = torch.zeros(nb, dtype=torch.int32, device=dev)
    B.decode_batch_device(comp.data_ptr(), coff.data_ptr(), clen.data_ptr(), out.data_ptr(),
                          roff.data_ptr(), rlen.data_ptr(), olen.data_ptr(), nb, st)
    torch.cuda.synchronize()
    assert bool((olen == bs).all())
    assert torch.equal(out, raw)
    ratio = float(clen.sum()) / (nb * bs)
    assert 0.47 < ratio < 0.53, ratio


def test_host_path_all_devices_split_and_scattered_layout(k4, chk):
    """K4LZ4_ALL_DEVICES (NCCL-free contiguous split over every visible GPU; one device here is the
    degenerate case) and a scattered, gap-filled layout that forces the packed staging path: results
    identical to the single-device contiguous call, sentinels between slots untouched."""
    from k4os.compression.lz4_b200 import _native as N
    blocks = [inputs.gen(kind, n, i) for i, (kind, n) in enumerate(
        [("text2", 70000), ("random", 300), ("lorem", 65536), ("synth525", 65536), ("lowent", 4097),
         ("runs", 20000), ("repeat", 65536), ("text2", 13), ("text2", 12), ("synth435", 131072)] * 3)]
    ref_enc, ref_len = k4.batch.encode_batch_host(blocks)
    for i in (0, 3, 9):
        assert (int(ref_len[i]), ref_enc[i]) == chk.encode(blocks[i])
    # scattered layout: 4 KiB gaps between source blocks and between destination slots
    gap = 4096
    src_len = np.array([len(b) for b in blocks], dtype=np.int32)
    src_off = np.cumsum(np.concatenate([[gap], src_len[:-1].astype(np.int64) + gap])).astype(np.int64)
    src = np.full(int(src_off[-1] + src_len[-1] + gap), 0xEE, dtype=np.uint8)
    for o, b in zip(src_off, blocks):
        src[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    cap = np.array([k4.LZ4Codec.MaximumOutputSize(len(b)) for b in blocks], dtype=np.int32)
    dst_off = np.cumsum(np.concatenate([[gap], cap[:-1].astype(np.int64) + 64 * gap])).astype(np.int64)
    dst = np.full(int(dst_off[-1] + cap[-1] + gap), 0xCD, dtype=np.uint8)
    out = k4.batch.encode_batch_flat_host(src, src_off, src_len, dst, dst_off, cap, device=N.ALL_DEVICES)
    assert out.tolist() == ref_len.tolist()
    for i, (o, n) in enumerate(zip(dst_off, out)):
        assert dst[o:o + n].tobytes() == ref_enc[i]
        assert (dst[o + n:o + cap[i]] == 0xCD).all()
    # decode the scattered compressed slots back into exact-size slots (direct D2H path) and into
    # oversized slots (staging + scatter path)
    for extra in (0, 100):
        dcap = (src_len + extra).astype(np.int32)
        doff = np.cumsum(np.concatenate([[0], dcap[:-1].astype(np.int64)])).astype(np.int64)
        back = np.full(int(dcap.sum()) + 1, 0xCD, dtype=np.uint8)
        got = k4.batch.decode_batch_flat_host(dst, dst_off, out, back, doff, dcap, device=N.ALL_DEVICES)
        assert got.tolist() == src_len.tolist()
        for i, b in enumerate(blocks):
            assert back[doff[i]:doff[i] + len(b)].tobytes() == b
            assert (back[doff[i] + len(b):doff[i] + dcap[i]] == 0xCD).all()


def test_pickler_batch_at_scale_property(k4):
    """BASELINE configs[3] shape at 131 072 messages (256 B - 4 KiB mixed): unpickle(pickle(x)) == x,
    sizes agree, header bytes well-formed; 64 messages compared byte for byte with the oracle."""
    import torch
    import oracle
    port = oracle.Port()
    B = k4.batch
    n = 1 << 17
    rng = np.random.default_rng(42)
    sizes = np.where(rng.random(n) < 0.5, rng.choice([256, 512, 1024, 2048, 4096], n),
                     rng.integers(256, 4097, n)).astype(np.int32)
    off = np.zeros(n, dtype=np.int64); off[1:] = np.cumsum(sizes[:-1], dtype=np.int64)
    total = int(sizes.sum())
    dev = torch.device("cuda", 0); st = torch.cuda.current_stream().cuda_stream
    raw = torch.empty(((total + 65535) // 65536) * 65536, dtype=torch.uint8, device=dev)
    B.synth_device(raw.data_ptr(), raw.numel() // 65536, 65536, 435, 42, 0, st)
    d_off, d_len = torch.from_numpy(off).to(dev), torch.from_numpy(sizes).to(dev)
    poff = np.zeros(n, dtype=np.int64); poff[1:] = np.cumsum(sizes[:-1].astype(np.int64) + 1)
    d_poff = torch.from_numpy(poff).to(dev)
    pk = torch.full((int(sizes.sum()) + n + 16,), 0xCD, dtype=torch.uint8, device=dev)
    plen = torch.zeros(n, dtype=torch.int32, device=dev)
    B.pickle_batch_device(raw.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), pk.data_ptr(), d_poff.data_ptr(),
                          plen.data_ptr(), n, 0, st)
    usz = torch.zeros(n, dtype=torch.int32, device=dev)
    B.unpickled_size_batch_device(pk.data_ptr(), d_poff.data_ptr(), plen.data_ptr(), usz.data_ptr(), n, st)
    out = torch.zeros(total + 16, dtype=torch.uint8, device=dev)
    olen = torch.zeros(n, dtype=torch.int32, device=dev)
    B.unpickle_batch_device(pk.data_ptr(), d_poff.data_ptr(), plen.data_ptr(), out.data_ptr(), d_off.data_ptr(),
                            d_len.data_ptr(), olen.data_ptr(), n, st)
    torch.cuda.synchronize()
    assert bool((usz == d_len).all()) and bool((olen == d_len).all())
    assert torch.equal(out[:total], raw[:total])
    assert bool((plen <= d_len + 1).all()) and bool((plen > 0).all())
    h_raw, h_pk, h_pl = raw[:int(off[64])].cpu().numpy(), pk[:int(poff[64])].cpu().numpy(), plen[:64].cpu().numpy()
    for i in range(64):
        assert h_pk[poff[i]:poff[i] + h_pl[i]].tobytes() == port.pickle(h_raw[off[i]:off[i] + sizes[i]].tobytes()), i


def test_datagen_blocks_encode_and_decode_gpu(k4, chk):
    """The workload the survey names (RDG_genBuffer 0.63 / 0.55): every block encoded by the GPU is
    byte-identical to the reference engine's output, decodes back, and stays on the tile path."""
    import oracle
    port = oracle.Port()
    bs, nb = 65536, 192
    for mp in (0.63, 0.55):
        raw = port.datagen(nb * bs, mp, 0.0, 1234)
        blocks = [raw[i * bs:(i + 1) * bs].tobytes() for i in range(nb)]
        enc, lens = k4.batch.encode_batch_host(blocks)
        for i, b in enumerate(blocks):
            assert (int(lens[i]), enc[i]) == chk.encode(b), (mp, i)
        k4.batch.decode_stats(0, reset=True)
        dec, dl = k4.batch.decode_batch_host(enc, [bs] * nb)
        st = k4.batch.decode_stats(0, reset=True)
        assert dec == blocks and dl.tolist() == [bs] * nb
        assert st["tile"] + st["tile_big"] == nb and st["generic"] == 0, st   # clean data never needs the exact fallback


def test_encode_many_blocks_through_both_kernels_and_chunks(k4, chk):
    """More blocks than the shared-memory-table kernel takes in one round: the global-table kernel runs
    beside it and the host path cuts the batch into several chunks (graded sizes).  Every block, whichever
    warp kind encoded it, must be the reference's bytes -- including a few blocks of >= 65 547 bytes (u32
    table in the global workspace), empty blocks and limited-output failures."""
    import oracle
    port = oracle.Port()
    rng = np.random.default_rng(77)
    n = 9000
    raw = port.datagen(40 << 20, 0.55, 0.0, 99)
    sizes = rng.integers(0, 8192, n)
    sizes[rng.integers(0, n, 40)] = 0
    for k, big in zip(rng.integers(0, n, 6), (65546, 65547, 70000, 131072, 65600, 90000)):
        sizes[k] = big
    off = np.concatenate([[0], np.cumsum(sizes)[:-1]]) % ((40 << 20) - 140000)
    blocks = [raw[o:o + z].tobytes() for o, z in zip(off, sizes)]
    caps = [k4.LZ4Codec.MaximumOutputSize(len(b)) for b in blocks]
    tight = rng.integers(0, n, 200)
    for k in tight:
        caps[k] = max(0, len(blocks[k]) // 3)                       # forces limitedOutput paths, mostly failures
    enc, lens = k4.batch.encode_batch_host(blocks, caps)
    for i, b in enumerate(blocks):
        r, c = chk.encode(b, caps[i])
        assert int(lens[i]) == (r if r > 0 else (0 if len(b) == 0 else -1)), (i, len(b), caps[i], int(lens[i]), r)
        if r > 0:
            assert enc[i] == c, (i, len(b))


def test_issue64_block0_reencoded_by_gpu(k4, chk):
    expect = open(os.path.join(G, "issue64_block0.bin"), "rb").read()
    enc, lens = k4.batch.encode_batch_host([expect])
    assert (int(lens[0]), enc[0]) == chk.encode(expect)
    out = bytearray(65536)
    assert k4.LZ4Codec.Decode(enc[0], out) == 65536 and bytes(out) == expect


def test_tile_path_with_oversized_capacity(k4):
    """dstCap > 64 KiB while the decoded size is <= 64 KiB must stay on the tile path and leave the
    slack untouched (BlockRoundtripTests.cs:44-61 decodes into a 2x buffer)."""
    import oracle
    port = oracle.Port()
    datas = [inputs.gen(k, n, 3) for k in ("text2", "synth525", "lorem", "runs") for n in (65536, 40000, 1000)]
    enc = [port.encode(d)[1] for d in datas]
    k4.batch.decode_stats(0, reset=True)
    caps = [200000, 65537, 131072] * 4
    dec, dl = k4.batch.decode_batch_host(enc, caps)
    st = k4.batch.decode_stats(0, reset=True)
    assert dec == datas and dl.tolist() == [len(d) for d in datas]
    assert st["tile"] + st["tile_big"] == len(datas), st
    big = bytearray(b"\xCD" * 200000)
    assert k4.LZ4Codec.Decode(enc[0], big) == 65536 and bytes(big[65536:]) == b"\xCD" * (200000 - 65536)


def test_decode_paths_cover_every_engine(k4):
    """Incompressible blocks (compressed size > 65535 / > the small stage), a block of more than
    16384 sequences and a multi-megabyte length-byte run all take their designated engine and agree
    with the oracle."""
    import oracle
    port = oracle.Port()
    rnd = inputs.gen("random", 65536, 1)                                   # -> 65 794 compressed bytes: generic
    mid = inputs.gen("random", 45000, 2) + inputs.gen("repeat", 20536, 7)  # ~45 KB compressed: big stage
    streams = [port.encode(rnd)[1], port.encode(mid)[1]]
    caps = [65536, 65536]
    # 5 MB of 0xFF length bytes (ADVICE round 1: 32-bit length overflow): must be rejected, not crash
    streams.append(b"\xF0" + b"\xFF" * (5 << 20) + b"\x00")
    caps.append(65536)
    streams.append(b"\x0F" + b"\x01\x00" + b"\xFF" * (9 << 20) + b"\x00" + b"\x50abcde")
    caps.append(65536)
    k4.batch.decode_stats(0, reset=True)
    dec, dl = k4.batch.decode_batch_host(streams, caps)
    st = k4.batch.decode_stats(0, reset=True)
    for i, (c, cap) in enumerate(zip(streams, caps)):
        r, ref = port.decode(c, cap)
        assert int(dl[i]) == r, (i, int(dl[i]), r)
        if r > 0:
            assert dec[i] == ref
    assert st["generic"] >= 3 and st["tile_big"] == 1, st


def test_dictionary_decode_gpu(k4):
    """LZ4Codec.Decode(source, target, dictionary) (LZ4Codec.cs:144-157): the reference's second
    golden vector, then mutated streams against the restatement of LL64.dec.cs:338-378."""
    import oracle
    port = oracle.Port()
    comp = open(os.path.join(G, "issue64_block1.lz4"), "rb").read()
    expect = open(os.path.join(G, "issue64_block1.bin"), "rb").read()
    dic = open(os.path.join(G, "issue64_block0.bin"), "rb").read()
    out = bytearray(b"\xCD" * 4000)
    assert k4.LZ4Codec.Decode(comp, out, dic) == 3034 and bytes(out[:3034]) == expect
    assert bytes(out[3034:]) == b"\xCD" * (4000 - 3034)
    assert k4.LZ4Codec.Decode(comp, bytearray(3034)) == -1                 # without the dictionary
    assert k4.LZ4Codec.Decode(comp, 0, len(comp), out, 0, 3034, dic, 0, len(dic)) == 3034
    rng = np.random.default_rng(21)
    streams, caps, dicts = [], [], []
    for it in range(1500):
        n = int(rng.choice([40, 200, 1000, 5000]))
        c = bytearray(port.encode(inputs.gen(["text2", "lowent", "runs", "lorem", "random"][it % 5], n, it))[1])
        if it % 3 and len(c) > 8:
            for _ in range(3):
                c[int(rng.integers(1, len(c) - 2))] = int(rng.integers(0, 256))
        streams.append(bytes(c)); caps.append(int(rng.choice([n, n + 9, n - 1, 2 * n])))
        dicts.append(inputs.gen("text2", int(rng.choice([0, 1, 7, 64, 300, 4096, 70000])), it + 1))
    dec, got = k4.batch.decode_dict_batch_host(streams, caps, dicts)
    for i in range(len(streams)):
        r, ref = port.decode_dict(streams[i], caps[i], dicts[i]) if dicts[i] else port.decode(streams[i], caps[i])
        assert int(got[i]) == r, (i, int(got[i]), r)
        if r > 0 and not inputs.uses_zero_offset(streams[i]):
            assert dec[i] == ref, i


def test_partial_decode_gpu(k4):
    """LZ4Codec.PartialDecode (LZ4Codec.cs:123-134; PartialDecompressionTests.cs:10-46)."""
    import oracle
    port = oracle.Port()
    for size, num in [(127, 127), (128, 128), (256, 256), (512, 17), (511, 13), (511, 31)]:
        src = inputs.gen("lorem", size, 0)
        enc = bytearray(k4.LZ4Codec.MaximumOutputSize(size))
        n = k4.LZ4Codec.Encode(src, enc)
        dec = bytearray(b"\xCD" * size)
        assert k4.LZ4Codec.PartialDecode(bytes(enc[:n]), 0, n, dec, 0, num) == num
        assert bytes(dec[:num]) == src[:num] and bytes(dec[num:]) == b"\xCD" * (size - num)
    rng = np.random.default_rng(4)
    streams, targets = [], []
    for it in range(1500):
        n = int(rng.choice([30, 100, 1000, 5000, 70000]))
        c = port.encode(inputs.gen(["text2", "lowent", "runs", "lorem", "random"][it % 5], n, it))[1]
        if it % 4 == 3:
            c = inputs.mutate(c, rng)
        streams.append(c)
        targets.append(int(rng.choice([0, 1, 5, 12, 13, n // 3, n // 2, n - 1, n, n + 1, 2 * n])))
    dec, got = k4.batch.partial_decode_batch_host(streams, targets)
    for i in range(len(streams)):
        r, ref = port.partial_decode(streams[i], targets[i])
        assert int(got[i]) == r, (i, int(got[i]), r)
        if r > 0 and not inputs.uses_zero_offset(streams[i]):
            assert dec[i] == ref, i


def test_block_encoder_decoder_batched_topup(k4):
    """SURVEY 8f row 1: LZ4BlockEncoder / LZ4BlockDecoder with a batched top-up equal N single-block
    reference calls (Encoders/LZ4EncoderBase.cs:47-87, LZ4BlockEncoder.cs:18-23, LZ4BlockDecoder.cs:39-55)."""
    import oracle
    port = oracle.Port()
    bs = 65536
    data = (inputs.gen("text2", 3 * bs, 1) + inputs.gen("random", bs, 2) + inputs.gen("synth525", 2 * bs, 3)
            + inputs.gen("lorem", 5000, 4))                                   # last block is short
    enc = k4.LZ4BlockEncoder(k4.LZ4Level.L00_FAST, bs, batch_blocks=16)
    assert enc.BlockSize == bs
    assert enc.TopupMany(data) == len(data) and enc.BlocksQueued == 7
    got = enc.EncodeMany(allowCopy=True)
    assert len(got) == 7 and enc.BlocksQueued == 0
    blocks = [data[i:i + bs] for i in range(0, len(data), bs)]
    for (n, payload), raw in zip(got, blocks):
        r, ref = port.encode(raw)                                             # LZ4Codec.Encode per block
        if r >= len(raw):
            assert n == -len(raw) and payload == raw                          # allowCopy: stored raw
        else:
            assert (n, payload) == (r, ref)
    assert got[3][0] == -bs                                                   # the random block did not compress
    # allowCopy=False keeps the expanded stream
    assert enc.TopupMany(blocks[3]) == bs
    (n, payload), = enc.EncodeMany(allowCopy=False)
    assert (n, payload) == port.encode(blocks[3])
    # single-block interface (Topup / Encode) and the too-small-target error
    assert enc.Topup(blocks[0][:1000]) == 1000 and enc.BytesReady == 1000
    tgt = bytearray(k4.LZ4Codec.MaximumOutputSize(1000))
    n = enc.Encode(tgt, allowCopy=True)
    assert (n, bytes(tgt[:n])) == port.encode(blocks[0][:1000])
    assert enc.Topup(blocks[3][:5000]) == 5000
    with pytest.raises(RuntimeError):
        enc.Encode(bytearray(100), allowCopy=True)
    # decoder: one call for the whole list, raw blocks passed through, Drain/Peek on the last one
    dec = k4.LZ4BlockDecoder(bs)
    out = dec.DecodeMany([(p, n < 0) for n, p in got])
    assert out == blocks
    assert dec.BytesReady == len(blocks[-1])
    tail = bytearray(10)
    dec.Drain(tail, -10, 10)
    assert bytes(tail) == blocks[-1][-10:]
    assert dec.Decode(port.encode(blocks[0])[1]) == bs and bytes(dec.Peek(-bs)) == blocks[0]
    with pytest.raises(RuntimeError):
        dec.DecodeMany([b"\x10"])            # one literal announced, none present


def test_pickle_writer_variant_matches_oracle(k4):
    """Pickle<TBufferWriter> (LZ4Pickler.pickle.cs:113-148): pessimistic header, capacity-n encode --
    different bytes than the byte[] variant for some inputs, same round trip."""
    import oracle
    port = oracle.Port()
    rng = np.random.default_rng(8)
    msgs = [b"x", inputs.gen("random", 300, 1), b"a" * 200, b"a" * 300, b"a" * 5000, b"a" * 70000, b"ab" * 40000]
    for i in range(400):
        n = int(rng.integers(1, 4097)) if i % 3 else int(rng.choice([255, 256, 257, 270, 1004, 1023, 1024, 1025, 4096]))
        msgs.append(inputs.gen(["text2", "synth435", "lorem", "random", "lowent"][i % 5], n, i))
    pk, lens = k4.batch.pickle_writer_batch_host(msgs)
    differ = 0
    for m, p in zip(msgs, pk):
        assert p == port.pickle_writer(m), len(m)
        assert k4.LZ4Pickler.Unpickle(p) == m if len(m) in (1, 200, 300, 70000) else True
        differ += p != port.pickle(m)
    assert differ > 0                       # the two variants are not byte-identical (SURVEY 8a P1')
    un, ul = k4.batch.unpickle_batch_host(pk)
    assert un == msgs
    w = bytearray(b"head")
    k4.LZ4Pickler.PickleTo(b"a" * 300, w)
    assert bytes(w) == b"head" + port.pickle_writer(b"a" * 300)


def test_enforce32_engine_gpu(k4):
    """LL.Enforce32 (LL.tools.cs:29-36): the 32-bit engine differs from the 64-bit one only for inputs of
    >= 65 547 bytes (hash4 instead of hash5 on the u32 table); both variants against the restatement."""
    import ctypes as C
    import oracle
    port = oracle.Port()
    L = k4._native.lib()
    for n in (1000, 65546, 65547, 100000, 149130):
        d = inputs.gen("text2", n, 3)
        src = np.frombuffer(d, dtype=np.uint8)
        cap = k4.LZ4Codec.MaximumOutputSize(n)
        dst = np.zeros(cap, dtype=np.uint8)
        r32 = int(L.k4lz4_encode_x32(src.ctypes.data, n, dst.ctypes.data, cap, 0))
        assert (r32, dst[:r32].tobytes()) == port.encode(d, enforce32=True), n
        r64 = int(L.k4lz4_encode(src.ctypes.data, n, dst.ctypes.data, cap, 0))
        assert (r64, dst[:r64].tobytes()) == port.encode(d), n
        out = bytearray(n)
        assert k4.LZ4Codec.Decode(dst[:r64].tobytes(), out) == n and bytes(out) == d
    a, b = port.encode(inputs.gen("text2", 149130, 3)), port.encode(inputs.gen("text2", 149130, 3), enforce32=True)
    assert a != b                                    # the two engines really differ above the threshold


def test_all_devices_split_uses_every_gpu(k4):
    """K4LZ4_ALL_DEVICES on a box with >= 2 GPUs: one host-memory call, every GPU decodes its contiguous
    slice (decode path counters per device), results identical to the single-device call.  Skipped on a
    1-GPU machine."""
    from k4os.compression.lz4_b200 import _native as N
    ndev = N.lib().k4lz4_device_count()
    if ndev < 2:
        pytest.skip("needs at least two GPUs")
    import oracle
    port = oracle.Port()
    bs, nb = 65536, 64 * ndev
    raw = port.datagen(nb * bs, 0.63, 0.0, 4321)
    blocks = [raw[i * bs:(i + 1) * bs].tobytes() for i in range(nb)]
    enc1, len1 = k4.batch.encode_batch_host(blocks, device=0)
    encA, lenA = k4.batch.encode_batch_host(blocks, device=N.ALL_DEVICES)
    assert encA == enc1 and lenA.tolist() == len1.tolist()
    for d in range(ndev):
        k4.batch.decode_stats(d, reset=True)
    src, so, sl = k4.batch._pack(enc1)
    caps = np.full(nb, bs, dtype=np.int32)
    doff = np.arange(nb, dtype=np.int64) * bs
    dst = np.zeros(nb * bs, dtype=np.uint8)
    got = k4.batch.decode_batch_flat_host(src, so, sl, dst, doff, caps, device=N.ALL_DEVICES)
    assert got.tolist() == [bs] * nb and dst.tobytes() == raw.tobytes()
    per_dev = [k4.batch.decode_stats(d, reset=True)["tile"] for d in range(ndev)]
    assert sum(per_dev) == nb and all(v > 0 for v in per_dev), per_dev


def test_frame_container_interoperates_with_upstream(k4):
    """SURVEY 8f row 2: LZ4 frames of independent blocks written by frame.write_frame decode with
    upstream lz4frame.c, upstream's frames decode with frame.read_frame, checksums (GPU XXH32 per
    block, host XXH32 for header / content) included; corruption is detected."""
    import oracle
    from k4os.compression.lz4_b200 import frame as F
    if not oracle.have_ref():
        pytest.skip("needs oracle/_ref (upstream lz4frame.c)")
    ref = oracle.Ref()
    port = oracle.Port()
    rng = np.random.default_rng(6)
    datas = [b"", b"a", inputs.gen("text2", 1000, 1), inputs.gen("synth525", 3 * 65536 + 777, 2),
             inputs.gen("random", 65536 + 5, 3), port.datagen(5 * 65536, 0.63).tobytes()]
    for d in datas:
        a = np.frombuffer(d, dtype=np.uint8)
        assert F.xxh32(d, 7) == port.xxh32(a, 7)
        for bc in (False, True):
            for cc in (False, True):
                mine = F.write_frame(d, 65536, bc, cc)
                assert ref.frame_decompress(mine, len(d) + 16) == d, (len(d), bc, cc)
                assert F.read_frame(mine) == d
                theirs = ref.frame_compress(d, bc, cc)
                assert F.read_frame(theirs) == d, (len(d), bc, cc)
    # header bytes follow LZ4FrameWriter.cs:64-102: magic, FLG = version 01 | independent | flags, BD = 4 << 4, HC
    f = F.write_frame(datas[3], 65536, True, True)
    assert f[:6] == bytes([0x04, 0x22, 0x4D, 0x18, 0x40 | 0x20 | 0x10 | 0x04, 0x40])
    assert f[6] == (port.xxh32(np.frombuffer(f[4:6], dtype=np.uint8), 0) >> 8) & 0xFF
    # the incompressible block is stored raw (bit 31 of its length code), blocking.cs:22-33 / LZ4EncoderBase.cs:79-83
    g = F.write_frame(datas[4], 65536, False, False)
    import struct
    assert struct.unpack_from("<I", g, 7)[0] == 0x80000000 | 65536
    # corruption: block payload, block checksum, header checksum, content checksum
    for at in (20, len(f) - 3, 6):
        bad = bytearray(f); bad[at] ^= 0x55
        with pytest.raises(F.InvalidDataException):
            F.read_frame(bytes(bad))
    # per-block checksums of a big batch: GPU XXH32 == restatement
    blocks = [datas[5][i:i + 65536] for i in range(0, len(datas[5]), 65536)]
    base = np.frombuffer(datas[5], dtype=np.uint8)
    got = F.xxh32_batch(base, np.arange(5) * 65536, np.array([65536, 65535, 17, 3, 0], dtype=np.int32), 9)
    want = [port.xxh32(np.frombuffer(b[:n], dtype=np.uint8), 9) for b, n in zip(blocks, [65536, 65535, 17, 3, 0])]
    assert got.tolist() == want


def test_jump_table_edge_streams_gpu(k4):
    """Streams aimed at the boundaries of the parse's jump table (csrc/parse_table.cuh): literal-length
    extension bytes 222..255 and chains of them, match-length extension bytes 253..255 and chains, sequences
    that end exactly at / one before / one behind the end of the stream, all packed back to back so that
    every stage alignment occurs.  Return codes and bytes must equal the oracle's."""
    import oracle
    port = oracle.Port()
    rng = np.random.default_rng(5)
    streams, caps = [], []

    def seq(lit, mlen, off, last=False):
        """one hand-assembled sequence: `lit` literal bytes, then (unless last) a match of mlen >= 4 at distance off"""
        out = bytearray()
        lt = min(lit, 15)
        mt = 0 if last else min(mlen - 4, 15)
        out.append((lt << 4) | mt)
        if lit >= 15:
            rest = lit - 15
            out += b"\xFF" * (rest // 255) + bytes([rest % 255])
        out += rng.integers(1, 255, lit, dtype=np.uint8).tobytes()
        if not last:
            out += bytes([off & 0xFF, off >> 8])
            if mlen - 4 >= 15:
                rest = mlen - 4 - 15
                out += b"\xFF" * (rest // 255) + bytes([rest % 255])
        return bytes(out)

    for lit in (14, 15, 16, 15 + 222, 15 + 223, 15 + 224, 15 + 254, 15 + 255, 15 + 256, 15 + 510, 15 + 511, 900):
        for mlen in (4, 18, 19, 20, 19 + 253, 19 + 254, 19 + 255, 19 + 256, 19 + 510, 19 + 765, 3000):
            body = seq(40, 8, 7) + seq(lit, mlen, 5) + seq(3, 6, 2) + seq(12, 0, 0, last=True)
            total = 40 + 8 + lit + mlen + 3 + 6 + 12
            for cut in (0, 1, 2, 5):            # truncated tails: the last sequences end at / behind the end
                s = body[:len(body) - cut] if cut else body
                streams.append(s); caps.append(total + 20)
            streams.append(body + b"\x00"); caps.append(total + 20)          # one byte behind a complete block
    # the same shapes at the far end of long valid blocks (table entries near n, big distances)
    for n in (5000, 33000, 65536):
        base = port.encode(inputs.gen("text2", n, n))[1]
        for tail in (seq(15 + 224, 19 + 255, 9) + seq(9, 0, 0, last=True), seq(300, 600, 300) + seq(5, 0, 0, last=True)):
            # a valid block is token-complete: append more sequences by re-opening its terminal literal run is not
            # possible in general, so just check the concatenation is handled like the oracle handles it
            streams.append(base + tail); caps.append(70000)
    dec, got = k4.batch.decode_batch_host(streams, caps)
    n_ok = 0
    for i, (c, cap) in enumerate(zip(streams, caps)):
        r, ref = port.decode(c, cap)
        assert int(got[i]) == r, (i, len(c), cap, int(got[i]), r)
        if r > 0 and not inputs.uses_zero_offset(c):
            assert dec[i] == ref, i
            n_ok += 1
    assert n_ok >= 100, n_ok       # the complete hand-assembled blocks decode
