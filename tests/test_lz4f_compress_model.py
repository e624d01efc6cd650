"""k4lz4_lz4f_compress_batch's rule, on the CPU: the restatement in tests/lz4f_ref.py (the per-frame block size,
mode and content size, then upstream's block calls with capacity n - 1 and raw storage when they fail) equals
upstream's LZ4F_compressFrame on every frame of the grid, and the grid covers what it must.  Also the bound and
the argument checks, which need no GPU.  Needs the reference engine that __graft_entry__.build() compiles into
oracle/_ref/."""
import struct

import pytest

from tests import lz4f_ref as R


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return R.Lz4fUpstream()


def _parse(f: bytes):
    """-> (FLG, BD, [(length, raw), ...]) of a frame the assembly wrote."""
    flg, bd = f[4], f[5]
    p = 7 + (8 if flg & 8 else 0)
    blocks = []
    while True:
        code = struct.unpack_from("<I", f, p)[0]
        p += 4
        if code == 0:
            return flg, bd, blocks
        blocks.append((code & 0x7FFFFFFF, bool(code >> 31)))
        p += (code & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)


def test_assembly_equals_upstream_on_the_grid(up):
    for data, bs, fl, kind in R.grid():
        assert up.assemble(data, bs, fl) == up.frame(data, bs, fl), (len(data), bs, fl, kind)


def test_grid_covers_the_rule(up):
    cases = R.grid()
    sizes = {len(c[0]) for c in cases}
    assert set(R.SMALL_SIZES) <= sizes
    assert {s + d for s in R.BLOCK_SIZES for d in (-1, 0, 1)} <= sizes
    combos = {(bs, fl & 15) for _, bs, fl, _ in cases}
    assert combos == {(bs, R.flags_of(l, bc, cc, cs)) for bs in R.BLOCK_SIZES for l in (True, False)
                      for bc, cc in R.CHECKSUMS for cs in (False, True)}
    assert {k for *_, k in cases} == {"text", "random", "zeros", "mixed"}
    seen = set()
    for data, bs, fl, kind in cases:
        flg, bd, blocks = _parse(up.assemble(data, bs, fl))
        size = 1 << (8 + 2 * ((bd >> 4) & 7))
        if size < bs:
            seen.add("shrunk")
        if not (fl & R.INDEPENDENT) and flg & 0x20:
            seen.add("one block made independent")
        if not (flg & 0x20) and len(blocks) > 1:
            seen.add("linked")
            if any(raw and 0 < k < len(blocks) - 1 for k, (_, raw) in enumerate(blocks)) and not blocks[-1][1]:
                seen.add("linked raw mid-stream")
        if fl & R.CONTENT_SIZE:
            seen.add("content size" if flg & 8 else "content size dropped")
        if len(blocks) > 1:
            seen.add(f"multi-block {bs}")
        if any(raw for _, raw in blocks):
            seen.add("raw")
        if any(not raw for _, raw in blocks):
            seen.add("compressed")
    want = {"shrunk", "one block made independent", "linked", "linked raw mid-stream", "content size",
            "content size dropped", "raw", "compressed"} | {f"multi-block {bs}" for bs in R.BLOCK_SIZES}
    assert want <= seen, sorted(want - seen)


def test_bound_equals_upstream(native, up):
    for bs in R.BLOCK_SIZES:
        for fl in range(16):
            for n in (0, 1, 65535, 65536, 65537, bs - 1, bs, bs + 1, 3 * bs + 5, (1 << 31) - 1):
                assert native.k4lz4_lz4f_compress_bound(n, bs, fl) == up.bound(n, bs, fl), (n, bs, fl)


def test_argument_checks(native):
    from k4os.compression.lz4_b200 import _native as N
    assert native.k4lz4_lz4f_compress_bound(10, 1 << 16, 16) == N.E_ARG
    assert native.k4lz4_lz4f_compress_bound(-1, 1 << 16, 0) == N.E_ARG
    for bs in (0, 1024, 65535, 65537, 1 << 17, 8 << 20):
        assert native.k4lz4_lz4f_compress_bound(10, bs, 0) == N.E_ARG
        assert native.k4lz4_lz4f_compress_batch(None, None, None, None, None, None, None, 0, bs, 0, 0,
                                                N.MEM_HOST, None, 0) == N.E_ARG
    assert native.k4lz4_lz4f_compress_batch(None, None, None, None, None, None, None, 0, 1 << 16, 16, 0,
                                            N.MEM_HOST, None, 0) == N.E_ARG
    assert native.k4lz4_lz4f_compress_batch(None, None, None, None, None, None, None, 0, 1 << 16, 0, 0,
                                            7, None, 0) == N.E_ARG
    assert native.k4lz4_lz4f_compress_batch(None, None, None, None, None, None, None, 1, 1 << 16, 0, 0,
                                            N.MEM_HOST, None, 0) == N.E_ARG
