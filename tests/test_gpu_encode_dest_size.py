"""Encoding into fixed-size destinations on the GPU (k4lz4_encode_dest_size_batch / k4lz4_encode_dest_size),
compared byte for byte with upstream lz4's LZ4_compress_destSize, and pages of a long input packed by stepping
calls and decoded back."""
import ctypes as C

import numpy as np
import pytest

from tests import dest_size_ref as D
from tests.lz4_blocks import parse

pytestmark = pytest.mark.gpu

CANARY = 0xCD


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


@pytest.fixture(scope="module")
def up():
    import oracle
    if not oracle.have_ref():
        pytest.fail("oracle/_ref/libk4ref.so missing: run __graft_entry__.build() where the reference is present")
    return D.Upstream()


@pytest.fixture(scope="module")
def grid(up):
    """[(src, target)] over the whole grid of the model test: every size, content and target."""
    pairs = []
    for kind in D.KINDS:
        for n in D.SIZES:
            src = D.content(kind, n, 7 + n)
            pairs += [(src, t) for t in D.targets(n, 11 + n, 48)]
    return pairs


def _host(native, pairs):
    """One host-memory call -> (dst buffer, dst offsets, outLen, srcUsed)."""
    from k4os.compression.lz4_b200 import _native as N, batch
    src, so, sl = batch._pack([s for s, _ in pairs])
    dst, doff, dc = batch._slots([t for _, t in pairs])
    out = np.full(len(pairs), -7, dtype=np.int32)
    used = np.full(len(pairs), -7, dtype=np.int32)
    N.check(native.k4lz4_encode_dest_size_batch(src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                doff.ctypes.data, dc.ctypes.data, out.ctypes.data, used.ctypes.data,
                                                len(pairs), N.MEM_HOST, None, 0))
    return dst, doff, out, used


def _device(pairs, stream=0):
    """The same batch in device memory, the destinations filled with the canary first."""
    import torch
    from k4os.compression.lz4_b200 import batch
    src, so, sl = batch._pack([s for s, _ in pairs])
    dst, doff, dc = batch._slots([t for _, t in pairs])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    g = [t(src), t(so), t(sl), t(dst), t(doff), t(dc),
         torch.full((len(pairs),), -7, dtype=torch.int32, device="cuda"),
         torch.full((len(pairs),), -7, dtype=torch.int32, device="cuda")]
    batch.encode_dest_size_batch_device(*[x.data_ptr() for x in g], len(pairs), stream=stream, device=0)
    torch.cuda.synchronize()
    return g[3].cpu().numpy(), doff, g[6].cpu().numpy(), g[7].cpu().numpy()


def _check(up, pairs, dst, doff, out, used):
    for i, (src, t) in enumerate(pairs):
        r, u, want = up.dest_size(src, t)
        if r == 0:
            u = 0
        o = int(doff[i])
        assert (out[i], used[i]) == (r, u), (i, len(src), t, out[i], used[i], r, u)
        assert dst[o:o + r].tobytes() == want, (i, len(src), t)
        assert (dst[o + r:o + max(t, 0)] == CANARY).all(), ("written past the result", i, len(src), t)


def test_grid_equals_upstream_host_memory(k4, native, up, grid):
    assert len(grid) >= 2000
    _check(up, grid, *_host(native, grid))


def test_grid_equals_upstream_device_memory(k4, up, grid):
    pytest.importorskip("torch")
    _check(up, grid, *_device(grid))


def test_python_mirror_and_single_call(k4, native, up):
    from k4os.compression.lz4_b200 import batch
    srcs = [D.content("datagen", 70000, 3), D.content("runs", 5000, 4), b"", D.content("random", 300, 5)]
    targets = [4096, 100, 7, 200]
    res, out, used = batch.encode_dest_size_batch_host(srcs, targets)
    for i, (s, t) in enumerate(zip(srcs, targets)):
        r, u, want = up.dest_size(s, t)
        assert (out[i], used[i], res[i]) == (r, u, want), i
        buf = np.full(t + 8, CANARY, dtype=np.uint8)
        size = C.c_int32(len(s))
        sp = np.frombuffer(s, dtype=np.uint8).ctypes.data if s else None
        assert native.k4lz4_encode_dest_size(sp, buf.ctypes.data, C.byref(size), t) == r
        assert size.value == u and buf[:r].tobytes() == want and (buf[r:] == CANARY).all(), i


def test_rule_families(k4, native, up):
    """Per input, the targets at which the model says each rule first fires; the match-length rule on run data on
    both sides of 65 547 bytes."""
    pairs, seen = [], set()
    for kind in D.KINDS:
        for n in (13, 14, 4096, 65535, 65546, 65547, 65548, 300000, 1 << 20):
            src = D.content(kind, n, 100 + n)
            seqs = parse(up.plain(src))
            for rule, t in D.rule_targets(seqs, n).items():
                for dt in (-1, 0, 1):
                    if t + dt >= 1:
                        pairs.append((src, t + dt))
                seen.add((kind, rule, n >= D.LIMIT_64K))
    assert ("runs", 3, False) in seen and ("runs", 3, True) in seen, sorted(seen)
    assert {(r, big) for _, r, big in seen} == {(r, big) for r in (1, 2, 3, 4) for big in (False, True)}
    _check(up, pairs, *_host(native, pairs))


def test_both_warp_kinds(k4, native, up):
    """More blocks below 65 547 bytes than the shared-memory warps take in one round: the global-table warps encode
    some of them, and every block is bit-exact."""
    from k4os.compression.lz4_b200 import batch
    nb = 6000
    rng = np.random.default_rng(61)
    body = D.content("datagen", nb * 4096, 62)
    pairs = []
    for i in range(nb):
        n = int(rng.integers(13, 8192))
        s = body[(i * 4096) % (len(body) - n):][:n]
        t = int(rng.integers(1, D.bound(n) + 1)) if i % 4 else D.bound(n)
        pairs.append((s, t))
    batch.encode_stats(0, reset=True)
    got = _host(native, pairs)
    st = batch.encode_stats(0, reset=True)
    assert st["smem"] > 0 and st["gtab"] > 0 and st["smem"] + st["gtab"] == nb, st
    _check(up, pairs, *got)


def test_page_packing(k4, native, up):
    """Inputs of up to 1 MiB packed into 4 KiB pages: each call encodes the next page of every unfinished input,
    from where the input's earlier pages ended.  Every page decodes alone and the pages concatenate to the input."""
    from k4os.compression.lz4_b200 import batch
    page = 4096
    inputs = [D.content("datagen", 1 << 20, 71), D.content("random", 300000, 72), D.content("runs", 1 << 20, 73),
              D.content("datagen", 100000, 74), D.content("runs", 65547, 75)]
    pos = [0] * len(inputs)
    pages = [[] for _ in inputs]
    for _ in range(400):
        live = [i for i, s in enumerate(inputs) if pos[i] < len(s)]
        if not live:
            break
        rest = [inputs[i][pos[i]:] for i in live]
        res, out, used = batch.encode_dest_size_batch_host(rest, [page] * len(live))
        for k, i in enumerate(live):
            r, u, want = up.dest_size(rest[k], page)
            assert (out[k], used[k], res[k]) == (r, u, want), (i, pos[i])
            assert 0 < used[k] <= len(rest[k]) and out[k] <= page
            pages[i].append((res[k], int(used[k])))
            pos[i] += int(used[k])
    assert all(p == len(s) for p, s in zip(pos, inputs))
    flat = [(blk, u) for ps in pages for blk, u in ps]
    dec, dl = batch.decode_batch_host([blk for blk, _ in flat], [u for _, u in flat])
    assert list(dl) == [u for _, u in flat]
    for i, s in enumerate(inputs):
        k0 = sum(len(ps) for ps in pages[:i])
        assert b"".join(dec[k0:k0 + len(pages[i])]) == s, i
