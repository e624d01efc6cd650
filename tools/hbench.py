"""Host-memory benchmark of the synchronous staged calls: dictionary, partial and chained decode, chained encode,
XXH32, decoded sizes, and whole-frame encode (linked and independent), decode and content sizes.  Every batch
stages more than 256 MiB, so each call runs in at least two chunks.  Rows repeat 64 distinct sources, so host
memory stays small while the staged bytes do not.

    python tools/hbench.py [--lib A.so,B.so] [--reps 3]

With several libraries (default: the in-tree build) each row is timed in two alternating rounds, A B A B, after
one warm-up call per library; a round is the best of --reps calls, timed on the host clock around the call
(host-memory calls return when their results are in place).  The outputs of every library must be equal.
Prints the card name and power limit, then one JSON line per row with GB/s of source bytes per round."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.fbench import card  # noqa: E402

BS = 1 << 16
SB = 16400


def a16(x: int) -> int:
    return (x + 15) // 16 * 16


def pack(parts, rows, pre=None):
    """Distinct byte strings stored once (16-aligned, each with pre[k] bytes of its own in front) -> (buffer,
    offset of row i's part, length of row i's part)."""
    offs, at = [], 0
    for k, p in enumerate(parts):
        at = a16(at + (len(pre[k]) if pre else 0))
        offs.append(at)
        at += len(p)
    buf = np.zeros(at + 16, dtype=np.uint8)
    for k, (o, p) in enumerate(zip(offs, parts)):
        h = pre[k] if pre else b""
        buf[o - len(h):o + len(p)] = np.frombuffer(h + p, dtype=np.uint8)
    return (buf, np.array([offs[r] for r in rows], dtype=np.int64),
            np.array([len(parts[r]) for r in rows], dtype=np.int32))


def slots(n, cap, hist=None):
    """n destination slots of `cap` bytes, each with `hist` in front of it -> (buffer, offsets, capacities)."""
    h = len(hist) if hist else 0
    stride = a16(h + cap + 32)
    dst = np.zeros(n * stride + 16, dtype=np.uint8)
    do = np.arange(n, dtype=np.int64) * stride + a16(h)
    if hist:
        for o in do:
            dst[o - h:o] = np.frombuffer(hist, dtype=np.uint8)
    return dst, do, np.full(n, cap, dtype=np.int32)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default="", help="comma-separated builds of libk4lz4.so to compare (default: in-tree)")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from k4os.compression.lz4_b200 import _native as N, batch as B
    print("card:", card(), flush=True)
    paths = [os.path.abspath(p) for p in a.lib.split(",") if p] or [N.SO_PATH]
    libs = []
    for p in paths:
        L = C.CDLL(p)
        for name, (args, res) in N.SIGNATURES.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = args, res
        libs.append((os.path.relpath(p), L))

    raw = B.synth_host(64, BS, 525, seed=5)
    plain = [raw[i * BS:(i + 1) * BS].tobytes() for i in range(64)]
    enc, _ = B.encode_batch_host(plain)
    big = b"".join(plain)
    contents = [big[k * 4099:k * 4099 + (1 << 20)] for k in range(64)]
    P = lambda x: x.ctypes.data                                                  # noqa: E731
    H = N.MEM_HOST

    def rows_of(n):
        return [i % 64 for i in range(n)]

    work = {}                  # name -> (source bytes, prepare() -> fresh outputs, call(L, outputs))

    def add(name, nbytes, prepare, call):
        work[name] = (nbytes, prepare, call)

    def out_only(n, dtype=np.int32):
        return lambda: (np.zeros(n, dtype),)

    def with_slots(n, cap, hist=None, state=False):
        def prepare():
            dst, do, dc = slots(n, cap, hist)
            return (np.zeros(n, np.int32), dst, do, dc) + ((np.zeros(n * SB, np.uint8),) if state else ())
        return prepare

    n = 3000
    s1, so1, sl1 = pack(enc, rows_of(n))
    dic = np.frombuffer(plain[63], dtype=np.uint8).copy()
    dio, dil = np.zeros(n, np.int64), np.full(n, BS, np.int32)
    add("dict_decode", int(sl1.sum()), with_slots(n, BS), lambda L, o, n=n: L.k4lz4_decode_dict_batch(
        P(s1), P(so1), P(sl1), P(o[1]), P(o[2]), P(o[3]), P(dic), P(dio), P(dil), P(o[0]), n, H, None, 0))

    n = 4000
    s2, so2, sl2 = pack(enc, rows_of(n))
    add("partial_decode", int(sl2.sum()), with_slots(n, BS - 1000), lambda L, o, n=n: L.k4lz4_partial_decode_batch(
        P(s2), P(so2), P(sl2), P(o[1]), P(o[2]), P(o[3]), P(o[0]), n, H, None, 0))

    n = 2500
    s3, so3, sl3 = pack(enc, rows_of(n))
    pre3 = np.full(n, BS, np.int32)
    add("chain_decode", int(sl3.sum()), with_slots(n, BS, plain[7]), lambda L, o, n=n: L.k4lz4_decode_chain_batch(
        P(s3), P(so3), P(sl3), P(o[1]), P(o[2]), P(o[3]), P(pre3), P(o[0]), n, H, None, 0))

    n = 1500
    s4, so4, sl4 = pack(plain, rows_of(n), pre=[plain[(k + 63) % 64] for k in range(64)])
    pl4 = np.full(n, BS, np.int32)
    sto = np.arange(n, dtype=np.int64) * SB
    add("chain_encode", int(sl4.sum()), with_slots(n, BS + BS // 255 + 16, state=True),
        lambda L, o, n=n: L.k4lz4_encode_chain_batch(P(s4), P(so4), P(sl4), P(pl4), P(o[1]), P(o[2]), P(o[3]), P(o[4]),
                                                     P(sto), P(o[0]), n, 0, H, None, 0))

    n = 6000
    s5, so5, sl5 = pack(plain, rows_of(n))
    add("xxh32", int(sl5.sum()), out_only(n, np.uint32), lambda L, o, n=n: L.k4lz4_xxh32_batch(
        P(s5), P(so5), P(sl5), 9, P(o[0]), n, H, None, 0))

    n = (512 << 20) // int(np.mean([len(e) for e in enc]))
    s6, so6, sl6 = pack(enc, rows_of(n))
    add("decoded_size", int(sl6.sum()), out_only(n), lambda L, o, n=n: L.k4lz4_decoded_size_batch(
        P(s6), P(so6), P(sl6), P(o[0]), n, H, None, 0))

    n = 300
    s7, so7, sl7 = pack(contents, rows_of(n))
    frames = []
    for mode, fl in (("linked", 0), ("independent", N.FRAME_INDEPENDENT)):
        bound = int(libs[0][1].k4lz4_frame_bound(1 << 20, BS, fl))
        call = lambda L, o, n=n, fl=fl: L.k4lz4_frame_encode_batch(  # noqa: E731
            P(s7), P(so7), P(sl7), P(o[1]), P(o[2]), P(o[3]), P(o[0]), n, BS, fl, 0, H, None, 0)
        add(f"frame_encode_{mode}", int(sl7.sum()), with_slots(n, bound), call)
        o = with_slots(n, bound)()
        N.check(call(libs[0][1], o))
        frames += [o[1][d:d + r].tobytes() for d, r in zip(o[2][:64], o[0][:64])]

    n = 300
    s8, so8, sl8 = pack(frames, [i % 128 for i in range(n)])
    add("frame_decode", int(sl8.sum()), with_slots(n, 1 << 20), lambda L, o, n=n: L.k4lz4_frame_decode_batch(
        P(s8), P(so8), P(sl8), P(o[1]), P(o[2]), P(o[3]), P(o[0]), n, H, None, 0))

    n = (512 << 20) // int(np.mean([len(f) for f in frames]))
    s9, so9, sl9 = pack(frames, [i % 128 for i in range(n)])
    add("frame_content_size", int(sl9.sum()), out_only(n), lambda L, o, n=n: L.k4lz4_frame_content_size_batch(
        P(s9), P(so9), P(sl9), P(o[0]), n, H, None, 0))

    for name, (nbytes, prepare, call) in work.items():
        outs = {}
        for tag, L in libs:                      # warm-up: staging buffers, module loads
            o = prepare()
            N.check(call(L, o))
            outs[tag] = o
        ref = outs[libs[0][0]]
        for tag, _ in libs[1:]:
            assert all(np.array_equal(x, y) for x, y in zip(outs[tag], ref)), (name, tag)
        assert (ref[0].view(np.int32) > 0).any(), name
        del outs
        rounds = {tag: [] for tag, _ in libs}
        for _ in range(2):
            for tag, L in libs:
                best = float("inf")
                for _ in range(a.reps):
                    o = prepare()
                    t0 = time.perf_counter()
                    rc = call(L, o)
                    best = min(best, time.perf_counter() - t0)
                    N.check(rc)
                rounds[tag].append(round(nbytes / best / 1e9, 3))
        print(json.dumps({"row": name, "source_MB": round(nbytes / 1e6, 1), "GBps": rounds}), flush=True)


if __name__ == "__main__":
    main()
