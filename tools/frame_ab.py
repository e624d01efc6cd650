"""A/B of two builds of libk4lz4.so on the whole-frame encoders and decoders, in one process: the reference's
LZ4FrameWriter frames (k4lz4_frame_encode_batch, _x32), upstream's CDict frames (k4lz4_frame_encode_dict_batch) and
upstream's LZ4F_compressFrame (k4lz4_lz4f_compress_batch), and the readers of each.

Part 1, equality: every format x linked / independent x the four checksum pairs x content size (where the format
has one), in host and device memory, on seeded datagen and random content of 0 B .. 1.5 MiB per frame, with
destinations at the bound, below it and far below it, a mixed LZ4F call, and CDict frames with and without IDs.
Each call runs on both builds with the same inputs; the whole destination buffer (frames, slack and the 0xCD fill
around them) and every result must be byte-identical.  The launch count of each call (k4lz4_launch_count) is
reported for both builds; B must never launch more than A, and exactly as many for the reference's frames.

Part 2, decode equality: the whole-frame decoders -- k4lz4_frame_decode_batch, _decode_dict_batch (with the
dictionaries, with empty ones and with dictBase null), _content_size_batch, _info_batch, k4lz4_lz4f_decompress_batch
(with and without dictionaries) and _decompressed_size_batch -- on every frame part 1's baseline wrote (one input
set larger than a 256 MiB host staging chunk), the seeded grids of tests/lz4f_dec_ref.py and tests/frame_dict_ref.py,
and a truncated reference frame larger than its destination, which must stay K4LZ4_R_CORRUPT.  Destinations of the
content size, one byte less, half, 10 bytes and 64 KiB more, each entry getting each in turn.  rc, every result
column, the whole destination buffer and the k4lz4_decode_stats deltas must be identical; B launches exactly as many
kernels as A, except the info call: one fewer per device call and per host chunk.

Part 3, time: the workloads of tools/fbench.py, dfbench.py and lz4fbench.py (1 MiB datagen frames, 64 KiB and
4 MiB blocks, a 64 KiB dictionary; small record-like messages against a dictionary), each encoded and then decoded
by its reader, lz4f streams of 16 frames and legacy streams, device memory, CUDA events, the two builds alternating
rep by rep, in the order AB, then BA.

    python tools/frame_ab.py --a OLD.so [--b NEW.so] [--reps 15] [--only TEXT] [--out DIR]

--only TEXT: skip parts 1 and 2 and time only the workloads whose label contains TEXT.

Prints the card name and power limit, then JSON lines; with --out also writes them to DIR/frame_ab.jsonl."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fbench import card  # noqa: E402

MB = 1 << 20


def load(path: str):
    from k4os.compression.lz4_b200 import _native as N
    L = ctypes.CDLL(os.path.abspath(path))
    for name, (args, res) in N.SIGNATURES.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = args, res
    return L


class Inputs:
    """One call's frames, in host memory and (lazily) on the device."""

    def __init__(self, frames, caps, dicts=None, ids=None):
        self.frames, self.n = frames, len(frames)
        sizes = [len(f) for f in frames]
        self.src = np.concatenate(frames + [np.zeros(1, np.uint8)]).astype(np.uint8)
        self.so = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if frames else np.zeros(0, np.int64)
        self.sl = np.array(sizes, dtype=np.int32)
        self.dc = np.array(caps, dtype=np.int32)
        slack = 64
        self.do = np.concatenate([[slack], slack + np.cumsum(np.array(caps) + slack)[:-1]]).astype(np.int64)
        self.dst_bytes = int(self.do[-1] + caps[-1] + slack)
        self.dicts = dicts
        if dicts is not None:
            self.dsrc = np.concatenate(dicts + [np.zeros(1, np.uint8)]).astype(np.uint8)
            dl = [len(d) for d in dicts]
            self.doff = np.concatenate([[0], np.cumsum(dl)[:-1]]).astype(np.int64)
            self.dlen = np.array(dl, dtype=np.int32)
        self.ids = None if ids is None else np.array(ids, dtype=np.uint32).view(np.int32)

    def args(self, mem: str):
        """(src, srcOff, srcLen, dst, dstOff, dstCap, out, dict args | None, ids | None, keep-alive)."""
        import torch
        dst = np.full(self.dst_bytes, 0xCD, dtype=np.uint8)
        out = np.full(self.n, 0x7F7F7F7F, dtype=np.int32)
        arrs = [self.src, self.so, self.sl, dst, self.do, self.dc, out]
        d = [] if self.dicts is None else [self.dsrc, self.doff, self.dlen]
        ids = [] if self.ids is None else [self.ids]
        if mem == "device":
            t = [torch.from_numpy(a).cuda() for a in arrs + d + ids]
            ptr = [x.data_ptr() for x in t]
        else:
            t = arrs + d + ids
            ptr = [a.ctypes.data for a in t]
        dp = ptr[7:10] if d else None
        ip = ptr[-1] if ids else None
        return ptr[:7], dp, ip, t

    @staticmethod
    def result(t, mem):
        if mem == "device":
            import torch
            torch.cuda.synchronize()
            return t[3].cpu().numpy().copy(), t[6].cpu().numpy().copy()
        return t[3].copy(), t[6].copy()


def call(L, kind, inp, mem, bs, flags, level=0, st=None):
    from k4os.compression.lz4_b200 import _native as N
    p, dp, ip, t = inp.args(mem)
    mk = N.MEM_DEVICE if mem == "device" else N.MEM_HOST
    before = L.k4lz4_launch_count()
    if kind == "writer":
        rc = L.k4lz4_frame_encode_batch(*p[:6], p[6], inp.n, bs, flags, level, mk, st, -1)
    elif kind == "writer_x32":
        rc = L.k4lz4_frame_encode_batch_x32(*p[:6], p[6], inp.n, bs, flags, level, mk, st, -1)
    elif kind == "cdict":
        rc = L.k4lz4_frame_encode_dict_batch(*p[:6], *dp, ip, p[6], inp.n, bs, flags, level, mk, st, -1)
    else:
        rc = L.k4lz4_lz4f_compress_batch(*p[:6], p[6], inp.n, bs, flags, level, mk, st, -1)
    dst, out = Inputs.result(t, mem)
    return rc, dst, out, L.k4lz4_launch_count() - before


def equality(A, B, emit, written=None) -> bool:
    """Part 1; `written`, a list, gets every (frame, dictionary) the baseline wrote in host memory."""
    import oracle
    from k4os.compression.lz4_b200 import _native as N
    port = oracle.Port()
    rng = np.random.default_rng(20261018)
    sizes = [0, 1, 13, 100, 4096, 65535, 65536, 65537, 100000, 262145, MB, MB + MB // 2]
    frames = []
    for i, n in enumerate(sizes):
        frames.append(port.datagen(n, 0.63, 0.0, 500 + i) if n else np.zeros(0, np.uint8))
        frames.append(rng.integers(0, 256, n, dtype=np.uint8))
    frames = [np.asarray(f, dtype=np.uint8) for f in frames]
    # per-frame dictionaries: none, small, 64 KiB, larger than the window; IDs: zero and non-zero
    dicts = [np.asarray(port.datagen([0, 700, 65536, 100000][i % 4], 0.63, 0.0, 900 + i), dtype=np.uint8)
             if i % 4 else np.zeros(0, np.uint8) for i in range(len(frames))]
    ids = [0 if i % 3 == 0 else 0x1000 * i + 7 for i in range(len(frames))]
    bound = lambda L, kind, n, bs, fl, did: (  # noqa: E731
        int(L.k4lz4_lz4f_compress_bound(n, bs, fl)) if kind == "lz4f" else
        int(L.k4lz4_frame_bound(n, bs, fl & 7)) + (4 if did else 0))

    def caps_for(kind, bs, fl, did):
        caps = []
        for i, f in enumerate(frames):
            b = bound(A, kind, len(f), bs, fl, did and ids[i])
            caps.append(b if i % 5 else (b // 2 if i % 10 else 10))
        return caps

    ok, counts = True, {}
    plan = []
    for fl in range(8):
        for bs in (65536, 100000, 4 << 20):
            plan.append(("writer", bs, fl, False))
        plan.append(("writer_x32", 65536, fl, False))
        for bs in (65536, 1 << 20):
            plan.append(("cdict", bs, fl, False))
            plan.append(("cdict", bs, fl, True))
        for bs in (65536, 1 << 22):
            plan.append(("lz4f", bs, fl, False))
            plan.append(("lz4f", bs, fl | N.FRAME_CONTENT_SIZE, False))
    for kind, bs, fl, did in plan:
        inp = Inputs(frames, caps_for(kind, bs, fl, did), dicts if kind == "cdict" else None,
                     ids if did else None)
        for mem in ("host", "device"):
            ra, da, oa, la = call(A, kind, inp, mem, bs, fl)
            rb, db, ob, lb = call(B, kind, inp, mem, bs, fl)
            same = ra == rb and np.array_equal(da, db) and np.array_equal(oa, ob)
            launch_ok = lb <= la and (lb == la or not kind.startswith("writer"))
            if written is not None and mem == "host":
                written += [(da[inp.do[i]:inp.do[i] + oa[i]], dicts[i]) for i in range(inp.n) if oa[i] > 0]
            ok &= same and launch_ok and ra == 0
            key = (kind, mem, "indep" if fl & 1 else "linked")
            counts.setdefault(key, []).append((la, lb))
            if not (same and launch_ok and ra == 0):
                emit({"mismatch": [kind, mem, bs, fl, did], "rc": [ra, rb], "launches": [la, lb],
                      "bytes_equal": bool(np.array_equal(da, db)), "results_equal": bool(np.array_equal(oa, ob))})
    # a mixed LZ4F call: many small frames beside one long linked frame
    small = [np.asarray(port.datagen(4096, 0.63, 0.0, 3000 + i), dtype=np.uint8) for i in range(300)]
    big = np.asarray(port.datagen(10 * MB, 0.63, 0.0, 77), dtype=np.uint8)
    for bs in (65536, 1 << 22):
        items = small + [big]
        inp = Inputs(items, [int(A.k4lz4_lz4f_compress_bound(len(x), bs, 0)) for x in items])
        for mem in ("host", "device"):
            ra, da, oa, la = call(A, "lz4f", inp, mem, bs, 0)
            rb, db, ob, lb = call(B, "lz4f", inp, mem, bs, 0)
            same = ra == rb == 0 and np.array_equal(da, db) and np.array_equal(oa, ob) and bool((oa > 0).all())
            ok &= same and lb <= la
            emit({"mixed_lz4f": f"300 x 4 KiB + 1 x 10 MiB, block {bs}", "mem": mem, "identical": bool(same),
                  "launches_a": la, "launches_b": lb})
    for (kind, mem, mode), v in sorted(counts.items()):
        la, lb = zip(*v)
        emit({"launches": [kind, mem, mode], "calls": len(v), "a_total": int(sum(la)), "b_total": int(sum(lb)),
              "b_minus_a": sorted(set(int(y - x) for x, y in v))})
    emit({"equality_calls": 2 * len(plan) + 4, "all_identical": bool(ok)})
    return ok


DECODES = ("frame", "dict", "dict_empty", "dict_null", "lz4f", "lz4f_dict")
SIZES = ("content_size", "info", "lz4f_size")
STAGE_BYTES = 256 * MB          # k4lz4_api.cu: the staged bytes of one host chunk


def decode_stats(L) -> np.ndarray:
    v = np.zeros(4, dtype=np.uint64)
    assert L.k4lz4_decode_stats(0, v.ctypes.data, 0) == 0
    return v


def dcall(L, kind, inp, mem):
    """One decode call of `kind` on inp -> (rc, destination buffer, [outLen and the call's other result columns],
    launches, k4lz4_decode_stats delta)."""
    import torch
    from k4os.compression.lz4_b200 import _native as N
    n = inp.n
    a = {"src": inp.src, "so": inp.so, "sl": inp.sl, "dst": np.full(inp.dst_bytes, 0xCD, dtype=np.uint8),
         "do": inp.do, "dc": inp.dc, "o0": np.full(n, 0x7F7F7F7F, dtype=np.int32)}
    if kind == "info":
        a["o1"] = np.full(n, 0x7F7F7F7F7F7F7F7F, dtype=np.int64)
    if kind.startswith("lz4f"):
        a["o1"], a["o2"] = np.full(n, 0x7F7F7F7F, dtype=np.int32), np.full(n, 0x7F7F7F7F, dtype=np.int32)
    if kind in ("dict", "dict_empty", "lz4f_dict"):
        a.update(db=inp.dsrc, dof=inp.doff, dl=inp.dlen if kind != "dict_empty" else np.zeros(n, dtype=np.int32))
    if mem == "device":
        t = {k: torch.from_numpy(v).cuda() for k, v in a.items()}
        p = {k: x.data_ptr() for k, x in t.items()}
    else:
        t, p = a, {k: v.ctypes.data for k, v in a.items()}
    src, dst, dic = (p["src"], p["so"], p["sl"]), (p["dst"], p["do"], p["dc"]), (p.get("db"), p.get("dof"), p.get("dl"))
    outs = [p[k] for k in ("o0", "o1", "o2") if k in p]
    call = (N.MEM_DEVICE if mem == "device" else N.MEM_HOST, None, -1)
    s0, before = decode_stats(L), L.k4lz4_launch_count()
    if kind == "frame":
        rc = L.k4lz4_frame_decode_batch(*src, *dst, *outs, n, *call)
    elif kind.startswith("dict"):
        rc = L.k4lz4_frame_decode_dict_batch(*src, *dst, *dic, *outs, n, *call)
    elif kind == "lz4f_size":
        rc = L.k4lz4_lz4f_decompressed_size_batch(*src, *outs, n, *call)
    elif kind.startswith("lz4f"):
        rc = L.k4lz4_lz4f_decompress_batch(*src, *dst, *dic, *outs, n, *call)
    elif kind == "content_size":
        rc = L.k4lz4_frame_content_size_batch(*src, *outs, n, *call)
    else:
        rc = L.k4lz4_frame_info_batch(*src, *outs, n, *call)
    launches = L.k4lz4_launch_count() - before
    if mem == "device":
        torch.cuda.synchronize()
        t = {k: x.cpu().numpy() for k, x in t.items() if k == "dst" or k.startswith("o")}
    return rc, t["dst"], [t[k] for k in ("o0", "o1", "o2") if k in t], launches, decode_stats(L) - s0


def host_chunks(inp, sized: bool) -> int:
    """The chunks frame_host stages a host call of inp in (a size call has no destinations, dictionaries ignored)."""
    a16 = lambda x: (int(x) + 15) & ~15              # noqa: E731
    chunks, used = 0, None
    for i in range(inp.n):
        add = a16(inp.sl[i]) + (0 if sized else 2 * a16(max(int(inp.dc[i]), 0))) + 64
        if used is None or used + add > STAGE_BYTES:
            chunks, used = chunks + 1, 0
        used += add
    return chunks


def decode_sets(A, written):
    """The decode part's inputs: name -> list of (input, dictionary)."""
    import oracle
    from tests import frame_dict_ref as FD
    from tests import lz4f_dec_ref as DR
    port = oracle.Port()
    u8 = lambda b: np.frombuffer(bytes(b), dtype=np.uint8)      # noqa: E731
    sets = {"encoded": written,
            "lz4f_grid": [(u8(x), u8(d if d is not None else b"")) for _, x, d in DR.grid()]}
    up = FD.FrameDictUpstream()
    sets["dict_grid"] = [(u8(up.cdict_frame(x, d, bs, linked, bc, cc, i)), u8(d))
                         for x, d, bs, linked, bc, cc, i in FD.grid()]
    # a truncated reference frame larger than its destination: K4LZ4_R_CORRUPT (its first error, the truncation),
    # never K4LZ4_R_DST_SMALL
    content = np.asarray(port.datagen(600000, 0.63, 0.0, 4711), dtype=np.uint8)
    cap = int(A.k4lz4_frame_bound(len(content), 65536, 0))
    inp = Inputs([content], [cap])
    _, da, oa, _ = call(A, "writer", inp, "host", 65536, 0)
    frame = da[inp.do[0]:inp.do[0] + oa[0]]
    sets["trap"] = [(frame[:len(frame) * 2 // 3], np.zeros(0, np.uint8)), (frame, np.zeros(0, np.uint8))]
    return sets


def decode_equality(A, B, emit, written) -> bool:
    """Part 2: every decode call on both builds with the same inputs, in host and device memory."""
    ok, counts = True, {}
    for name, items in decode_sets(A, written).items():
        frames, dicts = [x for x, _ in items], [d for _, d in items]
        n = len(frames)
        sized = Inputs(frames, [0] * n, dicts)
        content = {}
        for reader, kind in (("ref", "info"), ("lz4f", "lz4f_size")):
            _, _, o, _, _ = dcall(A, kind, sized, "host")
            content[reader] = [int(c) if c >= 0 else 65536 for c in o[0]]
        emit({"decode_set": name, "inputs": n, "bytes": int(sum(len(f) for f in frames))})

        def runs():
            for kind in SIZES:
                yield kind, sized, None
            for rot in range(5):  # entry i gets destination (i + rot) % 5: content, - 1, half, 10 B, + 64 KiB
                for kind in DECODES:
                    c = content["lz4f" if kind.startswith("lz4f") else "ref"]
                    caps = [max([c[i], c[i] - 1, c[i] // 2, 10, c[i] + 65536][(i + rot) % 5], 0) for i in range(n)]
                    yield kind, Inputs(frames, caps, dicts), rot

        for kind, inp, rot in runs():
            for mem in ("host", "device"):
                ra, da, oa, la, sa = dcall(A, kind, inp, mem)
                rb, db, ob, lb, sb = dcall(B, kind, inp, mem)
                chunks = host_chunks(inp, kind in SIZES) if mem == "host" else 1
                same = ra == rb and np.array_equal(da, db) and all(np.array_equal(x, y) for x, y in zip(oa, ob))
                good = same and np.array_equal(sa, sb) and la - lb == (chunks if kind == "info" else 0)
                ok &= good
                c = counts.setdefault((name, kind, mem), [0, 0, 0, 0])
                c[0] += 1
                c[1] += la
                c[2] += lb
                c[3] = max(c[3], chunks)
                if not good:
                    emit({"decode_mismatch": [name, kind, mem, rot], "rc": [ra, rb], "launches": [la, lb],
                          "bytes_equal": bool(np.array_equal(da, db)), "stats": [sa.tolist(), sb.tolist()],
                          "results_equal": [bool(np.array_equal(x, y)) for x, y in zip(oa, ob)]})
                if name == "trap" and kind == "frame":
                    ok &= bool(oa[0][0] == -1000)
                    emit({"trap": "truncated reference frame larger than its destination", "mem": mem,
                          "dst_cap": int(inp.dc[0]), "out_a": int(oa[0][0]), "out_b": int(ob[0][0])})
    for (name, kind, mem), (calls, la, lb, chunks) in counts.items():
        emit({"decode_launches": [name, kind, mem], "calls": calls, "a_total": int(la), "b_total": int(lb),
              "host_chunks": chunks})
    emit({"decode_all_identical": bool(ok)})
    return ok


def timing(A, B, reps: int, emit, only=None) -> None:
    import torch
    import oracle
    from k4os.compression.lz4_b200 import _native as N
    port = oracle.Port()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    base = [np.asarray(port.datagen(MB, 0.63, 0.0, 1000 + i), dtype=np.uint8) for i in range(64)]
    dic = np.asarray(port.datagen(65536, 0.63, 0.0, 4242), dtype=np.uint8)

    def race(label, fa, fb, nbytes, same):
        """Times fa and fb, alternating AB / BA rep by rep, after one warm-up call each."""
        arms = {"a": fa, "b": fb}
        for f in arms.values():
            f()
        torch.cuda.synchronize()
        ts = {k: [] for k in arms}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for r in range(reps):
            for k in ("ab" if r % 2 == 0 else "ba"):
                f = arms[k]
                ev[0].record(); f(); ev[1].record(); torch.cuda.synchronize()
                ts[k].append(ev[0].elapsed_time(ev[1]) / 1e3)
        best = {k: min(v) for k, v in ts.items()}
        med = {k: float(np.median(v)) for k, v in ts.items()}
        emit({"workload": label, "a_ms": round(best["a"] * 1e3, 3), "b_ms": round(best["b"] * 1e3, 3),
              "a_median_ms": round(med["a"] * 1e3, 3), "b_median_ms": round(med["b"] * 1e3, 3),
              "b_over_a_best": round(best["b"] / best["a"], 4), "b_over_a_median": round(med["b"] / med["a"], 4),
              "a_spread": round(max(ts["a"]) / best["a"] - 1, 4), "b_spread": round(max(ts["b"]) / best["b"] - 1, 4),
              "GBps_b": round(nbytes / best["b"] / 1e9, 2), "identical": bool(same())})

    def dworkload(kind, frames, contents, label, dictionary=False):
        """Decode: the inputs `frames` (host bytes, one per input) of contents `contents` bytes, into destinations of
        exactly that size, by reader `kind`: frame (k4lz4_frame_decode_batch), dict (_decode_dict_batch against the
        64 KiB dictionary) or lz4f (k4lz4_lz4f_decompress_batch)."""
        if only and only not in label:
            return
        S = len(frames)
        src = torch.from_numpy(np.concatenate(frames)).to(dev)
        so = torch.tensor(np.concatenate([[0], np.cumsum([len(f) for f in frames])[:-1]]), dtype=torch.int64,
                          device=dev)
        sl = torch.tensor([len(f) for f in frames], dtype=torch.int32, device=dev)
        dc = torch.tensor(contents, dtype=torch.int32, device=dev)
        do = torch.tensor(np.concatenate([[0], np.cumsum(contents)[:-1]]), dtype=torch.int64, device=dev)
        dst = {k: torch.zeros(sum(contents), dtype=torch.uint8, device=dev) for k in "ab"}
        out = {k: torch.zeros(3, S, dtype=torch.int32, device=dev) for k in "ab"}
        dsrc = torch.from_numpy(dic).to(dev)
        doff = torch.zeros(S, dtype=torch.int64, device=dev)
        dlen = torch.full((S,), len(dic), dtype=torch.int32, device=dev)
        d = [dsrc.data_ptr(), doff.data_ptr(), dlen.data_ptr()] if dictionary else [None] * 3

        def fn(L, k):
            p = [src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst[k].data_ptr(), do.data_ptr(), dc.data_ptr()]
            o = [out[k][j].data_ptr() for j in range(3)]
            if kind == "frame":
                rc = L.k4lz4_frame_decode_batch(*p, o[0], S, N.MEM_DEVICE, st, -1)
            elif kind == "dict":
                rc = L.k4lz4_frame_decode_dict_batch(*p, *d, o[0], S, N.MEM_DEVICE, st, -1)
            else:
                rc = L.k4lz4_lz4f_decompress_batch(*p, *d, *o, S, N.MEM_DEVICE, st, -1)
            assert rc == 0, rc

        want = torch.tensor(contents, dtype=torch.int32, device=dev)
        race(label, lambda: fn(A, "a"), lambda: fn(B, "b"), sum(contents), lambda: torch.equal(out["a"], out["b"]) and
             torch.equal(dst["a"], dst["b"]) and torch.equal(out["a"][0], want))

    def encoded(kind, content, sizes, bs, fl):
        """The frames A's `kind` encoder writes of `sizes`, in host memory; cdict: against the 64 KiB dictionary."""
        inp = Inputs([content[o:o + n] for o, n in zip(np.concatenate([[0], np.cumsum(sizes)[:-1]]), sizes)],
                     [int(A.k4lz4_lz4f_compress_bound(n, bs, fl)) if kind == "lz4f" else
                      int(A.k4lz4_frame_bound(n, bs, fl)) for n in sizes])
        if kind == "cdict":
            inp.dicts, inp.dsrc = True, dic
            inp.doff, inp.dlen = np.zeros(inp.n, np.int64), np.full(inp.n, len(dic), np.int32)
        rc, da, oa, _ = call(A, kind, inp, "host", bs, fl)
        assert rc == 0 and (oa > 0).all(), rc
        return [da[o:o + n] for o, n in zip(inp.do, oa)]

    def workload(kind, content, sizes, bs, fl, label):
        if only and only not in label:
            return
        S = len(sizes)
        src = torch.from_numpy(content).to(dev)
        so = torch.tensor(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=torch.int64, device=dev)
        sl = torch.tensor(sizes, dtype=torch.int32, device=dev)
        caps = [int(A.k4lz4_lz4f_compress_bound(n, bs, fl)) if kind == "lz4f" else int(A.k4lz4_frame_bound(n, bs, fl))
                for n in sizes]
        dc = torch.tensor(caps, dtype=torch.int32, device=dev)
        do = torch.tensor(np.concatenate([[0], np.cumsum(caps)[:-1]]), dtype=torch.int64, device=dev)
        dst = {k: torch.zeros(sum(caps), dtype=torch.uint8, device=dev) for k in "ab"}
        out = {k: torch.zeros(S, dtype=torch.int32, device=dev) for k in "ab"}
        dsrc = torch.from_numpy(dic).to(dev)
        doff = torch.zeros(S, dtype=torch.int64, device=dev)
        dlen = torch.full((S,), len(dic), dtype=torch.int32, device=dev)

        def fn(L, k):
            p = [src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst[k].data_ptr(), do.data_ptr(), dc.data_ptr()]
            if kind == "writer":
                rc = L.k4lz4_frame_encode_batch(*p, out[k].data_ptr(), S, bs, fl, 0, N.MEM_DEVICE, st, -1)
            elif kind == "cdict":
                rc = L.k4lz4_frame_encode_dict_batch(*p, dsrc.data_ptr(), doff.data_ptr(), dlen.data_ptr(), None,
                                                     out[k].data_ptr(), S, bs, fl, 0, N.MEM_DEVICE, st, -1)
            else:
                rc = L.k4lz4_lz4f_compress_batch(*p, out[k].data_ptr(), S, bs, fl, 0, N.MEM_DEVICE, st, -1)
            assert rc == 0, rc

        race(label, lambda: fn(A, "a"), lambda: fn(B, "b"), sum(sizes), lambda: torch.equal(out["a"], out["b"]) and
             torch.equal(dst["a"], dst["b"]) and bool((out["a"] > 0).all()))

    readers = {"writer": ("frame", False), "cdict": ("dict", True), "lz4f": ("lz4f", False)}
    for S in (264, 1024):
        content = np.concatenate([base[i % 64] for i in range(S)])
        for linked in (True, False):
            fl = 0 if linked else N.FRAME_INDEPENDENT
            mode = "linked" if linked else "indep"
            for kind in ("writer", "cdict", "lz4f"):
                workload(kind, content, [MB] * S, 65536, fl, f"{kind} {S} x 1 MiB, 64 KiB blocks, {mode}")
                reader, withd = readers[kind]
                label = f"decode {reader} {S} x 1 MiB, 64 KiB blocks, {mode}"
                if not only or only in label:
                    dworkload(reader, encoded(kind, content, [MB] * S, 65536, fl), [MB] * S, label, withd)
    content = np.concatenate([base[i % 64] for i in range(1024)])
    workload("lz4f", content, [MB] * 1024, 1 << 22, 0, "lz4f 1024 x 1 MiB, 4 MiB blocks")
    for kind in ("writer", "lz4f"):
        label = f"decode {readers[kind][0]} 1024 x 1 MiB, 4 MiB blocks"
        if not only or only in label:
            dworkload(readers[kind][0], encoded(kind, content, [MB] * 1024, 1 << 22, 0), [MB] * 1024, label)
    # lz4f streams of 16 concatenated 64 KiB frames, and legacy streams (lz4 -l) of one 4 MiB block
    label = "decode lz4f 1024 streams of 16 x 64 KiB frames"
    if not only or only in label:
        fr16 = encoded("lz4f", content, [65536] * (16 * 1024), 65536, 0)
        dworkload("lz4f", [np.concatenate(fr16[i:i + 16]) for i in range(0, len(fr16), 16)], [16 * 65536] * 1024,
                  label)
    label = "decode lz4f 256 legacy streams of 4 MiB"
    if not only or only in label:
        from tests import lz4f_dec_ref as DR
        from tests import lz4f_ref as LR
        up = LR.Lz4fUpstream()
        legs = [np.frombuffer(DR.legacy(up, content[i * 4 * MB:(i + 1) * 4 * MB].tobytes()), dtype=np.uint8)
                for i in range(256)]
        dworkload("lz4f", legs, [4 * MB] * 256, label)
    # dfbench (a): record-like messages of 256 B .. 4 KiB, one independent frame each, against the dictionary
    rng = np.random.default_rng(1)
    sizes = rng.integers(256, 4097, 200_000).tolist()
    big = np.concatenate([base[i % 64] for i in range(1024)])
    offs = rng.integers(0, len(big) - 4096, len(sizes))
    msgs = np.concatenate([big[o:o + n] for o, n in zip(offs, sizes)])
    for kind in ("writer", "cdict", "lz4f"):
        workload(kind, msgs, sizes, 65536, N.FRAME_INDEPENDENT, f"{kind} 200000 messages of 256 B - 4 KiB, indep")
    label = "decode dict 200000 messages of 256 B - 4 KiB, indep"
    if not only or only in label:
        dworkload("dict", encoded("cdict", msgs, sizes, 65536, N.FRAME_INDEPENDENT), sizes, label, True)
    small = [base[i % 64][(i * 4096) % MB:][:4096] for i in range(10000)]
    big40 = np.concatenate([base[i % 64] for i in range(40)])
    items = small + [big40]
    workload("lz4f", np.concatenate(items), [len(x) for x in items], 1 << 22, 0,
             "lz4f mixed: 10000 x 4 KiB + 1 x 40 MiB linked, 4 MiB blocks")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="the baseline build of libk4lz4.so")
    ap.add_argument("--b", default=None, help="the build under test (default: the tree's)")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from k4os.compression.lz4_b200 import _native as N
    A, B = load(a.a), load(a.b or N.SO_PATH)
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    emit({"card": card()})
    written = []
    ok = a.only is not None or (equality(A, B, emit, written) & decode_equality(A, B, emit, written))
    timing(A, B, a.reps, emit, a.only)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "frame_ab.jsonl"), "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
