"""Reading benchmark: .lz4 streams through k4lz4_lz4f_decompress_batch (upstream's `lz4 -d` rules: member walk, then
the frame machinery over members) against k4lz4_frame_decode_batch (the reference's reader, one frame per entry) on the
same frames, in device memory, the two arms alternating rep by rep, timed with CUDA events.  Every output of every rep
is checked against the content.

Rows:
  * S streams of one upstream frame of 1 MiB of reference datagen 0.63, 64 KiB and 4 MiB blocks, both arms;
  * the same content as streams of 16 concatenated 64 KiB frames, and as legacy streams (new call only);
  * one stream of 1 GiB as 16 384 concatenated 64 KiB frames (the serial member walk shows here);

    python tools/lz4fdbench.py [--sizes 264,1024,4096] [--reps 7] [--big 1]

Prints the card name and power limit, then one JSON line per row: best and median ms per arm, the ratio of medians,
GB/s of content at the best time."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fbench import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="264,1024,4096")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--big", type=int, default=1)
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import _native as N
    from tests import lz4f_ref as R, lz4f_dec_ref as M
    print("card:", card(), flush=True)
    MB = 1 << 20
    port = oracle.Port()
    up = R.Lz4fUpstream()
    base = [port.datagen(MB, 0.63, 0.0, 1000 + i).tobytes() for i in range(16)]
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream()
    lib = N.lib()

    def setup(streams, content_len, n):
        lens = np.array([len(s) for s in streams], dtype=np.int32)
        so = np.zeros(n, dtype=np.int64)
        so[1:] = np.cumsum(lens[:-1], dtype=np.int64)
        src = torch.from_numpy(np.frombuffer(b"".join(streams), dtype=np.uint8).copy()).to(dev)
        do = torch.arange(n, dtype=torch.int64, device=dev) * content_len
        return dict(src=src, so=torch.from_numpy(so).to(dev), sl=torch.from_numpy(lens).to(dev),
                    dst=torch.zeros(n * content_len, dtype=torch.uint8, device=dev), do=do,
                    dc=torch.full((n,), content_len, dtype=torch.int32, device=dev),
                    out=torch.zeros(n, dtype=torch.int32, device=dev),
                    err=torch.zeros(n, dtype=torch.int32, device=dev),
                    end=torch.zeros(n, dtype=torch.int32, device=dev), n=n)

    def new(b):
        N.check(lib.k4lz4_lz4f_decompress_batch(
            b["src"].data_ptr(), b["so"].data_ptr(), b["sl"].data_ptr(), b["dst"].data_ptr(), b["do"].data_ptr(),
            b["dc"].data_ptr(), None, None, None, b["out"].data_ptr(), b["err"].data_ptr(), b["end"].data_ptr(),
            b["n"], N.MEM_DEVICE, st.cuda_stream, -1))

    def old(b):
        N.check(lib.k4lz4_frame_decode_batch(
            b["src"].data_ptr(), b["so"].data_ptr(), b["sl"].data_ptr(), b["dst"].data_ptr(), b["do"].data_ptr(),
            b["dc"].data_ptr(), b["out"].data_ptr(), b["n"], N.MEM_DEVICE, st.cuda_stream, -1))

    def timed(fn, b, expect, content_len):
        b["dst"].zero_()
        b["out"].fill_(-7)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn(b)
        e1.record(st)
        torch.cuda.synchronize()
        assert bool((b["out"] == content_len).all()), "result"
        assert torch.equal(b["dst"], expect), "content"
        return e0.elapsed_time(e1)

    def row(name, arms, n, content_len, expect):
        times = {k: [] for k in arms}
        for k, (fn, b) in arms.items():          # warm-up
            timed(fn, b, expect, content_len)
        for r in range(a.reps):
            order = list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]
            for k, (fn, b) in order:
                times[k].append(timed(fn, b, expect, content_len))
        res = {"row": name, "streams": n, "content_MiB": n * content_len / MB}
        for k, t in times.items():
            res[f"{k}_best_ms"] = round(min(t), 3)
            res[f"{k}_median_ms"] = round(float(np.median(t)), 3)
            res[f"{k}_GBps"] = round(n * content_len / min(t) / 1e6, 1)
        if len(times) == 2:
            res["new_over_ref_median"] = round(float(np.median(times["lz4f"]) / np.median(times["ref"])), 4)
        print(json.dumps(res), flush=True)

    for S in [int(x) for x in a.sizes.split(",")]:
        content = [base[i % 16] for i in range(S)]
        expect = torch.from_numpy(np.frombuffer(b"".join(content), dtype=np.uint8).copy()).to(dev)
        for bs in (1 << 16, 1 << 22):
            frames = {i: up.frame(base[i], bs, R.flags_of(True, False, True, False)) for i in range(16)}
            b = setup([frames[i % 16] for i in range(S)], MB, S)
            row(f"one-frame/{bs >> 10}K", {"lz4f": (new, b), "ref": (old, b)}, S, MB, expect)
        cat = {i: b"".join(up.frame(base[i][o:o + (1 << 16)], 1 << 16, R.flags_of(True, False, True, False))
                           for o in range(0, MB, 1 << 16)) for i in range(16)}
        b = setup([cat[i % 16] for i in range(S)], MB, S)
        row("16-frames/64K", {"lz4f": (new, b)}, S, MB, expect)
        leg = {i: M.legacy(up, base[i]) for i in range(16)}
        b = setup([leg[i % 16] for i in range(S)], MB, S)
        row("legacy", {"lz4f": (new, b)}, S, MB, expect)
        del b, expect
        torch.cuda.empty_cache()
    if a.big:
        one = b"".join(up.frame(base[i % 16][(i // 16 % 16) << 16:((i // 16 % 16) + 1) << 16], 1 << 16,
                                R.flags_of(True, False, False, False)) for i in range(16 * 16))
        total = 1 << 30
        stream = one * (total // (16 * MB))
        content = b"".join(base[i % 16][(i // 16 % 16) << 16:((i // 16 % 16) + 1) << 16] for i in range(256))
        expect = torch.from_numpy(np.frombuffer(content, dtype=np.uint8).copy()).to(dev).repeat(total // (16 * MB))
        b = setup([stream], total, 1)

        def timed_big(fn, bb, ex, cl):
            bb["out"].fill_(-7)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            fn(bb)
            e1.record(st)
            torch.cuda.synchronize()
            assert int(bb["out"][0]) == total and torch.equal(bb["dst"], ex), "1 GiB stream"
            return e0.elapsed_time(e1)
        ts = [timed_big(new, b, expect, total) for _ in range(max(3, a.reps // 2))]
        print(json.dumps({"row": "one-stream/1GiB/16384-frames", "lz4f_best_ms": round(min(ts), 3),
                          "lz4f_median_ms": round(float(np.median(ts)), 3),
                          "lz4f_GBps": round(total / min(ts) / 1e6, 1)}), flush=True)


if __name__ == "__main__":
    main()
