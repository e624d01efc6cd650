"""Upstream-frame benchmark: S frames of 1 MiB of reference datagen 0.63 through k4lz4_lz4f_compress_batch
(upstream's LZ4F_compressFrame: capacity n - 1 per block, raw where that fails) against k4lz4_frame_encode_batch
(the reference's LZ4FrameWriter) on the same content in the same process, in device memory, the two arms alternating
rep by rep.  64 KiB blocks, linked and independent, and one row of 4 MiB-block frames (the lz4 CLI's default; a
1 MiB frame then shrinks to one 1 MiB independent block).  Every output is checked in the same run: the upstream
arm's frames equal LZ4F_compressFrame's on a sample, and both arms' frames decode back to their content.

    python tools/lz4fbench.py [--sizes 264,1024,4096] [--reps 15]

Prints the card name and power limit, then one JSON line per (S, block size, mode) with both arms' best time, the
ratio of their medians and each arm's spread (slowest rep over best), and one line for a mixed call; GB/s are of
content."""
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
    ap.add_argument("--reps", type=int, default=15)
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import LZ4F, LZ4Frame, _native as N
    from tests import lz4f_ref as R
    print("card:", card(), flush=True)
    MB = 1 << 20
    port = oracle.Port()
    base = [port.datagen(MB, 0.63, 0.0, 1000 + i) for i in range(64)]
    up = R.Lz4fUpstream()
    L = N.lib()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    rows = [(S, 1 << 16, linked) for S in (int(s) for s in a.sizes.split(",")) for linked in (True, False)]
    rows.append((1024, 1 << 22, True))
    for S, bs, linked in rows:
        content = np.concatenate([base[i % 64] for i in range(S)])
        src = torch.from_numpy(content).to(dev)
        so = torch.arange(S, dtype=torch.int64, device=dev) * MB
        sl = torch.full((S,), MB, dtype=torch.int32, device=dev)
        fl = 0 if linked else N.FRAME_INDEPENDENT
        cap = max(int(L.k4lz4_lz4f_compress_bound(MB, bs, fl)), int(L.k4lz4_frame_bound(MB, bs, fl)))
        dst = {k: torch.zeros(S * cap, dtype=torch.uint8, device=dev) for k in ("frame", "lz4f")}
        do = torch.arange(S, dtype=torch.int64, device=dev) * cap
        dc = torch.full((S,), cap, dtype=torch.int32, device=dev)
        out = {k: torch.zeros(S, dtype=torch.int32, device=dev) for k in ("frame", "lz4f")}
        arms = {
            "frame": lambda: N.check(L.k4lz4_frame_encode_batch(
                src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst["frame"].data_ptr(), do.data_ptr(), dc.data_ptr(),
                out["frame"].data_ptr(), S, bs, fl, 0, N.MEM_DEVICE, st, -1)),
            "lz4f": lambda: LZ4F.compress_many_device(src, so, sl, dst["lz4f"], do, dc, out["lz4f"], bs, linked,
                                                      stream=st),
        }
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
        ts = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, fn in arms.items():
                ts[k].append(timed_once(fn))
        best = {k: min(v) for k, v in ts.items()}
        # checks: both arms decode back; the upstream arm equals LZ4F_compressFrame on a sample
        ok = True
        for k in arms:
            lens = out[k].cpu().numpy()
            if (lens <= 0).any():
                ok = False
                continue
            d = dst[k].cpu().numpy()
            frames = [d[i * cap:i * cap + int(lens[i])].tobytes() for i in range(S)]
            pick = range(0, S, max(S // 16, 1))
            got, res = LZ4Frame.DecodeMany([frames[i] for i in pick])
            ok &= all(g == base[i % 64].tobytes() for g, i in zip(got, pick))
            if k == "lz4f":
                ok &= all(frames[i] == up.frame(base[i % 64].tobytes(), bs, fl) for i in list(pick)[:4])
        gb = S * MB / 1e9
        print(json.dumps({"S": S, "block": bs, "linked": linked, "frame_ms": round(best["frame"] * 1e3, 3),
                          "lz4f_ms": round(best["lz4f"] * 1e3, 3), "frame_GBps": round(gb / best["frame"], 2),
                          "lz4f_GBps": round(gb / best["lz4f"], 2),
                          "lz4f_over_frame": round(best["lz4f"] / best["frame"], 4),
                          "median_ratio": round(float(np.median(ts["lz4f"]) / np.median(ts["frame"])), 4),
                          "frame_spread": round(max(ts["frame"]) / best["frame"] - 1, 4),
                          "lz4f_spread": round(max(ts["lz4f"]) / best["lz4f"] - 1, 4), "checked": bool(ok)}), flush=True)
        del src, dst, out
    mixed(a.reps, base, up)


def timed_once(fn) -> float:
    import torch
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record(); fn(); ev[1].record(); torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / 1e3


def mixed(reps: int, base, up) -> None:
    """10 000 frames of 4 KiB beside one linked frame of 40 MiB, 4 MiB blocks, in one call: the linked steps run over
    the one linked frame, so the call costs what its two passes cost apart.  Reported: the mixed call, and the
    small frames and the large frame each in a call of their own."""
    import torch
    from k4os.compression.lz4_b200 import LZ4F, _native as N
    L = N.lib()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    big = np.concatenate([base[i % 64] for i in range(40)])
    small = [base[i % 64][(i * 4096) % (1 << 20):][:4096] for i in range(10000)]
    bs = 1 << 22

    def call(items):
        sizes = [len(x) for x in items]
        src = torch.from_numpy(np.concatenate(items)).to(dev)
        so = torch.tensor(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=torch.int64, device=dev)
        sl = torch.tensor(sizes, dtype=torch.int32, device=dev)
        caps = [int(L.k4lz4_lz4f_compress_bound(x, bs, 0)) for x in sizes]
        dst = torch.zeros(sum(caps), dtype=torch.uint8, device=dev)
        do = torch.tensor(np.concatenate([[0], np.cumsum(caps)[:-1]]), dtype=torch.int64, device=dev)
        dc = torch.tensor(caps, dtype=torch.int32, device=dev)
        out = torch.zeros(len(items), dtype=torch.int32, device=dev)
        fn = lambda: LZ4F.compress_many_device(src, so, sl, dst, do, dc, out, bs, stream=st)  # noqa: E731
        fn()
        torch.cuda.synchronize()
        before = L.k4lz4_launch_count()
        fn()
        torch.cuda.synchronize()
        launches = L.k4lz4_launch_count() - before
        ok = bool((out > 0).all())
        if ok and len(items) > 1:
            o, d, c = out.cpu().numpy(), dst.cpu().numpy(), do.cpu().numpy()
            ok = d[c[-1]:c[-1] + o[-1]].tobytes() == up.frame(items[-1].tobytes(), bs, 0)
        return min(timed_once(fn) for _ in range(reps)), launches, ok

    both, small_alone, big_alone = call(small + [big]), call(small), call([big])
    print(json.dumps({"mixed": "10000 x 4 KiB + 1 x 40 MiB linked, 4 MiB blocks", "mixed_ms": round(both[0] * 1e3, 3),
                      "mixed_launches": both[1], "small_alone_ms": round(small_alone[0] * 1e3, 3),
                      "big_alone_ms": round(big_alone[0] * 1e3, 3), "checked": both[2] and small_alone[2]
                      and big_alone[2]}), flush=True)


if __name__ == "__main__":
    main()
