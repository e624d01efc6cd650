"""Frame writer benchmark: S streams, each writing 1 MiB of reference datagen 0.63 into a frame writer group
(k4lz4_frame_writer_group_write, then _close) in writes of W bytes, with 64 KiB linked or independent blocks, in
device and host memory, against one k4lz4_frame_encode_batch call over the same contents in the same memory kind.
The gap is the cost of writing incrementally: per-call launches, the one step-count wait per write, and moving
the partial blocks through the rings.  Every stream's concatenated output is checked equal to the frame call's.

    python tools/wbench.py [--sizes 264,1024,4096] [--writes 4096,65536,1048576] [--reps 3]

Prints the card name, power limit and max SM clock, then one JSON line per (S, mode, memory, W) with GB/s of
content."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> str:
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def timed(fn, reps: int) -> float:
    import torch
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="264,1024,4096")
    ap.add_argument("--writes", default="4096,65536,1048576")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-max", type=int, default=1024, help="largest S also run in host memory")
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import FrameWriterGroup, LZ4Frame, _native as N
    print("card:", card(), flush=True)
    MB, BS = 1 << 20, 1 << 16
    port = oracle.Port()
    base = [port.datagen(MB, 0.63, 0.0, 1000 + i) for i in range(64)]
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    L = N.lib()
    for S in [int(x) for x in a.sizes.split(",")]:
        host = np.concatenate([base[i % 64] for i in range(S)])
        src = torch.from_numpy(host).to(dev)
        so = torch.arange(S, dtype=torch.int64, device=dev) * MB
        sl = torch.full((S,), MB, dtype=torch.int32, device=dev)
        streams = torch.arange(S, dtype=torch.int32, device=dev)
        h_streams = np.arange(S, dtype=np.int32)
        for chaining in (True, False):
            mode = "linked" if chaining else "independent"
            fl = 0 if chaining else N.FRAME_INDEPENDENT
            fb = int(L.k4lz4_frame_bound(MB, BS, fl))
            fdst = torch.zeros(S * fb, dtype=torch.uint8, device=dev)
            fdo = torch.arange(S, dtype=torch.int64, device=dev) * fb
            fdc = torch.full((S,), fb, dtype=torch.int32, device=dev)
            fol = torch.zeros(S, dtype=torch.int32, device=dev)
            t_frame = timed(lambda: LZ4Frame.encode_many_device(src, so, sl, fdst, fdo, fdc, fol, BS, chaining,
                                                                stream=st), a.reps)
            want = [fdst[i * fb:i * fb + int(n)] for i, n in enumerate(fol.cpu().tolist())]
            h_frame = None
            with FrameWriterGroup(S, BS, chaining=chaining) as g:
                cb = g.close_bound()
                for W in [int(x) for x in a.writes.split(",")]:
                    wb = g.bound(W)
                    region = (fb + wb + 15) // 16 * 16
                    dst = torch.zeros(S * region, dtype=torch.uint8, device=dev)
                    start = torch.arange(S, dtype=torch.int64, device=dev) * region
                    pos = start.clone()
                    cap = torch.full((S,), wb, dtype=torch.int32, device=dev)
                    ccap = torch.full((S,), cb, dtype=torch.int32, device=dev)
                    wl = torch.full((S,), W, dtype=torch.int32, device=dev)
                    offs = [so + k * W for k in range(MB // W)]
                    ol = torch.zeros(S, dtype=torch.int32, device=dev)

                    def run_dev():
                        pos.copy_(start)
                        for o in offs:
                            g.write_device(streams.data_ptr(), src.data_ptr(), o.data_ptr(), wl.data_ptr(),
                                           dst.data_ptr(), pos.data_ptr(), cap.data_ptr(), ol.data_ptr(), S, stream=st)
                            pos.add_(ol)
                        g.close_device(streams.data_ptr(), dst.data_ptr(), pos.data_ptr(), ccap.data_ptr(),
                                       ol.data_ptr(), S, stream=st)
                        pos.add_(ol)
                    t_w = timed(run_dev, a.reps)
                    ends = (pos - start).cpu().tolist()
                    for i in range(S):
                        assert torch.equal(dst[i * region:i * region + ends[i]], want[i]), (S, mode, W, i)
                    gb = S * MB / 1e9
                    print(json.dumps({"S": S, "mode": mode, "mem": "device", "write": W,
                                      "writer_GBps": round(gb / t_w, 2), "frame_call_GBps": round(gb / t_frame, 2),
                                      "calls": len(offs) + 1}), flush=True)
                    del dst
                    if S > a.host_max:
                        continue
                    # host memory: the same writes on host buffers through the C ABI
                    hdst = np.zeros(S * region, dtype=np.uint8)
                    hstart = np.arange(S, dtype=np.int64) * region
                    hpos = hstart.copy()
                    hcap = np.full(S, wb, dtype=np.int32)
                    hccap = np.full(S, cb, dtype=np.int32)
                    hwl = np.full(S, W, dtype=np.int32)
                    hoffs = [np.arange(S, dtype=np.int64) * MB + k * W for k in range(MB // W)]
                    hol = np.zeros(S, dtype=np.int32)

                    def run_host():
                        hpos[:] = hstart
                        for o in hoffs:
                            N.check(L.k4lz4_frame_writer_group_write(g.handle, h_streams.ctypes.data, host.ctypes.data,
                                                                     o.ctypes.data, hwl.ctypes.data, hdst.ctypes.data,
                                                                     hpos.ctypes.data, hcap.ctypes.data,
                                                                     hol.ctypes.data, S, N.MEM_HOST, None))
                            hpos[:] += hol
                        N.check(L.k4lz4_frame_writer_group_close(g.handle, h_streams.ctypes.data, hdst.ctypes.data,
                                                                 hpos.ctypes.data, hccap.ctypes.data, hol.ctypes.data,
                                                                 S, N.MEM_HOST, None))
                        hpos[:] += hol
                    t_hw = timed(run_host, a.reps)
                    if h_frame is None:
                        hf = np.zeros(S * fb, dtype=np.uint8)
                        hfo = np.arange(S, dtype=np.int64) * fb
                        hfc = np.full(S, fb, dtype=np.int32)
                        hfl = np.zeros(S, dtype=np.int32)
                        hso = np.arange(S, dtype=np.int64) * MB
                        hsl = np.full(S, MB, dtype=np.int32)
                        h_frame = timed(lambda: N.check(L.k4lz4_frame_encode_batch(
                            host.ctypes.data, hso.ctypes.data, hsl.ctypes.data, hf.ctypes.data, hfo.ctypes.data,
                            hfc.ctypes.data, hfl.ctypes.data, S, BS, fl, 0, N.MEM_HOST, None, 0)), a.reps)
                    for i in range(0, S, 37):
                        assert hdst[hstart[i]:hpos[i]].tobytes() == want[i].cpu().numpy().tobytes(), (S, mode, W, i)
                    print(json.dumps({"S": S, "mode": mode, "mem": "host", "write": W,
                                      "writer_GBps": round(gb / t_hw, 2), "frame_call_GBps": round(gb / h_frame, 2),
                                      "calls": len(offs) + 1}), flush=True)
                    del hdst
            del fdst
            torch.cuda.empty_cache()
        del src


if __name__ == "__main__":
    main()
