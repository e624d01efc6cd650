"""Frame reader group throughput: S streams, each reading one frame of 1 MiB of reference datagen 0.63 in 64 KiB
blocks (linked / independent, without / with both checksums), fed in chunks of W bytes with dstCap = 16 x blockCap,
in device and host memory, against one k4lz4_frame_decode_batch over the same frames in the same memory kind.
Every stream's content is checked in the run.  Prints one JSON line per configuration (GB/s of content, best of
--reps) and the card, power limit and maximum SM clock read in the same run.  --cap adds byte reads
(k4lz4_frame_reader_group_read_bytes) at those dstCaps ("16b": 16 x blockCap; --interactive: interactive mode),
beside the plain reads at 16 x blockCap."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="264,1024,4096")
    ap.add_argument("--chunks", default="4096,65536,1048576")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cap", default="", help="byte reads at these dstCaps, e.g. 4096,65536,16b")
    ap.add_argument("--interactive", action="store_true")
    a = ap.parse_args()
    import torch
    import oracle
    import k4os.compression.lz4_b200 as k4
    N = k4._native
    L = N.lib()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": q}), flush=True)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    data = oracle.Port().datagen(1 << 20, 0.63, 0.0, 1234).tobytes()
    for fl in (0, 6, 1, 7):
        fr, _ = k4.LZ4Frame.EncodeMany([data], 65536, not fl & 1, bool(fl & 2), bool(fl & 4))
        f = fr[0]
        cap_b = 65536 + (8 if fl & 1 else 0)
        for S in [int(x) for x in a.streams.split(",")]:
            blob = np.frombuffer(f * S, np.uint8)
            flen = len(f)
            d_src = torch.from_numpy(blob.copy()).to(dev)
            d_dst = torch.zeros(S << 20, dtype=torch.uint8, device=dev)
            offs = torch.arange(S, dtype=torch.int64, device=dev)
            base = {}
            # whole-frame decode, device and host
            so, sl = offs * flen, torch.full((S,), flen, dtype=torch.int32, device=dev)
            do, dc = offs << 20, torch.full((S,), 1 << 20, dtype=torch.int32, device=dev)
            ol = torch.zeros(S, dtype=torch.int32, device=dev)
            h_so, h_sl, h_do, h_dc = (x.cpu().numpy() for x in (so, sl, do, dc))
            h_dst = np.zeros(S << 20, np.uint8)
            h_ol = np.zeros(S, np.int32)

            def whole(mem):
                if mem == "device":
                    N.check(L.k4lz4_frame_decode_batch(d_src.data_ptr(), so.data_ptr(), sl.data_ptr(), d_dst.data_ptr(),
                                                       do.data_ptr(), dc.data_ptr(), ol.data_ptr(), S, N.MEM_DEVICE,
                                                       st, 0))
                    torch.cuda.synchronize()
                else:
                    N.check(L.k4lz4_frame_decode_batch(blob.ctypes.data, h_so.ctypes.data, h_sl.ctypes.data,
                                                       h_dst.ctypes.data, h_do.ctypes.data, h_dc.ctypes.data,
                                                       h_ol.ctypes.data, S, N.MEM_HOST, None, 0))

            def check(mem):
                out = d_dst.cpu().numpy() if mem == "device" else h_dst
                for s in range(0, S, max(S // 64, 1)):
                    assert out[s << 20:(s + 1) << 20].tobytes() == data, s
                assert np.array_equal(out.reshape(S, -1), np.broadcast_to(out[:1 << 20], (S, 1 << 20)))

            for mem in ("device", "host"):
                best = 1e9
                for r in range(a.reps + 1):
                    (d_dst.zero_() if mem == "device" else h_dst.fill(0))
                    t = time.perf_counter(); whole(mem); dt = time.perf_counter() - t
                    if r:
                        best = min(best, dt)
                check(mem)
                base[mem] = S * len(data) / best / 1e9
            arms = [("read", 16 * cap_b)] + [("read_bytes", 16 * cap_b if c == "16b" else int(c))
                                              for c in a.cap.split(",") if c]
            for W, mem, (arm, cap) in ((w, m, x) for w in [int(x) for x in a.chunks.split(",")]
                                       for m in ("device", "host") for x in arms):
                byte = arm == "read_bytes"
                g = k4.FrameReaderGroup(S, 65536)
                streams = torch.arange(S, dtype=torch.int32, device=dev)
                h_streams = streams.cpu().numpy()
                dcap = torch.full((S,), cap, dtype=torch.int32, device=dev)
                h_dcap = dcap.cpu().numpy()
                best = 1e9
                for r in range(a.reps + 1):
                    g.reset()
                    (d_dst.zero_() if mem == "device" else h_dst.fill(0))
                    at = np.zeros(S, np.int64)
                    wr = np.zeros(S, np.int64)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    done = np.zeros(S, bool)
                    while not done.all() if byte else (at < flen).any():
                        ln = np.minimum(flen - at, W).astype(np.int32)
                        soff = np.arange(S, dtype=np.int64) * flen + at
                        doff = (np.arange(S, dtype=np.int64) << 20) + wr
                        used = np.zeros(S, np.int32); outl = np.zeros(S, np.int32); end = np.zeros(S, np.int32)
                        if mem == "device":
                            t_so, t_sl, t_do = (torch.from_numpy(x).to(dev) for x in (soff, ln, doff))
                            t_u, t_o, t_e = (torch.zeros(S, dtype=torch.int32, device=dev) for _ in range(3))
                            p = [streams.data_ptr(), d_src.data_ptr(), t_so.data_ptr(), t_sl.data_ptr(),
                                 t_u.data_ptr(), d_dst.data_ptr(), t_do.data_ptr(), dcap.data_ptr(),
                                 t_o.data_ptr(), t_e.data_ptr(), S]
                            if byte:
                                g.read_bytes_device(*p, interactive=a.interactive, stream=st)
                            else:
                                g.read_device(*p, st)
                            used, outl, end = t_u.cpu().numpy(), t_o.cpu().numpy(), t_e.cpu().numpy()
                        else:
                            p = [g.handle, h_streams.ctypes.data, blob.ctypes.data, soff.ctypes.data, ln.ctypes.data,
                                 used.ctypes.data, h_dst.ctypes.data, doff.ctypes.data, h_dcap.ctypes.data,
                                 outl.ctypes.data, end.ctypes.data, S]
                            if byte:
                                N.check(L.k4lz4_frame_reader_group_read_bytes(
                                *p, N.READ_INTERACTIVE if a.interactive else 0, N.MEM_HOST, None))
                            else:
                                N.check(L.k4lz4_frame_reader_group_read(*p, N.MEM_HOST, None))
                        assert (outl >= 0).all()
                        at += used
                        wr += outl
                        done |= end == 1
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t
                    if r:
                        best = min(best, dt)
                assert (wr == len(data)).all() and (g.end() == 0).all()
                check(mem)
                g.free()
                gbs = S * len(data) / best / 1e9
                print(json.dumps({"flags": fl, "S": S, "W": W, "mem": mem, "arm": arm, "cap": cap,
                                  "interactive": bool(byte and a.interactive), "reader_GBps": round(gbs, 2),
                                  "frame_decode_GBps": round(base[mem], 2)}), flush=True)


if __name__ == "__main__":
    main()
