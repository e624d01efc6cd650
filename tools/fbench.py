"""Frame-layer benchmark: S frames of 1 MiB of reference datagen 0.63 in the reference's default settings (64 KiB
linked blocks) and as independent frames, through k4lz4_frame_encode_batch / _decode_batch in device and host
memory, against the same blocks through the block calls (k4lz4_encode_chain_batch / k4lz4_decode_chain_batch one
step at a time for linked frames, k4lz4_encode_batch / k4lz4_decode_batch for independent ones).  The gap is the
cost of the frame layer: parse, size walk, layout, checksums.  Every output is checked in the same run: frames
decode back to their content, and the block calls' bytes equal the frames' blocks.

    python tools/fbench.py [--sizes 264,1024,4096] [--reps 5]

Prints the card name and power limit, then one JSON line per (S, mode, memory) with GB/s of content."""
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
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        pl = f"unknown ({e})"
    return f"{name}, power limit {pl}"


def timed(fn, reps: int) -> float:
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(reps):
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / 1e3)
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="264,1024,4096")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import LZ4Frame, _native as N, batch as B
    print("card:", card(), flush=True)
    MB, BS = 1 << 20, 1 << 16
    NB = MB // BS
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
        for chaining in (True, False):
            fl = 0 if chaining else N.FRAME_INDEPENDENT
            bound = int(L.k4lz4_frame_bound(MB, BS, fl))
            dst = torch.zeros(S * bound, dtype=torch.uint8, device=dev)
            do = torch.arange(S, dtype=torch.int64, device=dev) * bound
            dc = torch.full((S,), bound, dtype=torch.int32, device=dev)
            ol = torch.zeros(S, dtype=torch.int32, device=dev)
            enc = lambda: LZ4Frame.encode_many_device(src, so, sl, dst, do, dc, ol, BS, chaining, stream=st)  # noqa: E731
            t_fe = timed(enc, a.reps)
            assert bool((ol > 0).all())
            out = torch.zeros(S * MB, dtype=torch.uint8, device=dev)
            rl = torch.zeros(S, dtype=torch.int32, device=dev)
            dec = lambda: LZ4Frame.decode_many_device(dst, do, ol, out, so, sl, rl, stream=st)  # noqa: E731
            t_fd = timed(dec, a.reps)
            assert bool((rl == MB).all()) and torch.equal(out, src), "frame round trip"
            # the same blocks through the block calls
            nb = S * NB
            bb = int(L.k4lz4_max_output_size(BS))
            bo = torch.arange(nb, dtype=torch.int64, device=dev) * BS
            bl = torch.full((nb,), BS, dtype=torch.int32, device=dev)
            cd = torch.zeros(nb * bb, dtype=torch.uint8, device=dev)
            co = torch.arange(nb, dtype=torch.int64, device=dev) * bb
            cc = torch.full((nb,), bb, dtype=torch.int32, device=dev)
            cl = torch.zeros(nb, dtype=torch.int32, device=dev)
            if chaining:
                state = torch.zeros(S * N.CHAIN_STATE_BYTES, dtype=torch.uint8, device=dev)
                sto = torch.arange(S, dtype=torch.int64, device=dev) * N.CHAIN_STATE_BYTES
                steps = [torch.arange(S, dtype=torch.int64, device=dev) * NB + k for k in range(NB)]
                pre = [torch.full((S,), k * BS, dtype=torch.int32, device=dev) for k in range(NB)]
                sub = [(bo[s].contiguous(), co[s].contiguous()) for s in steps]
                res = [torch.zeros(S, dtype=torch.int32, device=dev) for _ in range(NB)]

                def benc():
                    state.zero_()
                    for k in range(NB):
                        B.encode_chain_batch_device(src.data_ptr(), sub[k][0].data_ptr(), bl.data_ptr(), pre[k].data_ptr(),
                                                    cd.data_ptr(), sub[k][1].data_ptr(), cc.data_ptr(), state.data_ptr(),
                                                    sto.data_ptr(), res[k].data_ptr(), S, 0, st)
                blens = lambda: torch.stack(res, 1).reshape(-1)  # noqa: E731
                t_be = timed(benc, a.reps)
                cl.copy_(blens())
                bout = torch.zeros(S * MB, dtype=torch.uint8, device=dev)
                dres = [torch.zeros(S, dtype=torch.int32, device=dev) for _ in range(NB)]
                capS = torch.full((S,), BS, dtype=torch.int32, device=dev)
                clk = [cl[s].contiguous() for s in steps]

                def bdec():
                    for k in range(NB):
                        B.decode_chain_batch_device(cd.data_ptr(), sub[k][1].data_ptr(), clk[k].data_ptr(), bout.data_ptr(),
                                                    sub[k][0].data_ptr(), capS.data_ptr(), pre[k].data_ptr(),
                                                    dres[k].data_ptr(), S, st)
                t_bd = timed(bdec, a.reps)
            else:
                benc = lambda: B.encode_batch_device(src.data_ptr(), bo.data_ptr(), bl.data_ptr(), cd.data_ptr(),  # noqa: E731
                                                     co.data_ptr(), cc.data_ptr(), cl.data_ptr(), nb, 0, st)
                t_be = timed(benc, a.reps)
                bout = torch.zeros(S * MB, dtype=torch.uint8, device=dev)
                dl = torch.zeros(nb, dtype=torch.int32, device=dev)
                bdec = lambda: B.decode_batch_device(cd.data_ptr(), co.data_ptr(), cl.data_ptr(), bout.data_ptr(),  # noqa: E731
                                                     bo.data_ptr(), bl.data_ptr(), dl.data_ptr(), nb, st)
                t_bd = timed(bdec, a.reps)
            assert torch.equal(bout, src), "block round trip"
            # frame bytes == block bytes (raw blocks aside): total compressed size matches within the length codes
            fsum = int(ol.sum()) - S * (7 + 4 + 4 * NB)
            bsum = int(torch.minimum(cl, bl).sum())
            assert fsum == bsum, (fsum, bsum)
            gb = S * MB / 1e9
            mode = "linked" if chaining else "independent"
            print(json.dumps({"S": S, "mode": mode, "mem": "device", "frame_enc_GBps": round(gb / t_fe, 2),
                              "block_enc_GBps": round(gb / t_be, 2), "frame_dec_GBps": round(gb / t_fd, 2),
                              "block_dec_GBps": round(gb / t_bd, 2)}), flush=True)
            if S > 1024:                             # host memory: the frame calls on host buffers
                continue
            t0 = time.perf_counter()
            for _ in range(2):
                frames_h, r = LZ4Frame.EncodeMany([host[i * MB:(i + 1) * MB] for i in range(S)], BS, chaining)
            t_he = (time.perf_counter() - t0) / 2
            t0 = time.perf_counter()
            for _ in range(2):
                back, rr = LZ4Frame.DecodeMany(frames_h, [MB] * S)
            t_hd = (time.perf_counter() - t0) / 2
            assert (rr == MB).all() and b"".join(back) == host.tobytes()
            dev_frames = dst.cpu().numpy()
            assert frames_h[S // 2] == dev_frames[(S // 2) * bound:(S // 2) * bound + int(ol[S // 2])].tobytes()
            print(json.dumps({"S": S, "mode": mode, "mem": "host", "frame_enc_GBps": round(gb / t_he, 2),
                              "frame_dec_GBps": round(gb / t_hd, 2)}), flush=True)
            del dst, out, cd, bout
        del src
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
