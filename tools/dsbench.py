"""Fixed-size destination benchmark (k4lz4_encode_dest_size_batch), device memory, CUDA events:

(a) B blocks of 64 KiB of reference datagen 0.63, encoded into targets of compressBound (the plain path inside
    the fill kernels), 32 KiB, 16 KiB and 4 KiB, against one k4lz4_encode_batch over the same blocks.  The arms
    alternate in one process, best of --reps each.  Figures: GB/s of source consumed (the sum of srcUsed) and of
    source offered.  The first and last 64 blocks of every arm are compared with upstream lz4 (oracle/_ref/).
(b) P inputs of 1 MiB of the same data packed into 4 KiB pages: every call encodes the next page of each unfinished
    input from where its earlier pages ended, until every input is packed; pages per second over the whole loop
    (the per-call host read of how many inputs are left included).  The first and last inputs' pages are decoded
    with upstream and compared with their input.

    python tools/dsbench.py [--blocks 65536] [--inputs 1024] [--reps 3]

Prints the card name, power limit and SM clock, then one JSON line per row."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> str:
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        q = f"unknown ({e})"
    return f"{torch.cuda.get_device_name(0)}; power limit, SM clock, max SM clock: {q}"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--inputs", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import build, batch as B
    from tests.dest_size_ref import Upstream, bound
    build.build()
    up = Upstream()
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    BS = 65536
    nb = a.blocks
    host = oracle.Port().datagen(nb * BS, 0.63, 0.0, 1234)
    src = torch.from_numpy(host).to(dev)
    idx = torch.arange(nb, dtype=torch.int64, device=dev)
    so = idx * BS
    sl = torch.full((nb,), BS, dtype=torch.int32, device=dev)
    bnd = bound(BS)
    do = idx * bnd
    dst = torch.empty(nb * bnd, dtype=torch.uint8, device=dev)
    out = torch.empty(nb, dtype=torch.int32, device=dev)
    used = torch.empty(nb, dtype=torch.int32, device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(target):
        if target is None:
            caps = torch.full((nb,), bnd, dtype=torch.int32, device=dev)
            f = lambda: B.encode_batch_device(src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst.data_ptr(),   # noqa: E731
                                              do.data_ptr(), caps.data_ptr(), out.data_ptr(), nb, 0, st)
        else:
            caps = torch.full((nb,), target, dtype=torch.int32, device=dev)
            f = lambda: B.encode_dest_size_batch_device(src.data_ptr(), so.data_ptr(), sl.data_ptr(),   # noqa: E731
                                                        dst.data_ptr(), do.data_ptr(), caps.data_ptr(),
                                                        out.data_ptr(), used.data_ptr(), nb, st)
        f()
        torch.cuda.synchronize()
        ev0.record(); f(); ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / 1e3

    def spot(target):
        o, u = out.cpu().numpy(), used.cpu().numpy()
        k = min(64, nb)
        ends = {0: dst[:k * bnd].cpu().numpy(), nb - k: dst[(nb - k) * bnd:].cpu().numpy()}
        for i in sorted(set(range(k)) | set(range(nb - k, nb))):
            blk = host[i * BS:(i + 1) * BS].tobytes()
            e0 = 0 if i < k else nb - k
            got = ends[e0][(i - e0) * bnd:(i - e0) * bnd + o[i]].tobytes()
            if target is None:
                want = up.plain(blk)
                assert got == want, ("encode_batch", i)
            else:
                r, c, want = up.dest_size(blk, target)
                assert (o[i], u[i], got) == (r, c, want), (target, i)

    arms = [None, bnd, 32768, 16384, 4096]
    best = {t: float("inf") for t in arms}
    consumed = {}
    for _ in range(a.reps):
        for t in arms:
            best[t] = min(best[t], run(t))
            if t is not None:
                consumed[t] = int(used.sum().item())
            spot(t)
    offered = nb * BS
    base = best[None]
    for t in arms:
        name = "encode_batch" if t is None else ("dest_size@bound" if t == bnd else f"dest_size@{t}")
        c = offered if t is None else consumed[t]
        print(json.dumps({"case": "a", "call": name, "blocks": nb, "target": t or bnd, "ms": round(best[t] * 1e3, 3),
                          "consumed_GBps": round(c / best[t] / 1e9, 2), "offered_GBps": round(offered / best[t] / 1e9, 2),
                          "consumed_fraction": round(c / offered, 4), "time_vs_encode_batch": round(best[t] / base, 4)}),
              flush=True)

    # (b) page packing
    del dst, src
    P, MB, PAGE = a.inputs, 1 << 20, 4096
    hostb = host[:P * MB] if P * MB <= host.size else oracle.Port().datagen(P * MB, 0.63, 0.0, 99)
    srcb = torch.from_numpy(np.ascontiguousarray(hostb)).to(dev)
    maxPages = P * (MB // (PAGE - 64) + 2)
    pages = torch.empty(maxPages * PAGE, dtype=torch.uint8, device=dev)
    pageLen = torch.zeros(maxPages, dtype=torch.int32, device=dev)
    pageUsed = torch.zeros(maxPages, dtype=torch.int32, device=dev)
    pageOwner = torch.full((maxPages,), -1, dtype=torch.int64, device=dev)

    def pack():
        pos = torch.zeros(P, dtype=torch.int64, device=dev)
        total = 0
        live = torch.arange(P, dtype=torch.int64, device=dev)
        while live.numel() > 0:
            m = live.numel()
            s_off = live * MB + pos[live]
            s_len = (MB - pos[live]).to(torch.int32)
            d_off = (total + torch.arange(m, dtype=torch.int64, device=dev)) * PAGE
            caps = torch.full((m,), PAGE, dtype=torch.int32, device=dev)
            B.encode_dest_size_batch_device(srcb.data_ptr(), s_off.data_ptr(), s_len.data_ptr(), pages.data_ptr(),
                                            d_off.data_ptr(), caps.data_ptr(), pageLen[total:].data_ptr(),
                                            pageUsed[total:].data_ptr(), m, st)
            pageOwner[total:total + m] = live
            pos[live] += pageUsed[total:total + m].to(torch.int64)
            total += m
            live = live[pos[live] < MB]                   # the host reads how many inputs are left
        return total

    pack()
    torch.cuda.synchronize()
    bestb, npages = float("inf"), 0
    for _ in range(a.reps):
        ev0.record(); npages = pack(); ev1.record()
        torch.cuda.synchronize()
        bestb = min(bestb, ev0.elapsed_time(ev1) / 1e3)
    owner, plen, pused, pg = (pageOwner[:npages].cpu().numpy(), pageLen[:npages].cpu().numpy(),
                              pageUsed[:npages].cpu().numpy(), pages[:npages * PAGE].cpu().numpy())
    for i in (0, P - 1):
        ks = np.nonzero(owner == i)[0]
        back = b"".join(up.decode(pg[k * PAGE:k * PAGE + plen[k]].tobytes(), int(pused[k])) for k in ks)
        assert back == hostb[i * MB:(i + 1) * MB].tobytes(), ("page packing", i)
    print(json.dumps({"case": "b", "inputs": P, "input_bytes": MB, "page": PAGE, "pages": npages,
                      "ms": round(bestb * 1e3, 3), "pages_per_s": round(npages / bestb), "source_GBps":
                      round(P * MB / bestb / 1e9, 2), "fill": round(float(plen.sum()) / (npages * PAGE), 4)}),
          flush=True)


if __name__ == "__main__":
    main()
