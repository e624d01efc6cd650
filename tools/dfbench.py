"""Dictionary-frame benchmark, device memory, CUDA events:

(a) record-like messages of 256 B - 4 KiB (slices of seeded JSON-like records), one independent frame each, against
    one 64 KiB dictionary of the same vocabulary: k4lz4_frame_encode_dict_batch / _decode_dict_batch, against the
    same messages as frames without a dictionary (k4lz4_frame_encode_batch / _decode_batch) and as bare dictionary
    blocks (k4lz4_encode_dict_batch / k4lz4_decode_dict_batch);
(b) S frames of 1 MiB of reference datagen 0.63 with a 64 KiB dictionary (the first 64 KiB of another datagen
    stream of the same kind), linked and independent, against the frame calls without a dictionary.

Every output of the run is checked: each encode is decoded back and compared with its input.  Frame calls take
at most 32 768 frames each (the decode's scratch slots), timed over all of them.

    python tools/dfbench.py [--messages 1000000] [--sizes 264,1024,4096] [--reps 5]

Prints the card name and power limit, then one JSON line per row: GB/s of content, and the ratio."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fbench import card, timed  # noqa: E402


def gbps(nbytes: int, sec: float) -> float:
    return nbytes / sec / 1e9


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--messages", type=int, default=1_000_000)
    ap.add_argument("--sizes", default="264,1024,4096")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import oracle
    from k4os.compression.lz4_b200 import build, LZ4Codec
    from k4os.compression.lz4_b200 import _native as N
    build.build()
    L = N.lib()
    print(card(), flush=True)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    T = lambda x: torch.from_numpy(np.array(x)).to(dev)   # noqa: E731
    rng = np.random.default_rng(1)

    def dict_tensors(d: np.ndarray, n: int):
        return T(d), torch.zeros(n, dtype=torch.int64, device=dev), torch.full((n,), len(d), dtype=torch.int32,
                                                                                  device=dev)

    CHUNK = 32768     # frames per call: a frame decode holds a 64 KiB + block scratch slot per frame's last block

    def frame_calls(src, so, sl, cap_each, dic, linked, bs, reps, content_bytes, label):
        n = sl.numel()
        caps = torch.full((n,), cap_each, dtype=torch.int32, device=dev)
        do = torch.arange(n, dtype=torch.int64, device=dev) * cap_each
        dst = torch.zeros(n * cap_each, dtype=torch.uint8, device=dev)
        out = torch.zeros(n, dtype=torch.int32, device=dev)
        fl = 0 if linked else N.FRAME_INDEPENDENT
        back = torch.zeros_like(src)
        bl = torch.zeros(n, dtype=torch.int32, device=dev)
        db, doff, dl = dic if dic is not None else (None, None, None)
        P = lambda t, c0: t[c0:].data_ptr()   # noqa: E731

        def enc():
            for c0 in range(0, n, CHUNK):
                k = min(CHUNK, n - c0)
                if dic is not None:
                    N.check(L.k4lz4_frame_encode_dict_batch(
                        src.data_ptr(), P(so, c0), P(sl, c0), dst.data_ptr(), P(do, c0), P(caps, c0), db.data_ptr(),
                        P(doff, c0), P(dl, c0), None, P(out, c0), k, bs, fl, 0, N.MEM_DEVICE, st, 0))
                else:
                    N.check(L.k4lz4_frame_encode_batch(
                        src.data_ptr(), P(so, c0), P(sl, c0), dst.data_ptr(), P(do, c0), P(caps, c0), P(out, c0), k,
                        bs, fl, 0, N.MEM_DEVICE, st, 0))

        def dec():
            for c0 in range(0, n, CHUNK):
                k = min(CHUNK, n - c0)
                if dic is not None:
                    N.check(L.k4lz4_frame_decode_dict_batch(
                        dst.data_ptr(), P(do, c0), P(out, c0), back.data_ptr(), P(so, c0), P(sl, c0), db.data_ptr(),
                        P(doff, c0), P(dl, c0), P(bl, c0), k, N.MEM_DEVICE, st, 0))
                else:
                    N.check(L.k4lz4_frame_decode_batch(
                        dst.data_ptr(), P(do, c0), P(out, c0), back.data_ptr(), P(so, c0), P(sl, c0), P(bl, c0), k,
                        N.MEM_DEVICE, st, 0))
        te = timed(enc, reps)
        td = timed(dec, reps)
        assert bool((out > 0).all()), label
        assert torch.equal(bl, sl) and torch.equal(back, src), label
        ratio = float(out.sum().item()) / content_bytes
        return te, td, ratio

    # ---- (a) messages ------------------------------------------------------------------------------------
    from tests import dict_enc_ref as DR
    pool = np.frombuffer(DR.records(64 << 20, 5), dtype=np.uint8)
    dictionary = np.frombuffer(DR.records(65536, 6), dtype=np.uint8)
    m = a.messages
    lens = rng.integers(256, 4097, m).astype(np.int32)
    starts = rng.integers(0, len(pool) - 4096, m)
    so_np = np.zeros(m, dtype=np.int64)
    so_np[1:] = np.cumsum(lens[:-1].astype(np.int64))
    total = int(lens.sum())
    gpool = T(pool)
    src = torch.empty(total, dtype=torch.uint8, device=dev)
    g_so, g_sl, g_st = T(so_np), T(lens), T(starts.astype(np.int64))
    N.check(L.k4lz4_copy_blocks_device(gpool.data_ptr(), g_st.data_ptr(), src.data_ptr(), g_so.data_ptr(),
                                       g_sl.data_ptr(), m, st, 0))
    dic = dict_tensors(dictionary, m)
    fb = int(L.k4lz4_frame_bound(4096, 65536, N.FRAME_INDEPENDENT))
    for label, d in (("frame+dict", dic), ("frame", None)):
        te, td, r = frame_calls(src, g_so, g_sl, fb, d, False, 65536, a.reps, total, label)
        print(json.dumps({"case": "a", "call": label, "messages": m, "bytes": total, "enc_GBps": round(gbps(total, te), 2),
                          "dec_GBps": round(gbps(total, td), 2), "ratio": round(r, 4)}), flush=True)
    bb = LZ4Codec.MaximumOutputSize(4096)
    caps = torch.full((m,), bb, dtype=torch.int32, device=dev)
    do = torch.arange(m, dtype=torch.int64, device=dev) * bb
    dst = torch.zeros(m * bb, dtype=torch.uint8, device=dev)
    out = torch.zeros(m, dtype=torch.int32, device=dev)
    back = torch.zeros_like(src)
    bl = torch.zeros(m, dtype=torch.int32, device=dev)
    db, doff, dl = dic
    enc = lambda: N.check(L.k4lz4_encode_dict_batch(   # noqa: E731
        src.data_ptr(), g_so.data_ptr(), g_sl.data_ptr(), dst.data_ptr(), do.data_ptr(), caps.data_ptr(),
        db.data_ptr(), doff.data_ptr(), dl.data_ptr(), out.data_ptr(), m, N.MEM_DEVICE, st, 0))
    dec = lambda: N.check(L.k4lz4_decode_dict_batch(   # noqa: E731
        dst.data_ptr(), do.data_ptr(), out.data_ptr(), back.data_ptr(), g_so.data_ptr(), g_sl.data_ptr(),
        db.data_ptr(), doff.data_ptr(), dl.data_ptr(), bl.data_ptr(), m, N.MEM_DEVICE, st, 0))
    te, td = timed(enc, a.reps), timed(dec, a.reps)
    assert bool((out > 0).all()) and torch.equal(bl, g_sl) and torch.equal(back, src)
    print(json.dumps({"case": "a", "call": "blocks+dict", "messages": m, "bytes": total,
                      "enc_GBps": round(gbps(total, te), 2), "dec_GBps": round(gbps(total, td), 2),
                      "ratio": round(float(out.sum().item()) / total, 4)}), flush=True)
    del src, dst, back, gpool

    # ---- (b) 1 MiB frames of datagen 0.63 -------------------------------------------------------------------
    port = oracle.Port()
    MB = 1 << 20
    dgd = np.asarray(port.datagen(65536, 0.63, 0.0, 99))[:65536]
    base = np.concatenate([np.asarray(port.datagen(MB, 0.63, 0.0, 1000 + i))[:MB] for i in range(64)])
    for S in [int(x) for x in a.sizes.split(",")]:
        data = np.tile(base, (S + 63) // 64)[:S * MB]             # 64 distinct MiB, as tools/fbench.py
        src = T(data)
        so = torch.arange(S, dtype=torch.int64, device=dev) * MB
        sl = torch.full((S,), MB, dtype=torch.int32, device=dev)
        d = dict_tensors(dgd, S)
        fbm = int(L.k4lz4_frame_bound(MB, 65536, 0))
        for linked in (True, False):
            for label, dd in (("frame+dict", d), ("frame", None)):
                te, td, r = frame_calls(src, so, sl, fbm, dd, linked, 65536, a.reps, S * MB, label)
                print(json.dumps({"case": "b", "frames": S, "linked": linked, "call": label,
                                  "enc_GBps": round(gbps(S * MB, te), 2), "dec_GBps": round(gbps(S * MB, td), 2),
                                  "ratio": round(r, 4)}), flush=True)
        del src


if __name__ == "__main__":
    main()
