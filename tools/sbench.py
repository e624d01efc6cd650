"""Whole chained streams (k4lz4_decode_chain_streams) against stepping k4lz4_decode_chain_batch one block per stream
per call, and against k4lz4_frame_decode_batch on the same content as one linked frame per stream (upstream's
LZ4F_compressFrame, 64 KiB linked blocks), in the same process, alternating.

Workloads: `--mib` MiB of datagen 0.63 in linked 64 KiB blocks (upstream's LZ4_compress_fast_continue) as one stream
and split into S = 4, 16, 64 streams, plus a repetitive input in which every block copies from the one before (the
deepest chain).  Device memory (CUDA events around each call) and host memory (host clock around the synchronous
call).  GB/s are decoded bytes over call time.  A torch.profiler run of its own gives the four passes' kernel times
for one call, and from them the replay's time per block of the call (replay kernel time over all S x blocks).  The card's name and power limit are read in the
same run.  Needs the reference's C engine in oracle/_ref (built by __graft_entry__.build()).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from k4os.compression.lz4_b200 import batch as B  # noqa: E402
from k4os.compression.lz4_b200.frame import LZ4Frame  # noqa: E402
from tests import chain_ref as CR  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--mib", type=int, default=1024)
p.add_argument("--streams", default="1,4,16,64")
p.add_argument("--reps", type=int, default=3)
p.add_argument("--host-reps", type=int, default=1)
a = p.parse_args()
BS = 65536
dev = torch.device("cuda", 0)
up = CR.Upstream()


def make(kind: str, total: int, S: int):
    """S streams of total / S bytes each -> list of (data, blocks)"""
    import oracle
    per = total // S // BS * BS
    port = oracle.Port()
    out = []
    for s in range(S):
        if kind == "datagen":
            parts = [port.datagen(min(64 << 20, per - o), 0.63, 0.0, 1000 * s + o // (64 << 20)).tobytes()
                     for o in range(0, per, 64 << 20)]
            data = b"".join(parts)
        else:
            unit = np.random.default_rng(s).integers(0, 256, 40001, dtype=np.uint8).tobytes()
            data = (unit * (per // len(unit) + 1))[:per]
        out.append((data, up.encode_chain(data, BS), up.frame_linked(data, size_id=4)))
    return out


class Work:
    def __init__(self, streams):
        self.S = len(streams)
        self.nb = len(streams[0][1])
        blocks = [b for _, bl, _ in streams for b in bl]
        self.lens = np.array([len(b) for b in blocks], dtype=np.int32)
        self.soff = np.zeros(len(blocks), dtype=np.int64)
        self.soff[1:] = np.cumsum(self.lens[:-1], dtype=np.int64)
        self.src = np.frombuffer(b"".join(blocks), dtype=np.uint8)
        self.caps = np.full(len(blocks), BS, dtype=np.int32)
        self.es = np.arange(self.S + 1, dtype=np.int32) * self.nb
        self.doff = np.arange(self.S, dtype=np.int64) * self.nb * BS
        self.pre = np.zeros(self.S, dtype=np.int32)
        self.out_bytes = self.S * self.nb * BS
        self.want = b"".join(d for d, _, _ in streams)
        frames = [f for _, _, f in streams]
        self.flen = np.array([len(f) for f in frames], dtype=np.int32)
        self.foff = np.zeros(self.S, dtype=np.int64)
        self.foff[1:] = np.cumsum(self.flen[:-1], dtype=np.int64)
        self.fsrc = np.frombuffer(b"".join(frames), dtype=np.uint8)
        self.fcap = np.full(self.S, self.nb * BS, dtype=np.int32)
        # stepping: call k decodes block k of every stream, slot = the stream's region at k * BS
        e = np.arange(self.S)[None, :] * self.nb + np.arange(self.nb)[:, None]        # [step, stream]
        self.step_soff, self.step_len = self.soff[e], self.lens[e]
        self.step_doff = self.doff[None, :] + np.arange(self.nb)[:, None] * BS
        self.step_pre = np.broadcast_to(np.minimum(np.arange(self.nb) * BS, 65535)[:, None], e.shape).astype(np.int32)

    def to_device(self):
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        self.d = {k: t(getattr(self, k)) for k in ("src", "soff", "lens", "caps", "es", "doff", "pre", "step_soff",
                                                   "step_len", "step_doff", "step_pre", "flen", "foff", "fsrc",
                                                   "fcap")}
        self.d["fout"] = torch.empty(self.S, dtype=torch.int32, device=dev)
        self.d["dst"] = torch.empty(self.out_bytes + 16, dtype=torch.uint8, device=dev)
        self.d["out"] = torch.empty(len(self.lens), dtype=torch.int32, device=dev)
        self.d["cap1"] = torch.full((self.S,), BS, dtype=torch.int32, device=dev)

    def streams_dev(self):
        d = self.d
        B.decode_chain_streams_device(d["src"].data_ptr(), d["soff"].data_ptr(), d["lens"].data_ptr(), 0,
                                      d["caps"].data_ptr(), d["out"].data_ptr(), len(self.lens), d["es"].data_ptr(),
                                      d["dst"].data_ptr(), d["doff"].data_ptr(), d["pre"].data_ptr(), self.S,
                                      torch.cuda.current_stream().cuda_stream)

    def stepped_dev(self):
        d = self.d
        st = torch.cuda.current_stream().cuda_stream
        for k in range(self.nb):
            B.decode_chain_batch_device(d["src"].data_ptr(), d["step_soff"][k].data_ptr(), d["step_len"][k].data_ptr(),
                                        d["dst"].data_ptr(), d["step_doff"][k].data_ptr(), d["cap1"].data_ptr(),
                                        d["step_pre"][k].data_ptr(), d["out"].data_ptr(), self.S, st)

    def frame_dev(self):
        d = self.d
        LZ4Frame.decode_many_device(d["fsrc"], d["foff"], d["flen"], d["dst"], d["doff"], d["fcap"], d["fout"],
                                    torch.cuda.current_stream().cuda_stream)

    def check_dev(self):
        got = self.d["dst"][:self.out_bytes].cpu().numpy().tobytes()
        return got == self.want

    def streams_host(self, dst):
        out = B.decode_chain_streams_host(self.src, self.soff, self.lens, self.caps, self.es, dst, self.doff, self.pre)
        return int(out.min()) >= 0

    def stepped_host(self, dst):
        ok = True
        for k in range(self.nb):
            out = B.decode_chain_batch_host(self.src, self.step_soff[k], self.step_len[k], dst, self.step_doff[k],
                                            np.full(self.S, BS, dtype=np.int32), self.step_pre[k])
            ok &= int(out.min()) >= 0
        return ok


def time_dev(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    total = a.mib << 20
    loads = [("datagen", int(s)) for s in a.streams.split(",")] + [("repetitive", 1)]
    for kind, S in loads:
        t0 = time.time()
        w = Work(make(kind, total if kind == "datagen" else min(total, 256 << 20), S))
        w.to_device()
        gen = time.time() - t0
        w.d["dst"].zero_(); w.streams_dev(); torch.cuda.synchronize()
        ok_new = w.check_dev()
        w.d["dst"].zero_(); w.stepped_dev(); torch.cuda.synchronize()
        ok_step = w.check_dev()
        w.d["dst"].zero_(); w.frame_dev(); torch.cuda.synchronize()
        ok_frame = w.check_dev()
        tn, ts, tf = [], [], []
        for _ in range(a.reps):                                 # alternating
            tn.append(time_dev(w.streams_dev))
            ts.append(time_dev(w.stepped_dev))
            tf.append(time_dev(w.frame_dev))
        hdst = np.zeros(w.out_bytes + 16, dtype=np.uint8)
        hn, hs = [], []
        for _ in range(a.host_reps):
            t0 = time.perf_counter(); okh = w.streams_host(hdst); hn.append(time.perf_counter() - t0)
            okh &= hdst[:w.out_bytes].tobytes() == w.want
            hdst[:] = 0
            t0 = time.perf_counter(); oks = w.stepped_host(hdst); hs.append(time.perf_counter() - t0)
            oks &= hdst[:w.out_bytes].tobytes() == w.want
        gb = w.out_bytes / 1e9
        r = dict(workload=kind, streams=S, blocks_per_stream=w.nb, mib=w.out_bytes >> 20,
                 exact=dict(streams_dev=ok_new, stepped_dev=ok_step, frame_dev=ok_frame, streams_host=bool(okh),
                            stepped_host=bool(oks)),
                 dev_frame_gbs=round(gb / np.median(tf), 2),
                 dev_streams_gbs=round(gb / np.median(tn), 2), dev_stepped_gbs=round(gb / np.median(ts), 2),
                 host_streams_gbs=round(gb / np.median(hn), 2), host_stepped_gbs=round(gb / np.median(hs), 2),
                 dev_streams_ms=[round(x * 1e3, 2) for x in tn], dev_stepped_ms=[round(x * 1e3, 2) for x in ts],
                 gen_s=round(gen, 1))
        # the four passes of one call, in a profiler run of its own
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            w.streams_dev(); torch.cuda.synchronize()
        ker = {}
        for ev in prof.key_averages():
            if "stream_" in ev.key:
                ker[ev.key.split("(")[0].replace("void k4::", "")] = round(ev.device_time_total / max(ev.count, 1) / 1e3, 3)
        r["kernel_ms"] = ker
        rk = [v for k, v in ker.items() if "replay" in k]
        if rk:
            r["replay_us_per_block"] = round(rk[0] * 1e3 / (w.S * w.nb), 2)
        print(json.dumps(r), flush=True)
        del w
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
