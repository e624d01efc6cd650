"""tools/dbench.py -- kernel-only micro-benchmark used while tuning (not the headline bench).
Times k4lz4_decode_batch / k4lz4_encode_batch on device-resident blocks with CUDA events and
checks the result (decode: against the raw input; encode: round trip).
    python tools/dbench.py [--blocks N] [--data datagen|synth] [--mp 630] [--reps 5] [--what decode|encode|both]
--data datagen: the reference's generator (oracle/: RDG_genBuffer, matchProba = mp/1000, seed 1234 + chunk)
--data synth  : the library's own device generator
    python tools/dbench.py --what chain [--streams 264,1024,4096] [--chain-blocks 16]
S streams x B linked 64 KiB blocks of datagen, compressed by upstream's chained encoder
(LZ4_compress_fast_continue, oracle/_ref/): one k4lz4_decode_chain_batch call per step decodes block k of every
stream behind its history; GB/s of decoded output over all B steps, next to one k4lz4_decode_batch call over
the same raw bytes compressed as independent blocks.
    python tools/dbench.py --what chain-encode [--streams 264,1024,4096] [--chain-blocks 16]
S streams x B linked 64 KiB blocks of datagen: one k4lz4_encode_chain_batch call per step (device memory) encodes
block k of every stream behind its history; GB/s of input over all B steps, next to one k4lz4_encode_batch call
over the same raw bytes, with the encoder's path counters and a spot check against upstream's chained encoder.
    python tools/dbench.py --what size [--blocks 65536] [--size-libs scratch/libk4lz4_A.so,...]
k4lz4_decoded_size_batch over the compressed blocks in device memory: GB/s of compressed input, every size checked
equal to the block length; other builds (segment length and warm-up, K4_SW_SEG / K4_SW_WARM) alternate with the
shipped one in three rounds.  The card's name and power limit are printed with it.
    python tools/dbench.py --what dict-encode [--messages 1000000] [--reps 5]
k4lz4_encode_dict_batch in device memory: M messages of the pickler benchmark's length mix (256 B .. 4 KiB) of
JSON-like records against one 64 KiB dictionary of other records, beside k4lz4_encode_batch over the same messages
without one; then 65 536 x 64 KiB blocks of the same content against the dictionary, beside
k4lz4_encode_chain_batch over the same blocks (new streams); then the host-memory rate of the message workload, and
a torch.profiler run of one device call for the kernels' times (the dictionary load among them).  GB/s of source
bytes, compressed ratios, spot checks against upstream (oracle/_ref/), and the card's name and power limit.
The 32-bit engine (k4lz4_encode_chain_batch_x32, LZ4Codec.Enforce32) runs the same steps in the same process,
timed alternately with the plain one, with a spot check against upstream's chained encoder built as LL32; the card's
name and power limit are printed with it.  The host-memory form of one step is timed too, beside a host-memory k4lz4_encode_batch of the same blocks (the
chained call also moves each block's history and its 16 400-byte state each way).
Both chain arms also time a chain group (k4lz4_chain_group_*: rings and states resident on the GPU) and print
per-step times (one block of every stream) through host memory -- LZ4FastChainEncoder.EncodeMany /
LZ4ChainDecoder.DecodeMany (today's chained call with its ring staging), the group, one independent-block call
over the same blocks -- and through device memory -- the chained batch call, the group, and the independent call
over all steps divided by the step count.
"""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from k4os.compression.lz4_b200 import batch as B, _native as N
import k4os.compression.lz4_b200 as K
import time

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=32768)
ap.add_argument("--bs", type=int, default=65536)
ap.add_argument("--mp", type=int, default=630)
ap.add_argument("--data", default="datagen")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--what", default="decode")
ap.add_argument("--check", type=int, default=0, help="encode: compare every CHECK-th block with the oracle engine (bit-exact)")
ap.add_argument("--lib", default=None, help="alternative build of libk4lz4.so (e.g. a -DK4_DT_PROFILE build under scratch/)")
ap.add_argument("--streams", default="264,1024,4096", help="chain: stream counts")
ap.add_argument("--chain-blocks", type=int, default=16, help="chain: linked blocks per stream")
ap.add_argument("--messages", type=int, default=1000000, help="dict-encode: message count")
ap.add_argument("--size-libs", default="", help="size: other builds of libk4lz4.so (tools/build_variant.py), "
                                                "timed alternately with the shipped one in this process")
a = ap.parse_args()


def host_ms(fn, reps):
    """median wall time of fn() in ms after one warm-up call"""
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def timeit(fn, reps):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    return min(ts), float(np.median(ts))


def report(kind, S, Bk, host, dev):
    print(f"{kind}-group S={S} x {Bk} steps, ms per step | host memory: chained {host[0]:.2f}, group {host[1]:.2f}, "
          f"independent {host[2]:.2f} | device memory: chained {dev[0]:.3f}, group {dev[1]:.3f}, "
          f"independent {dev[2]:.3f}", flush=True)


def dict_encode():
    import subprocess
    from tests import dict_enc_ref as DR
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    up = DR.DictUpstream()
    dev, st = torch.device("cuda", 0), torch.cuda.current_stream().cuda_stream
    L = N.lib()
    rng = np.random.default_rng(7)
    pool = np.frombuffer(DR.records(8 << 20, 8), dtype=np.uint8)
    d = np.frombuffer(DR.records(65536, 9), dtype=np.uint8)
    M = a.messages
    lens = rng.integers(256, 4097, M).astype(np.int32)
    starts = rng.integers(0, len(pool) - 4096, M)
    offs = np.zeros(M, dtype=np.int64)
    offs[1:] = np.cumsum(lens[:-1], dtype=np.int64)
    total = int(lens.sum())
    hsrc = np.empty(total, dtype=np.uint8)
    for i in range(M):
        hsrc[offs[i]:offs[i] + lens[i]] = pool[starts[i]:starts[i] + lens[i]]
    caps = (lens + lens // 255 + 16).astype(np.int32)
    doffs = np.zeros(M, dtype=np.int64)
    doffs[1:] = np.cumsum(caps[:-1], dtype=np.int64)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    src, so, sl, dc, do_ = t(hsrc), t(offs), t(lens), t(caps), t(doffs)
    dst = torch.empty(int(caps.sum()), dtype=torch.uint8, device=dev)
    out = torch.zeros(M, dtype=torch.int32, device=dev)
    dd, zo, dlen = t(d), torch.zeros(M, dtype=torch.int64, device=dev), torch.full((M,), len(d), dtype=torch.int32, device=dev)

    def denc(n=M):
        B.encode_dict_batch_device(src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst.data_ptr(), do_.data_ptr(),
                                   dc.data_ptr(), dd.data_ptr(), zo.data_ptr(), dlen.data_ptr(), out.data_ptr(), n, st)

    def penc():
        B.encode_batch_device(src.data_ptr(), so.data_ptr(), sl.data_ptr(), dst.data_ptr(), do_.data_ptr(),
                              dc.data_ptr(), out.data_ptr(), M, 0, st)
    tm = {}
    for _ in range(3):                                   # alternate the two calls
        for name, fn in (("dict", denc), ("plain", penc)):
            tm.setdefault(name, []).append(timeit(fn, a.reps)[1])
    denc(); torch.cuda.synchronize()
    ho, hd = out.cpu().numpy(), dst.cpu().numpy()
    rd = float(ho.sum()) / total
    bad = 0
    for i in range(0, M, max(M // 500, 1)):
        r, want = up.encode(hsrc[offs[i]:offs[i] + lens[i]].tobytes(), d.tobytes())
        bad += int(ho[i]) != r or hd[doffs[i]:doffs[i] + r].tobytes() != want
    penc(); torch.cuda.synchronize()
    rp = float(out.sum()) / total
    md, mp = float(np.median(tm["dict"])), float(np.median(tm["plain"]))
    print(f"dict-encode messages M={M} ({total / 1e9:.2f} GB, 256 B..4 KiB) vs one 64 KiB dictionary: {md:.3f} ms "
          f"{total / md / 1e6:.1f} GB/s ratio {rd:.3f} (spot check vs upstream: {bad} differ) | k4lz4_encode_batch, "
          f"no dictionary: {mp:.3f} ms {total / mp / 1e6:.1f} GB/s ratio {rp:.3f} (medians of 3 alternating runs "
          f"of {a.reps})", flush=True)

    # host memory, the same messages (dictionary staged once per chunk)
    hdst = np.empty(int(caps.sum()), dtype=np.uint8)
    hout = np.zeros(M, dtype=np.int32)
    hzo, hdl = np.zeros(M, dtype=np.int64), np.full(M, len(d), dtype=np.int32)

    def henc():
        N.check(L.k4lz4_encode_dict_batch(hsrc.ctypes.data, offs.ctypes.data, lens.ctypes.data, hdst.ctypes.data,
                                          doffs.ctypes.data, caps.ctypes.data, d.ctypes.data, hzo.ctypes.data,
                                          hdl.ctypes.data, hout.ctypes.data, M, N.MEM_HOST, None, 0))
    hm = host_ms(henc, 3)
    print(f"dict-encode host memory M={M}: {hm:.1f} ms {total / hm / 1e6:.2f} GB/s, results equal to device: "
          f"{bool(np.array_equal(hout, ho))}", flush=True)
    del src, dst, out, so, sl, dc, do_, zo, dlen, hdst

    # 65 536 x 64 KiB blocks of the same content, against the dictionary and as new chained streams
    nb, bs = 65536, 65536
    big = t(pool).repeat((nb * bs + len(pool) - 1) // len(pool))[:nb * bs]
    bound = bs + bs // 255 + 16
    bo = torch.arange(nb, dtype=torch.int64, device=dev)
    so2, do2 = bo * bs, bo * bound
    sl2, dc2 = torch.full((nb,), bs, dtype=torch.int32, device=dev), torch.full((nb,), bound, dtype=torch.int32, device=dev)
    dst2 = torch.empty(nb * bound, dtype=torch.uint8, device=dev)
    out2 = torch.zeros(nb, dtype=torch.int32, device=dev)
    zo2, dl2 = torch.zeros(nb, dtype=torch.int64, device=dev), torch.full((nb,), len(d), dtype=torch.int32, device=dev)
    SB = N.CHAIN_STATE_BYTES
    states = torch.zeros(nb * SB, dtype=torch.uint8, device=dev)
    stoff, pre = bo * SB, torch.zeros(nb, dtype=torch.int32, device=dev)

    def denc2():
        B.encode_dict_batch_device(big.data_ptr(), so2.data_ptr(), sl2.data_ptr(), dst2.data_ptr(), do2.data_ptr(),
                                   dc2.data_ptr(), dd.data_ptr(), zo2.data_ptr(), dl2.data_ptr(), out2.data_ptr(), nb, st)

    def cenc2():
        states.zero_()
        B.encode_chain_batch_device(big.data_ptr(), so2.data_ptr(), sl2.data_ptr(), pre.data_ptr(), dst2.data_ptr(),
                                    do2.data_ptr(), dc2.data_ptr(), states.data_ptr(), stoff.data_ptr(),
                                    out2.data_ptr(), nb, 0, st)
    tm = {}
    for _ in range(3):
        for name, fn in (("dict", denc2), ("chain", cenc2)):
            tm.setdefault(name, []).append(timeit(fn, a.reps)[1])
    denc2(); torch.cuda.synchronize()
    rd2 = float(out2.sum()) / (nb * bs)
    o0 = out2[:4].cpu().numpy()
    h0 = dst2[:4 * bound].cpu().numpy()
    hb = big[:4 * bs].cpu().numpy()
    bad2 = sum(up.encode(hb[k * bs:(k + 1) * bs].tobytes(), d.tobytes())[1] != h0[k * bound:k * bound + o0[k]].tobytes()
               for k in range(4))
    cenc2(); torch.cuda.synchronize()
    rc2 = float(out2.sum()) / (nb * bs)
    md, mc = float(np.median(tm["dict"])), float(np.median(tm["chain"]))
    print(f"dict-encode blocks {nb} x 64 KiB vs 64 KiB dictionary: {md:.3f} ms {nb * bs / md / 1e6:.1f} GB/s ratio "
          f"{rd2:.3f} ({bad2} of 4 differ from upstream) | k4lz4_encode_chain_batch, new streams: {mc:.3f} ms "
          f"{nb * bs / mc / 1e6:.1f} GB/s ratio {rc2:.3f}", flush=True)
    del big, dst2, states

    # kernel times of one message call, in a profiler run of its own
    src, so, sl, dc, do_ = t(hsrc), t(offs), t(lens), t(caps), t(doffs)
    dst = torch.empty(int(caps.sum()), dtype=torch.uint8, device=dev)
    out = torch.zeros(M, dtype=torch.int32, device=dev)
    zo, dlen = torch.zeros(M, dtype=torch.int64, device=dev), torch.full((M,), len(d), dtype=torch.int32, device=dev)
    denc(); torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        denc(); torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "dict" in ev.key:
            print(f"   kernel {ev.key.split('(')[0]}: {ev.device_time_total / max(ev.count, 1) / 1e3:.3f} ms", flush=True)


if a.what == "dict-encode":
    dict_encode()
    sys.exit(0)
if a.what in ("chain", "chain-encode"):
    a.blocks = max(int(x) for x in a.streams.split(",")) * a.chain_blocks
if a.lib:
    N.SO_PATH = os.path.abspath(a.lib)
dev = torch.device("cuda", 0)
st = torch.cuda.current_stream().cuda_stream
nb, bs = a.blocks, a.bs
bound = bs + bs // 255 + 16
if a.data == "synth":
    raw = torch.empty(nb * bs, dtype=torch.uint8, device=dev)
    B.synth_device(raw.data_ptr(), nb, bs, a.mp, 1234, 0, st)
else:
    import oracle
    from concurrent.futures import ThreadPoolExecutor
    eng = oracle.best()
    host = np.empty(nb * bs, dtype=np.uint8)
    chunk = 1024 * bs
    nch = (nb * bs + chunk - 1) // chunk
    def gen(c):
        lo = c * chunk; hi = min(lo + chunk, nb * bs)
        eng.datagen(hi - lo, a.mp / 1000.0, 0.0, 1234 + c, out=host[lo:hi])
    with ThreadPoolExecutor(max_workers=min(64, os.cpu_count() or 1)) as ex:
        list(ex.map(gen, range(nch)))
    raw = torch.from_numpy(host).to(dev)
idx = torch.arange(nb, dtype=torch.int64, device=dev)
roff, coff = idx * bs, idx * bound
rlen = torch.full((nb,), bs, dtype=torch.int32, device=dev)
ccap = torch.full((nb,), bound, dtype=torch.int32, device=dev)
slots = torch.empty(nb * bound, dtype=torch.uint8, device=dev)
clen = torch.zeros(nb, dtype=torch.int32, device=dev)
def enc():
    B.encode_batch_device(raw.data_ptr(), roff.data_ptr(), rlen.data_ptr(), slots.data_ptr(), coff.data_ptr(),
                          ccap.data_ptr(), clen.data_ptr(), nb, 0, st)
if a.what != "chain-encode":
    enc(); torch.cuda.synchronize()
ratio = float(clen.sum()) / (nb * bs)
if a.what in ("encode", "both"):
    ms, med = timeit(enc, a.reps)
    if a.check:
        import oracle
        eng = oracle.best()
        hraw = raw.cpu().numpy(); hs = slots.cpu().numpy(); hl = clen.cpu().numpy()
        nbad = 0
        for i in range(0, nb, a.check):
            r, ref = eng.encode(hraw[i * bs:(i + 1) * bs])
            if r != int(hl[i]) or hs[i * bound:i * bound + r].tobytes() != ref: nbad += 1
        print(f"   encode check: {len(range(0, nb, a.check))} blocks vs oracle, {nbad} differ", flush=True)
    print(f"encode[{a.data}{a.mp}]: {ms:.3f} ms (median {med:.3f})  {nb*bs/ms/1e6:.1f} GB/s  ratio {ratio:.3f}", flush=True)
if a.what in ("decode", "both"):
    poff = torch.cumsum(clen.to(torch.int64), 0) - clen.to(torch.int64)
    packed = torch.empty(int(clen.sum()) + 64, dtype=torch.uint8, device=dev)
    B.copy_blocks_device(slots.data_ptr(), coff.data_ptr(), packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), nb, st)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device=dev)
    olen = torch.zeros(nb, dtype=torch.int32, device=dev)
    def dec():
        B.decode_batch_device(packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), out.data_ptr(), roff.data_ptr(),
                              rlen.data_ptr(), olen.data_ptr(), nb, st)
    B.decode_stats(0, reset=True)
    dec(); torch.cuda.synchronize()
    stats = B.decode_stats(0, reset=True)
    ok = bool(torch.equal(out, raw)) and bool((olen == bs).all())
    if not ok:
        bad = (olen != bs).nonzero().flatten()[:8].tolist()
        o2 = out.view(nb, bs); r2 = raw.view(nb, bs)
        neq = (o2 != r2).any(dim=1).nonzero().flatten()
        first = neq[:8].tolist()
        detail = ""
        if len(first):
            blk = first[0]
            pos = (o2[blk] != r2[blk]).nonzero().flatten()
            detail = f" first bad block {blk}: {len(pos)} bytes differ, first at {int(pos[0])}, last at {int(pos[-1])}"
        print(f"MISMATCH: bad lengths at {bad} ({int((olen != bs).sum())} blocks), differing blocks {len(neq)} {first}{detail}", flush=True)
    prof = None
    if hasattr(N.lib(), "k4lz4_debug_prof"):
        import ctypes as C
        v = (C.c_uint64 * 32)()
        fn = N.lib().k4lz4_debug_prof
        fn.argtypes = [C.c_void_p, C.c_int32]
        fn(C.addressof(v), 1)
        dec(); torch.cuda.synchronize()
        fn(C.addressof(v), 1)
        names = ["load", "pass1", "validate", "scan", "pass2", "hdr", "lit", "far", "bar1", "nearlist", "nearwork", "nearbar", "endbar", "store", "table"]
        nblk = max(int(v[20]), 1)
        prof = {nm: round(int(v[i]) / nblk) for i, nm in enumerate(names)}
        prof["total"] = sum(prof.values())
        prof.update(valrounds=round(int(v[16]) / nblk, 2), steps=round(int(v[17]) / nblk, 2), subrounds=round(int(v[18]) / nblk, 2), inner=round(int(v[19]) / nblk, 2))
    ms, med = timeit(dec, a.reps)
    if prof: print("   cycles/block (thread 0):", prof, flush=True)
    algo = (int(clen.sum()) + nb * bs)
    print(f"decode[{a.data}{a.mp}]: {ms:.3f} ms (median {med:.3f})  {nb*bs/ms/1e6:.1f} GB/s out  {algo/ms/1e6:.1f} GB/s algorithmic  "
          f"ok={ok} ratio {ratio:.3f} stats {stats}", flush=True)
if a.what == "size":
    import ctypes as C
    import subprocess
    poff = torch.cumsum(clen.to(torch.int64), 0) - clen.to(torch.int64)
    packed = torch.empty(int(clen.sum()) + 64, dtype=torch.uint8, device=dev)
    B.copy_blocks_device(slots.data_ptr(), coff.data_ptr(), packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), nb, st)
    osz = torch.zeros(nb, dtype=torch.int32, device=dev)
    libs = [("shipped", N.lib())] + [(os.path.basename(p), C.CDLL(os.path.abspath(p))) for p in a.size_libs.split(",") if p]
    def size_call(L):
        fn = L.k4lz4_decoded_size_batch
        fn.argtypes, fn.restype = N.SIGNATURES["k4lz4_decoded_size_batch"]
        return lambda: N.check(fn(packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), osz.data_ptr(), nb, N.MEM_DEVICE,
                                  st or None, -1))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    cbytes = int(clen.sum())
    res = {name: [] for name, _ in libs}
    for _ in range(3):
        for name, L in libs:
            f = size_call(L)
            osz.fill_(-7); f(); torch.cuda.synchronize()
            ok = bool((osz == bs).all())
            ms, med = timeit(f, a.reps)
            res[name].append((ms, med, ok))
    for name, rs in res.items():
        best = min(r[0] for r in rs)
        print(f"size[{a.data}{a.mp}] {name}: {best:.3f} ms (medians {', '.join(f'{r[1]:.3f}' for r in rs)})  "
              f"{cbytes/best/1e6:.1f} GB/s compressed  {nb*bs/best/1e6:.1f} GB/s decoded  ok={all(r[2] for r in rs)} "
              f"| {card}", flush=True)
if a.what == "chain":
    from concurrent.futures import ThreadPoolExecutor
    from tests import chain_ref as CR
    Bk = a.chain_blocks
    up = CR.Upstream()
    hraw = raw.cpu().numpy()
    S_all = nb // Bk
    with ThreadPoolExecutor(max_workers=min(64, os.cpu_count() or 1)) as ex:
        comp = list(ex.map(lambda s_: up.encode_chain(hraw[s_ * Bk * bs:(s_ + 1) * Bk * bs].tobytes(), bs), range(S_all)))
    for S in (int(x) for x in a.streams.split(",")):
        steps = []
        for k in range(Bk):
            blocks = [comp[s_][k] for s_ in range(S)]
            ln = np.array([len(b) for b in blocks], dtype=np.int32)
            so = np.zeros(S, dtype=np.int64)
            so[1:] = np.cumsum(ln[:-1])
            steps.append((torch.from_numpy(np.frombuffer(b"".join(blocks), dtype=np.uint8).copy()).to(dev),
                          torch.from_numpy(so).to(dev), torch.from_numpy(ln).to(dev),
                          torch.arange(S, dtype=torch.int64, device=dev) * (Bk * bs) + k * bs,
                          torch.full((S,), bs, dtype=torch.int32, device=dev),
                          torch.full((S,), k * bs, dtype=torch.int32, device=dev)))
        out = torch.zeros(S * Bk * bs, dtype=torch.uint8, device=dev)
        olen = torch.zeros(S, dtype=torch.int32, device=dev)
        def chain():
            for t_src, t_so, t_ln, t_do, t_cap, t_pre in steps:
                B.decode_chain_batch_device(t_src.data_ptr(), t_so.data_ptr(), t_ln.data_ptr(), out.data_ptr(),
                                            t_do.data_ptr(), t_cap.data_ptr(), t_pre.data_ptr(), olen.data_ptr(), S, st)
        B.decode_stats(0, reset=True)
        chain(); torch.cuda.synchronize()
        stats = B.decode_stats(0, reset=True)
        ok = bool(torch.equal(out, raw[:S * Bk * bs]))
        ms, med = timeit(chain, a.reps)
        cbytes = sum(len(comp[s_][k]) for s_ in range(S) for k in range(Bk))
        # the same raw bytes as independent blocks (the GPU encoder's output), one call
        n2 = S * Bk
        poff = torch.cumsum(clen[:n2].to(torch.int64), 0) - clen[:n2].to(torch.int64)
        packed = torch.empty(int(clen[:n2].sum()) + 64, dtype=torch.uint8, device=dev)
        B.copy_blocks_device(slots.data_ptr(), coff.data_ptr(), packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), n2, st)
        out2 = torch.zeros(n2 * bs, dtype=torch.uint8, device=dev)
        olen2 = torch.zeros(n2, dtype=torch.int32, device=dev)
        def indep():
            B.decode_batch_device(packed.data_ptr(), poff.data_ptr(), clen.data_ptr(), out2.data_ptr(), roff.data_ptr(),
                                  rlen.data_ptr(), olen2.data_ptr(), n2, st)
        ms2, med2 = timeit(indep, a.reps)
        ok2 = bool(torch.equal(out2, raw[:n2 * bs]))
        print(f"chain[{a.data}{a.mp}] S={S} B={Bk}: {ms:.3f} ms (median {med:.3f})  {n2*bs/ms/1e6:.1f} GB/s out  "
              f"ratio {cbytes/(n2*bs):.3f} ok={ok} stats {stats} | independent, one call: {ms2:.3f} ms "
              f"{n2*bs/ms2/1e6:.1f} GB/s ok={ok2}", flush=True)
        # the group: device memory, one call per step into the same destination
        gst = torch.arange(S, dtype=torch.int32, device=dev)
        with K.ChainDecoderGroup(S, bs) as g:
            def grp():
                g.reset_device(gst.data_ptr(), S, st)
                for t_src, t_so, t_ln, t_do, t_cap, t_pre in steps:
                    g.decode_device(gst.data_ptr(), t_src.data_ptr(), t_so.data_ptr(), t_ln.data_ptr(), out.data_ptr(),
                                    t_do.data_ptr(), t_cap.data_ptr(), olen.data_ptr(), S, st)
            out.zero_()
            grp(); torch.cuda.synchronize()
            gok = bool(torch.equal(out, raw[:S * Bk * bs]))
            gms, _ = timeit(grp, a.reps)
            # host memory: every step through the group, LZ4ChainDecoder.DecodeMany and one independent call
            hblocks = [[comp[s_][k] for s_ in range(S)] for k in range(Bk)]
            def grp_host():
                g.reset()
                for blocks in hblocks:
                    g.decode(blocks)
            def today_host():
                decs = [K.LZ4ChainDecoder(bs) for _ in range(S)]
                for blocks in hblocks:
                    K.LZ4ChainDecoder.DecodeMany(decs, blocks)
            hpk = clen[:n2].cpu().numpy().reshape(S, Bk)
            hsl = slots.cpu().numpy()
            iblocks = [hsl[(s_ * Bk + 1) * bound:(s_ * Bk + 1) * bound + int(hpk[s_, 1])].tobytes() for s_ in range(S)]
            host = [host_ms(today_host, 1) / Bk, host_ms(grp_host, max(a.reps // 2, 1)) / Bk,
                    host_ms(lambda: B.decode_batch_host(iblocks, [bs] * S), a.reps)]
        report("chain", S, Bk, host, [ms / Bk, gms / Bk, ms2 / Bk])
        print(f"   group ok={gok}", flush=True)
if a.what == "chain-encode":
    from tests import chain_ref as CR
    Bk, SB = a.chain_blocks, N.CHAIN_STATE_BYTES
    up = CR.Upstream()
    hraw = raw.cpu().numpy()
    print("gpu:", torch.cuda.get_device_name(0), flush=True)
    for S in (int(x) for x in a.streams.split(",")):
        n2 = S * Bk
        state = torch.zeros(S * SB, dtype=torch.uint8, device=dev)
        soff = torch.arange(S, dtype=torch.int64, device=dev) * SB
        dstc = torch.empty(S * Bk * bound, dtype=torch.uint8, device=dev)
        steps = [(torch.arange(S, dtype=torch.int64, device=dev) * (Bk * bs) + k * bs,
                  torch.full((S,), k * bs, dtype=torch.int32, device=dev),
                  torch.arange(S, dtype=torch.int64, device=dev) * (Bk * bound) + k * bound,
                  torch.zeros(S, dtype=torch.int32, device=dev)) for k in range(Bk)]
        rl, cc = rlen[:S], ccap[:S]
        def chain(x32=False):
            state.zero_()
            for t_so, t_pre, t_do, t_out in steps:
                B.encode_chain_batch_device(raw.data_ptr(), t_so.data_ptr(), rl.data_ptr(), t_pre.data_ptr(),
                                            dstc.data_ptr(), t_do.data_ptr(), cc.data_ptr(), state.data_ptr(),
                                            soff.data_ptr(), t_out.data_ptr(), S, 0, st, x32=x32)
        B.encode_stats(0, reset=True)
        chain(); torch.cuda.synchronize()
        stats = B.encode_stats(0, reset=True)
        ms, med = timeit(chain, a.reps)
        # spot check: streams 0 and S-1 against upstream's chained encoder
        hd = dstc.cpu().numpy()
        lens = [steps[k][3].cpu().numpy() for k in range(Bk)]
        ok = True
        for s_ in (0, S - 1):
            want = up.encode_chain(hraw[s_ * Bk * bs:(s_ + 1) * Bk * bs].tobytes(), bs)
            for k in range(Bk):
                o = (s_ * Bk + k) * bound
                ok &= int(lens[k][s_]) == len(want[k]) and hd[o:o + len(want[k])].tobytes() == want[k]
        cbytes = sum(int(l.sum()) for l in lens)
        # the 32-bit engine: the same steps, timed alternately with the plain engine, and its own spot check
        from tests import enforce32_ref as E32
        t64, t32 = [], []
        for _ in range(3):
            t64.append(timeit(chain, a.reps)[1]); t32.append(timeit(lambda: chain(True), a.reps)[1])
        chain(True); torch.cuda.synchronize()
        hd32, lens32, ok32 = dstc.cpu().numpy(), [steps[k][3].cpu().numpy() for k in range(Bk)], True
        up32 = E32.EncUpstream32()
        for s_ in (0, S - 1):
            want = up32.encode_chain(hraw[s_ * Bk * bs:(s_ + 1) * Bk * bs].tobytes(), bs)
            for k in range(Bk):
                o = (s_ * Bk + k) * bound
                ok32 &= int(lens32[k][s_]) == len(want[k]) and hd32[o:o + len(want[k])].tobytes() == want[k]
        m64, m32 = float(np.median(t64)), float(np.median(t32))
        import subprocess
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
        print(f"chain-encode-x32[{a.data}{a.mp}] S={S} B={Bk}: plain {m64:.3f} ms {n2*bs/m64/1e6:.1f} GB/s, x32 "
              f"{m32:.3f} ms {n2*bs/m32/1e6:.1f} GB/s (medians of 3 alternating runs of {a.reps}) x32/plain "
              f"{m32/m64:.3f} ratio32 {sum(int(l.sum()) for l in lens32)/(n2*bs):.3f} ok32={ok32} | {card}", flush=True)
        chain(); torch.cuda.synchronize()
        def indep():
            B.encode_batch_device(raw.data_ptr(), roff.data_ptr(), rlen.data_ptr(), slots.data_ptr(), coff.data_ptr(),
                                  ccap.data_ptr(), clen.data_ptr(), n2, 0, st)
        B.encode_stats(0, reset=True)
        indep(); torch.cuda.synchronize()
        stats2 = B.encode_stats(0, reset=True)
        ms2, med2 = timeit(indep, a.reps)
        # host memory: one step (block 1 of every stream, 64 KiB of history each) vs independent encode of it
        import time
        so = (np.arange(S, dtype=np.int64) * (Bk * bs) + bs)
        hs = np.zeros(S * SB, dtype=np.uint8)
        hso = np.arange(S, dtype=np.int64) * SB
        hdst = np.empty(S * bound, dtype=np.uint8)
        hdo = np.arange(S, dtype=np.int64) * bound
        args = (hraw, so, np.full(S, bs, np.int32))
        def host_chain():
            B.encode_chain_batch_host(hraw, so, args[2], np.full(S, bs, np.int32), hdst, hdo, np.full(S, bound, np.int32), hs, hso)
        def host_indep():
            B.encode_batch_flat_host(hraw, so, args[2], hdst, hdo, np.full(S, bound, np.int32))
        th = []
        for fn in (host_chain, host_indep):
            fn()
            t = []
            for _ in range(a.reps):
                t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
            th.append(float(np.median(t)))
        print(f"chain-encode[{a.data}{a.mp}] S={S} B={Bk}: {ms:.3f} ms (median {med:.3f})  {n2*bs/ms/1e6:.1f} GB/s in  "
              f"ratio {cbytes/(n2*bs):.3f} ok={ok} stats {stats} | independent, one call: {ms2:.3f} ms "
              f"{n2*bs/ms2/1e6:.1f} GB/s stats {stats2} | host memory, one step: chained {th[0]:.2f} ms, "
              f"independent {th[1]:.2f} ms, state {2*S*SB/2**20:.1f} MiB moved", flush=True)
        gst = torch.arange(S, dtype=torch.int32, device=dev)
        gout = [torch.zeros(S, dtype=torch.int32, device=dev) for _ in range(Bk)]
        gdst = torch.empty_like(dstc)
        with K.ChainEncoderGroup(S, bs) as g:
            def grp():
                g.reset_device(gst.data_ptr(), S, st)
                for (t_so, t_pre, t_do, t_out), t_g in zip(steps, gout):
                    g.encode_device(gst.data_ptr(), raw.data_ptr(), t_so.data_ptr(), rl.data_ptr(), gdst.data_ptr(),
                                    t_do.data_ptr(), cc.data_ptr(), t_g.data_ptr(), S, 0, st)
            grp(); torch.cuda.synchronize()
            gok = all(torch.equal(gout[k], steps[k][3]) for k in range(Bk))
            gd = gdst.cpu().numpy()
            for k in range(Bk):
                for s_ in range(0, S, 61):
                    o, r = (s_ * Bk + k) * bound, int(lens[k][s_])
                    gok &= gd[o:o + r].tobytes() == hd[o:o + r].tobytes()
            gms, _ = timeit(grp, a.reps)
            hblocks = [[hraw[(s_ * Bk + k) * bs:(s_ * Bk + k + 1) * bs].tobytes() for s_ in range(S)] for k in range(Bk)]
            def grp_host():
                g.reset()
                for blocks in hblocks:
                    g.encode(blocks)
            def today_host():
                encs = [K.LZ4FastChainEncoder(bs) for _ in range(S)]
                tg = [np.empty(bound, np.uint8) for _ in range(S)]
                for blocks in hblocks:
                    for e_, b_ in zip(encs, blocks):
                        e_.Topup(b_)
                    K.LZ4FastChainEncoder.EncodeMany(encs, tg)
            host = [host_ms(today_host, 1) / Bk, host_ms(grp_host, max(a.reps // 2, 1)) / Bk,
                    host_ms(lambda: B.encode_batch_host(hblocks[1]), a.reps)]
        report("chain-encode", S, Bk, host, [ms / Bk, gms / Bk, ms2 / Bk])
        print(f"   group ok={gok}", flush=True)
