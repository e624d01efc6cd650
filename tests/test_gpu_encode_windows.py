"""GPU tests of the encoder's search batches around the first-batch width (K4_ENC_WIN, csrc/encode_tile.cuh).

The first batch of a search run is W lanes wide, every later one 32.  These inputs put the first hit of runs at
probe 0, W - 1, W, W + 1, 31, 32, 33, 64, 65 and 64k +- 1; put stores with equal hashes on both sides of the W
boundary; make the post-match lane hit with a zero-length literal and overwrite the put(ip-2) inside the first
window; end runs at every lane of the first window; and fill runs with words that share the hash (and the tag of
the global-table warps) with an earlier probe while the bytes differ.  More than 4 224 full blocks go through one
launch, so both warp kinds encode, and every block -- full ones, blocks of 13 bytes and up, 64 KiB - 1 and
65 546 bytes -- must equal the reference engine's bytes.  W is read from the source, so the cases follow the
shipped width (W = 32 keeps every run in full batches, and the cases still pin the serial history)."""
import os
import re

import numpy as np
import pytest

from tests import inputs
from tests import lz4_blocks as LB

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MUL = LB.ENC_HASH_MUL
INV = pow(MUL, -1, 1 << 32)


def shipped_width() -> int:
    src = open(os.path.join(ROOT, "k4os", "compression", "lz4_b200", "csrc", "encode_tile.cuh")).read()
    w = int(re.search(r"#define K4_ENC_WIN (\d+)", src).group(1))
    return 32 if w == 0 else w


def _targets(W: int):
    return sorted({0, max(W - 1, 0), W, W + 1, 31, 32, 33, 64, 65, 127, 128, 129, 191, 192, 193})


def _collide(buf: bytearray, x: int, y: int, rng, tag: bool) -> None:
    """Make the word at x share the hash of the word at y (y + 4 <= x) with different bytes: prod + k keeps bits
    19..31, and bits 3..18 (the 16-bit tag of the global-table warps) too unless `tag`."""
    v = int.from_bytes(buf[y:y + 4], "little")
    prod = (v * MUL) & 0xFFFFFFFF
    if tag:
        k = 8 * int(rng.integers(1, 16))
        if ((prod >> 3) & 0xFFFF) + k // 8 > 0xFFFF:
            k = -k
    else:
        k = int(rng.integers(1, 8 - (prod & 7))) if (prod & 7) < 7 else -int(rng.integers(1, 8))
    buf[x:x + 4] = ((v + k * INV) & 0xFFFFFFFF).to_bytes(4, "little")


def window_block(rng, W: int, n: int = 65536, tail: int = 13, mode: str = "hit") -> bytes:
    """Random bytes with runs planted one after another.  Each run's first hit is meant for probe q (cycling through
    _targets), a copy of the word of an earlier probe of the same run -- of the post-match position for q = 0.
    mode "split": before the hit, words at probes W - 1 and W share the hash of probes 4 and 5 positions earlier
    (alternately with the same and with a different tag).  mode "post": every other match is followed by an
    offset-2 repeat, so that the post-match lane hits with no literal; the others get a word at probe 1 with the
    hash of the put(ip-2) word and a copy of the put(ip-2) word at probe 5, which must see the overwrite.
    The last match ends at n - tail, so the last run ends tail - 13 probes in."""
    buf = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    targets = _targets(W)
    base, t = 1, 0
    while True:
        q = targets[t % len(targets)]
        t += 1
        P = base + LB.probe_advance(q)
        L = 4 + int(rng.integers(0, 16))
        if P + L + 400 > n - tail:
            break
        if mode == "split" and q > W:
            for j in (W - 1, W):
                if j >= 5:
                    _collide(buf, base + j, base + j - 4 - (t & 1), rng, tag=bool(t & 2))
        if mode == "post" and base >= 3 and t % 2 == 0 and q > 5:
            _collide(buf, base + 1, base - 3, rng, tag=bool(t & 4))     # the put(ip-2) word: ip = base - 1
            buf[base + 5:base + 9] = buf[base - 3:base + 1]
        if q == 0:
            src = base - 1
        else:
            s = q - 1 - int(rng.integers(0, min(q, 8)))
            src = base + LB.probe_advance(s)
        for i in range(L):
            buf[P + i] = buf[src + i]
        base = P + L + 1
        if mode == "post" and t % 2 == 1:
            L2 = 4 + int(rng.integers(0, 8))
            E = P + L
            for i in range(L2):
                buf[E + i] = buf[E - 2 + i]
            base = E + L2 + 1
    # the last match: a repeat at distance 3 from base + 3 up to n - tail, broken there
    end = n - tail
    for p in range(base + 3, end):
        buf[p] = buf[p - 3]
    buf[end] = buf[end - 3] ^ 0x5A
    return bytes(buf)


def _run(k4, blocks):
    import torch
    dev = torch.device("cuda", 0)
    nb = len(blocks)
    caps = [k4.LZ4Codec.MaximumOutputSize(len(b)) for b in blocks]
    soff = np.zeros(nb, dtype=np.int64)
    soff[1:] = np.cumsum([len(b) for b in blocks])[:-1]
    doff = np.zeros(nb, dtype=np.int64)
    doff[1:] = np.cumsum(caps)[:-1]
    src = torch.from_numpy(np.frombuffer(b"".join(blocks), dtype=np.uint8).copy()).to(dev)
    dst = torch.full((int(sum(caps)) + 16,), 0xCD, dtype=torch.uint8, device=dev)
    t_soff, t_doff = torch.from_numpy(soff).to(dev), torch.from_numpy(doff).to(dev)
    t_len = torch.tensor([len(b) for b in blocks], dtype=torch.int32, device=dev)
    t_cap = torch.tensor(caps, dtype=torch.int32, device=dev)
    t_out = torch.full((nb,), -7, dtype=torch.int32, device=dev)
    B = k4.batch
    B.encode_stats(0, reset=True)
    B.encode_batch_device(src.data_ptr(), t_soff.data_ptr(), t_len.data_ptr(), dst.data_ptr(), t_doff.data_ptr(),
                          t_cap.data_ptr(), t_out.data_ptr(), nb, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return t_out.cpu().numpy(), dst.cpu().numpy(), doff, B.encode_stats(0, reset=True)


def test_window_edges_through_both_warp_kinds(native, port):
    import k4os.compression.lz4_b200 as k4
    import oracle
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    chk = oracle.best()
    W = shipped_width()
    rng = np.random.default_rng(31)
    blocks = []
    for i in range(96):
        mode = ("hit", "split", "post")[i % 3]
        blocks.append(window_block(rng, W, tail=12 + i % (W + 4), mode=mode))
    for n in (65535, 65546):
        for mode in ("hit", "split", "post"):
            blocks.append(window_block(rng, W, n=n, tail=12 + int(rng.integers(0, W + 4)), mode=mode))
    for i in range(48):
        blocks.append(LB.probe_step_input(rng, tail=12 + i % 2, collide=i % 2 == 1))
    raw = port.datagen(4200 * 65536, 0.55, 0.0, 4322)
    blocks += [raw[i * 65536:(i + 1) * 65536].tobytes() for i in range(4200)]
    n_full = len(blocks)
    assert n_full > 4224
    small = [inputs.gen(kind, z, z) for kind in ("text2", "repeat", "random") for z in range(13, 48)]
    small += [window_block(rng, min(W, 8), n=z, tail=12 + z % 8, mode="hit") for z in (600, 1000, 4096)]
    pos = sorted(rng.choice(n_full + len(small), len(small), replace=False))
    for p, b in zip(pos, small):
        blocks.insert(int(p), b)
    got, dst, doff, st = _run(k4, blocks)
    bad = []
    for i, b in enumerate(blocks):
        r, ref = chk.encode(b)
        o = int(doff[i])
        if int(got[i]) != r or dst[o:o + r].tobytes() != ref:
            bad.append((i, len(b), int(got[i]), r))
    assert not bad, f"{len(bad)} blocks differ from the reference engine, first {bad[:5]}"
    assert st["smem"] > 0 and st["gtab"] > 0 and st["generic"] == 0, st
    assert st["smem"] + st["gtab"] == len(blocks), st
