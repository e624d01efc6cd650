"""tools/enc_traffic.py -- CPU model of the block encoder's memory requests per sequence.

    python tools/enc_traffic.py [--blocks 16] [--wins 32,16,8,4] [--mp 550]

Replays the L00_FAST matcher for blocks below 64 KiB + 11 bytes (LL64.fast.cs, byU16 table) the way
`encode_spec_warp` (csrc/encode_tile.cuh) evaluates it: batches of lanes, one probe per lane, the first batch of
each search run `win` lanes wide (K4_ENC_WIN) and every later one 32, the put(ip-2) of the post-match probe and
the stores of earlier lanes forwarded to later lanes, the stores of lanes up to the first hit committed.  It
emits the LZ4 block, so the counts can be pinned to the real parse (tests/test_enc_traffic_model.py compares
the bytes with the oracle), and counts per batch what each table layout loads.  Mode 0 is the shared-memory
warps' (plain u16 slots), mode 2 the global-table warps' (32-bit slots, position | 16-bit tag); mode 3 (an 8-bit
tag table in front of the u16 slots) was measured on the GPU and is not in the encoder (DESIGN §7.2):

  probe words      4-byte reads of the lanes' own positions (two LDGs where the position is not 4-aligned)
  slot loads       mode 2: one 32-bit slot per lane
  tag loads        mode 3: one 8-bit tag per lane ...
  pos loads        ... and the 16-bit position, only where the tag agrees and no earlier store is forwarded
  cand words       4-byte candidate reads: mode 0 on every lane, modes 2 / 3 where the tag agrees; counted in
                   LDGs as above

The data is the bench's encode input (the reference generator, matchProba mp/1000, seed 1234 + chunk), from
the first block on.  The model counts requests, not time: which variant is faster is measured on the GPU.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

MUL = 2654435761
MINMATCH, LASTLITERALS, MFLIMIT, MINLENGTH = 4, 5, 12, 13
COUNTERS = ("seqs", "runs", "probes", "batches", "lanes", "probe_ldg", "slot", "tag3", "pos3",
            "cand0", "cand2", "cand3")


def probe_advance(q: int) -> int:
    """Distance of search probe q from probe 0 of its run (encode_tile.cuh probe_advance, LL64.fast.cs:159-170)."""
    if q <= 64:
        return q
    c = 63 + q
    k = c >> 6
    return 1 + 32 * k * (k - 1) + (c - 64 * k) * k


def _ldg(p: int) -> int:
    return 1 if (p & 3) == 0 else 2


def _run_header(out: bytearray, lit: int, ml_tok: int) -> None:
    if lit >= 15:
        out.append(0xF0 | ml_tok)
        rest = lit - 15
        while rest >= 255:
            out.append(255)
            rest -= 255
        out.append(rest)
    else:
        out.append((lit << 4) | ml_tok)


def encode_block(src: bytes, win: int = 32):
    """-> (LZ4 block of `src` at L00_FAST with full output capacity, counters).  len(src) < 65 547."""
    n = len(src)
    assert n < 65536 + 11
    win = 32 if win in (0, 32) else win
    cnt = dict.fromkeys(COUNTERS, 0)
    out = bytearray()
    anchor = 0
    if n >= MINLENGTH:
        w = np.frombuffer(src, dtype=np.uint8).astype(np.uint32)
        V = (w[:-3] | (w[1:-2] << 8) | (w[2:-1] << 16) | (w[3:] << 24)).tolist()
        prod = [(v * MUL) & 0xFFFFFFFF for v in V]
        H = [p >> 19 for p in prod]
        TAG2 = [(p >> 3) & 0xFFFF for p in prod]
        TAG3 = [(p >> 11) & 0xFF for p in prod]
        T = [0] * 8192
        mfl1, mlim = n - MFLIMIT + 1, n - LASTLITERALS
        T[H[0]] = 0
        ip, post, q0, base, width = 1, False, 0, 1, win
        run_probes = 0
        while True:
            # one batch: lane 0 is the post-match probe at ip when `post`, the others search probes q0, q0 + 1, ...
            cnt["batches"] += 1
            cnt["lanes"] += width
            view = {H[ip - 2]: ip - 2} if post else {}
            hit, lanes = None, []
            for lane in range(width):
                is_post = post and lane == 0
                q = q0 + lane - (1 if post else 0)
                pos = ip if is_post else base + probe_advance(q)
                if not (is_post or base + probe_advance(q + 1) <= mfl1):
                    break                                   # the end of the run; every later lane is past it too
                h = H[pos]
                fwd = h in view
                cand = view[h] if fwd else T[h]
                cnt["probe_ldg"] += _ldg(pos)
                cnt["slot"] += 1
                cnt["tag3"] += 1
                cnt["cand0"] += _ldg(cand)
                if TAG2[cand] == TAG2[pos]:
                    cnt["cand2"] += _ldg(cand)
                if TAG3[cand] == TAG3[pos]:
                    cnt["cand3"] += _ldg(cand)
                    cnt["pos3"] += 0 if fwd else 1
                view[h] = pos
                lanes.append((pos, cand))
                if hit is None and V[cand] == V[pos]:
                    hit = lane
            ended = len(lanes) < width
            if hit is None and ended:
                run_probes += len(lanes)
                cnt["probes"] += run_probes
                cnt["runs"] += 1
                break                                       # last literals
            upto = len(lanes) if hit is None else hit + 1
            run_probes += upto
            if post:
                T[H[ip - 2]] = ip - 2
            for pos, _ in lanes[:upto]:
                T[H[pos]] = pos
            if hit is None:
                if post:
                    post, base, q0 = False, ip + 1, width - 1
                else:
                    q0 += width
                width = 32
                continue
            cnt["probes"] += run_probes
            cnt["runs"] += 1
            run_probes = 0
            zero_lit = post and hit == 0
            ip, m = lanes[hit]
            hip, hm = ip, m
            if not zero_lit:                                # catch-up, LL64.fast.cs:237-242
                while ip > anchor and m > 0 and src[ip - 1] == src[m - 1]:
                    ip -= 1
                    m -= 1
            a, b = hip + MINMATCH, hm + MINMATCH            # LZ4_count from the hit: [ip, hip + 4) is equal
            while a < mlim and src[a] == src[b]:
                a += 1
                b += 1
            mc = a - ip - MINMATCH
            lit = ip - anchor
            _run_header(out, lit, min(mc, 15))
            out += src[anchor:ip]
            out += (ip - m).to_bytes(2, "little")
            if mc >= 15:
                rest = mc - 15
                out += b"\xFF" * (rest // 255)
                out.append(rest % 255)
            cnt["seqs"] += 1
            ip = a
            anchor = ip
            if ip >= mfl1:
                break
            post, q0, base, width = True, 0, ip + 1, win
    run = n - anchor
    _run_header(out, run, 0)
    out += src[anchor:]
    return bytes(out), cnt


def per_sequence(cnt: dict) -> dict:
    s = max(cnt["seqs"], 1)
    return {
        "probes/run": cnt["probes"] / max(cnt["runs"], 1),
        "batches/seq": cnt["batches"] / s,
        "probe LDG/seq": cnt["probe_ldg"] / s,
        "mode 2: slot/seq": cnt["slot"] / s,
        "mode 2: cand LDG/seq": cnt["cand2"] / s,
        "mode 3: tag/seq": cnt["tag3"] / s,
        "mode 3: pos/seq": cnt["pos3"] / s,
        "mode 3: cand LDG/seq": cnt["cand3"] / s,
        "mode 0: cand LDG/seq": cnt["cand0"] / s,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=16)
    ap.add_argument("--wins", default="32,16,8,4")
    ap.add_argument("--mp", type=int, default=550)
    a = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    raw = bench.gen_blocks(a.blocks, a.mp / 1000.0, 0)
    bs = bench.BLOCK
    rows, first = {}, None
    for win in (int(x) for x in a.wins.split(",")):
        tot = dict.fromkeys(COUNTERS, 0)
        outs = []
        for i in range(a.blocks):
            o, c = encode_block(raw[i * bs:(i + 1) * bs].tobytes(), win)
            outs.append(o)
            for k in COUNTERS:
                tot[k] += c[k]
        if first is None:
            first = outs
        assert outs == first, "the window must not change the parse"
        rows[win] = per_sequence(tot)
        rows[win]["seqs/block"] = tot["seqs"] / a.blocks
        ratio = sum(len(o) for o in outs) / (a.blocks * bs)
    print(f"{a.blocks} blocks of 64 KiB, datagen {a.mp / 1000}, ratio {ratio:.4f}")
    keys = list(next(iter(rows.values())))
    print(f"{'first-batch lanes':24s}" + "".join(f"{w:>10d}" for w in rows))
    for k in keys:
        print(f"{k:24s}" + "".join(f"{rows[w][k]:10.2f}" for w in rows))


if __name__ == "__main__":
    main()
