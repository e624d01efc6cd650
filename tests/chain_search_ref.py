"""Upstream's byU32 fast loop (LZ4_compress_generic with limitedOutput, acceleration 1: orig/lib/lz4.c:851-1240)
restated in plain Python for the chained and dictionary encoders, with a log of where things happen.

``encode`` runs one block in the prefix mode (the `d` bytes of history directly in front of the source:
withPrefix64k) or the extDict mode (the `d` kept bytes of a dictionary in a buffer of its own: usingExtDict,
lz4.c:1626-1631), with hash5 (8 bytes) or hash4 (4 bytes) into 4 096 slots of absolute indices.  It returns
upstream's result, bytes and state record, and an ``Events`` log.

The log places every probe in the batches of chain_search_warp (csrc/encode_chain.cuh): the block's first search
run has no post-match lane, so its probe q sits at lane q % 32 of batch q // 32; every later run follows a
post-match probe (lane 0 of its first batch), so its probe q sits at lane (q + 1) % 32 of batch (q + 1) // 32.
A batch holds the stores the GPU commits together: in a post batch put(ip-2), the post probe and the run's
probes up to the hit or the end.
"""
from __future__ import annotations

from collections import Counter

import numpy as np

from tests import chain_enc_ref as CE
from tests.chain_windows import hash4_12, hash5_12, probe_advance, probe_lane

MINMATCH, MFLIMIT, LASTLITERALS, MAX_DISTANCE = 4, 12, 5, 65535

# every kind the log knows; test_chain_windows_model asserts a count for each
EVENT_KINDS = ("hit", "post_hit", "offset2", "reject_dist", "reject_small", "reject_cmp", "dist_65535",
               "lane_forward", "slot_twice", "slot_thrice", "h2_forward", "same2", "end", "end_committed",
               "catchup_history", "catchup_floor", "straddle", "fail_lit", "fail_match", "fail_last")


class Events:
    """What one or more blocks did.  ``count[kind]`` counts events; ``at[kind]`` is the set of places (probe
    index, lane, layout, ...) each kind was seen at."""

    def __init__(self):
        self.count = Counter()
        self.at = {}

    def add(self, kind: str, where=None):
        assert kind in EVENT_KINDS, kind
        self.count[kind] += 1
        if where is not None:
            self.at.setdefault(kind, set()).add(where)

    def merge(self, other: "Events"):
        self.count.update(other.count)
        for k, v in other.at.items():
            self.at.setdefault(k, set()).update(v)


class _Batch:
    """The stores of one GPU batch in serial order; writer = lane, or -1 for put(ip-2)."""

    def __init__(self, layout: str, h2: int | None = None):
        self.layout, self.h2, self.last = layout, h2, {}
        self.writes = Counter()

    def store(self, h: int, writer: int):
        self.last[h] = writer
        self.writes[h] += 1

    def close(self, ev: Events):
        for h, k in self.writes.items():
            if k >= 2:
                ev.add("slot_twice", self.layout)
            if k >= 3:
                ev.add("slot_thrice", self.layout)
        if self.h2 is not None and self.last.get(self.h2, -1) != -1:
            ev.add("same2", self.last[self.h2])    # a later lane overwrote put(ip-2): the GPU drops that store


def encode(table, current_offset: int, dict_size: int, before: bytes, src: bytes, cap: int,
           h4: bool = False, ext: bool = False):
    """One block.  `before` is the history (prefix mode) or the dictionary (extDict mode, loaded by LZ4_loadDict:
    dict_size = its kept bytes).  The block reads the last d = min(dict_size, len(before)) bytes of it.  The
    state must not need renormalising (currentOffset + n <= 2 GiB).
    -> (result, bytes, state record after, Events)."""
    tab = np.array(table, dtype=np.uint32).copy()
    src = bytes(src)
    n = len(src)
    st = int(current_offset)
    d = min(int(dict_size), len(before))
    ev = Events()
    if ext and d < 4:                                   # lz4.c:1581-1587: a tiny dictionary is dropped
        d, ext = 0, False
    dict_small = d < 65536 and d < st
    hist = bytes(before[len(before) - d:])
    H = hash4_12 if h4 else hash5_12
    unit = 4 if h4 else 8
    after_dsize = n if ext else d + n

    def rd(p: int) -> int:
        return src[p] if p >= 0 else hist[d + p]

    def word(p: int) -> bytes:
        return bytes(rd(p + i) for i in range(4))

    def hash_at(p: int) -> int:
        return H(src[p:p + unit])

    def accept(idx: int, cur: int) -> bool:
        return not (dict_small and idx < st - d) and idx + MAX_DISTANCE >= cur

    def why_not(idx: int) -> str:
        return "reject_small" if dict_small and idx < st - d else "reject_dist"

    out = bytearray()

    def result(r: int):
        return r, bytes(out) if r else b"", CE.make_state(tab, st + n, after_dsize), ev

    def lit_run(k: int, tok: int):
        if k >= 15:
            out[tok] |= 0xF0
            r = k - 15
            while r >= 255:
                out.append(255); r -= 255
            out.append(r)
        else:
            out[tok] |= k << 4

    anchor = 0
    mfl1, mlim = n - MFLIMIT + 1, n - LASTLITERALS
    if n >= 13:
        tab[hash_at(0)] = st                            # :924
        ip = 1
        batch, post = _Batch("first"), False
        while True:
            # ---- a search run from `ip`: probe q at ip + probe_advance(q), :956-1014
            base, q, found = ip, 0, None
            layout = "post" if post else "first"
            while True:
                lane = probe_lane(q, post)
                if lane == 0 and q > 0:                 # the next batch of the run
                    batch.close(ev)
                    batch = _Batch(layout)
                p = base + probe_advance(q)
                if base + probe_advance(q + 1) > mfl1:  # :969, the run ends at lane `lane`
                    ev.add("end", (lane, layout))
                    if batch.writes:
                        ev.add("end_committed", lane)
                    batch.close(ev)
                    break
                h = hash_at(p)
                idx, cur = int(tab[h]), st + p
                w = batch.last.get(h)
                if w == -1:
                    ev.add("h2_forward", lane)
                elif w is not None:
                    ev.add("lane_forward", (lane - w, layout))
                tab[h] = cur
                batch.store(h, lane)
                if not accept(idx, cur):
                    ev.add(why_not(idx), (q, lane, layout))
                elif word(idx - st) == src[p:p + 4]:
                    ev.add("hit", (q, layout))
                    if cur - idx == MAX_DISTANCE:
                        ev.add("dist_65535", lane)
                    batch.close(ev)
                    found = (p, idx - st)
                    break
                else:
                    ev.add("reject_cmp", (q, lane, layout))
                q += 1
            if found is None:
                break
            ip, m = found
            zero_lit = False
            while True:                                 # the match at (ip, m); zero_lit: the post probe's
                if not zero_lit:                        # catch-up down to lowLimit, :1019
                    low = (-d if m < 0 else 0) if ext else -d
                    c = 0
                    while ip > anchor and m > low and rd(ip - 1) == rd(m - 1):
                        ip -= 1; m -= 1; c += 1
                    if c and m < 0:
                        ev.add("catchup_history", "ext" if ext else "prefix")
                    if ip > anchor and m == low:
                        ev.add("catchup_floor", ("dict" if low < 0 else "src") if ext else "prefix")
                lit = ip - anchor
                if not zero_lit and len(out) + 1 + lit + 8 + lit // 255 > cap:   # :1024-1027
                    ev.add("fail_lit", len(out))
                    return result(0)
                tok = len(out)
                out.append(0)
                if not zero_lit:
                    lit_run(lit, tok)
                    out += src[anchor:ip]
                off = ip - m
                out += bytes([off & 0xFF, off >> 8])
                # LZ4_count(ip + 4, m + 4, matchlimit); an extDict dictionary match runs on into src[0] (:1078-1089)
                a, b = ip + MINMATCH, m + MINMATCH
                k = 0
                while a + k < mlim and src[a + k] == rd(b + k):
                    k += 1
                if ext and m < 0 and b + k >= 0:
                    ev.add("straddle", (-b, min(b + k, 8)))
                if len(out) + 1 + LASTLITERALS + (k + 240) // 255 > cap:      # :1097-1121
                    ev.add("fail_match", len(out))
                    return result(0)
                if k >= 15:
                    out[tok] += 15
                    r = k - 15
                    while r >= 255:
                        out.append(255); r -= 255
                    out.append(r)
                else:
                    out[tok] += k
                ip += k + MINMATCH
                anchor = ip
                if ip >= mfl1:                          # :1143
                    break
                h2 = hash_at(ip - 2)                    # put(ip-2) and the post probe, :1146-1197
                tab[h2] = st + ip - 2
                batch = _Batch("post", h2)
                batch.store(h2, -1)
                h = hash_at(ip)
                idx, cur = int(tab[h]), st + ip
                if h == h2:
                    ev.add("h2_forward", 0)
                tab[h] = cur
                batch.store(h, 0)
                if accept(idx, cur) and word(idx - st) == src[ip:ip + 4]:
                    ev.add("post_hit", "h2" if h == h2 else "table")
                    if ip - (idx - st) == 2:
                        ev.add("offset2")
                    batch.close(ev)
                    m = idx - st
                    zero_lit = True
                    continue
                if not accept(idx, cur):
                    ev.add(why_not(idx), (-1, 0, "post"))
                else:
                    ev.add("reject_cmp", (-1, 0, "post"))
                ip += 1
                post = True
                break
            if anchor >= mfl1:
                break
    run = n - anchor                                    # last literals, :1204-1231
    if len(out) + run + 1 + (run + 255 - 15) // 255 > cap:
        ev.add("fail_last", len(out))
        return result(0)
    out.append(0)
    lit_run(run, len(out) - 1)
    out += src[anchor:]
    return result(len(out))


def upstream_ext(up, dictionary: bytes, src: bytes, cap: int):
    """Upstream's extDict block with its state: LZ4_loadDict(dictionary) in a buffer of its own, then
    LZ4_compress_fast_continue.  `up` is a dict_enc_ref.DictUpstream.  -> (result, bytes, state record after)."""
    dic = np.frombuffer(bytes(dictionary) + b"\0" * 8, dtype=np.uint8)
    s = np.frombuffer(bytes(src) + b"\0" * 8, dtype=np.uint8)
    st = up.lib.LZ4_createStream()
    try:
        up.lib.LZ4_loadDict(st, dic.ctypes.data, len(dictionary))
        r, out = up.compress(st, s.ctypes.data, len(src), cap)
        return r, out, up.state_of(st)
    finally:
        up.lib.LZ4_freeStream(st)


def run_case(c):
    """The restatement on a chain_windows.Case -> (result, bytes, state record after, Events)."""
    if c.ext:
        from tests import dict_enc_ref as DR
        loaded = DR.load_table(c.before).view(np.uint32)
        return encode(loaded[:4096], 65536, int(loaded[4097]), c.before, c.src, c.cap, ext=True)
    s = c.state.view(np.uint32)
    return encode(s[:4096], int(s[4096]), int(s[4097]), c.before, c.src, c.cap, h4=c.h4)


def upstream_case(up, up32, c):
    """Upstream on a chain_windows.Case -> (result, bytes, state record after)."""
    if c.ext:
        return upstream_ext(up, c.before, c.src, c.cap)
    return (up32 if c.h4 else up).step(c.state, c.before, c.src, c.cap)
