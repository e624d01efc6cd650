"""Whole chained streams in one call (csrc/decode_stream.cuh) restated in Python, and the streams the tests use.

``decode_streams`` runs the four passes of k4lz4_decode_chain_streams over lists of blocks: place (the size walk
and the per-stream scan), the deferred decode of every block on its own (literals and final-source matches
written, the rest recorded on the block's deferred list, a block past the budget marked whole), the verdicts and
the replay in stream order.  It makes the kernel's decisions in the kernel's form: the own-block test through the
last deferred interval and a binary search over the unmerged records (checked against merged spans at every match),
phase A in groups of 32 and phase B in the kernel's runs of lanes.  Every run of copies the kernel makes at the same
time asserts that all the bytes it reads are final before any of it is written, so the deferral rule and the
replay's partition are checked, not only the end result; ``Stats`` counts which rule decided what.  ``step_reference`` is the authority: upstream's
LZ4_decompress_safe_continue stepped block by block (what k4lz4_decode_chain_batch does per call).
"""
from __future__ import annotations

import bisect
from collections import Counter
from dataclasses import dataclass, field

from tests import chain_ref as CR

MINMATCH, MFLIMIT, LASTLITERALS = 4, 12, 5
BUDGET = 2048                         # K4_DS_BUDGET


def walk(s: bytes) -> int:
    """The decoded length of a token chain (size_walk.cuh), -1 where it runs past the end."""
    n, p, out = len(s), 0, 0
    if n <= 0:
        return -1
    while True:
        tok = s[p]; p += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if p >= n:
                    return -1
                x = s[p]; p += 1; lit += x
                if x != 255:
                    break
        p += lit
        if p == n:
            return out + lit
        if p + 2 > n:
            return -1
        p += 2
        ml = tok & 15
        if ml == 15:
            while True:
                if p >= n:
                    return -1
                x = s[p]; p += 1; ml += x
                if x != 255:
                    break
        if p >= n:
            return -1
        out += lit + ml + 4


@dataclass
class Stats:
    out_bytes: int = 0
    deferred_bytes: int = 0
    deferred_copies: int = 0
    blocks: int = 0
    whole_blocks: int = 0                  # accepted blocks decoded whole
    max_copies: int = 0
    per_block: list = field(default_factory=list)
    # pass 2: which test of DeferOut::match decided each match with a nonzero offset
    dec_earlier: int = 0                   # deferred: the source touches an earlier block of the call
    dec_last: int = 0                      # deferred: the source touches the last deferred interval
    dec_search: int = 0                    # deferred: the binary search over the older records found one
    dec_gap: int = 0                       # written: the search ran and the source lies between intervals
    whole_failed: int = 0                  # blocks over the budget that then fail (the stream's first failure)
    whole_prewritten: int = 0              # blocks over the budget after pass 2 wrote some of their bytes
    # pass 4
    phase_a: int = 0                       # phase-A records
    phase_a_long: int = 0                  # ... longer than the lane copy (one by one with the whole warp)
    runs: int = 0                          # phase-B windows
    stops_dep: int = 0                     # windows stopped by a lane that reads an earlier lane's destination
    stops_len: int = 0                     # ... by a long lane
    stop_lanes: Counter = field(default_factory=Counter)
    dep_pairs: Counter = field(default_factory=Counter)      # (earlier lane, stop lane) of every dependency stop
    cross_window: int = 0                  # phase-B records reading a record of the window before theirs


@dataclass(frozen=True)
class Rules:
    """The replay's partition rules (decode_stream.cuh replay_block).  The defaults are the kernel's; the others
    exist so that a test can check that the model's finality assertions catch a wrong rule."""
    lane_copy: int = 64                    # DS_LANE_COPY
    dep_gap: int = 0                       # lane i is an earlier lane of lane l when i + dep_gap < l
    phase_a_hi: int = 0                    # phase A: the source ends at or before block byte phase_a_hi


KERNEL = Rules()


def _periodic(buf: bytearray, at: int, match: int, length: int, offset: int) -> None:
    if offset == 0:
        buf[at:at + length] = bytes(length)
    elif offset >= length:
        buf[at:at + length] = buf[match:match + length]
    else:
        pat = bytes(buf[match:match + offset])
        buf[at:at + length] = (pat * (length // offset + 1))[:length]


def _final(known: bytearray, a: int, b: int) -> bool:
    return known.find(0, a, b) < 0


def _deferred_decode(src: bytes, cap: int, P: int, off: int, out: bytearray, known: bytearray, base: int,
                     budget: int, st: Stats):
    """decode_block_warp with DeferOut: -> (r, copies or None for whole), also for a failing block.  Block byte x is
    out[base + x]; [base - off, base) are this call's earlier blocks.  The own-block test is made twice: in the
    kernel's form (the last interval in registers, then a binary search over the unmerged records before it) and over
    merged spans; the two must agree at every match."""
    n = len(src)
    low = -min(P, 65535)
    copies, spans = [], []                     # spans: [lo, hi) deferred intervals, increasing
    last_lo, last_hi = 0, -1                   # DeferOut::lastLo / lastHi
    whole = False
    written = 0                                # bytes pass 2 wrote
    ip = op = 0
    iend, oend = n, cap
    shortiend, shortoend = iend - 16, oend - 32

    def copy_match(match: int, length: int, offset: int) -> None:
        nonlocal whole, last_lo, last_hi, written
        if whole:
            return
        lo, hi = match, match + min(length, offset)
        dep = offset != 0 and max(lo, -off) < min(hi, 0)
        if offset != 0:
            st.dec_earlier += dep
        if offset != 0 and not dep and hi > 0:
            qlo = max(lo, 0)
            k = bisect.bisect_left(spans, (hi, -1)) - 1
            by_spans = k >= 0 and spans[k][1] > qlo
            # DeferOut::match
            dep = last_lo < hi and last_hi > qlo
            st.dec_last += dep
            if not dep and len(copies) > 1 and qlo < last_lo:
                a, b = 0, len(copies) - 2
                while a < b:
                    m = (a + b + 1) >> 1
                    if copies[m][0] < hi:
                        a = m
                    else:
                        b = m - 1
                c_op, c_len, _ = copies[a]
                dep = c_op < hi and c_op + c_len > qlo
                st.dec_search += dep
                st.dec_gap += not dep and c_op < hi
            assert dep == by_spans, ("the kernel's own-block test and the spans disagree", match, length, offset)
        if not dep:
            assert offset == 0 or _final(known, base + lo, base + hi), "a final-source copy reads a deferred byte"
            _periodic(out, base + op, base + match, length, offset)
            known[base + op:base + op + length] = b"\x01" * length
            written += length
            return
        if len(copies) == budget:
            whole = True
            st.whole_prewritten += written > 0
            return
        copies.append((op, length, offset))
        last_lo, last_hi = op, op + length
        if spans and spans[-1][1] == op:
            spans[-1] = (spans[-1][0], op + length)
        else:
            spans.append((op, op + length))

    def lits(a: int, length: int) -> None:
        nonlocal written
        if not whole:
            out[base + op:base + op + length] = src[a:a + length]
            known[base + op:base + op + length] = b"\x01" * length
            written += length

    def fail():
        return -1, (None if whole else copies)

    while True:
        token = src[ip]; ip += 1
        length = token >> 4
        shortcut = length != 15 and ip < shortiend and op <= shortoend
        if not shortcut:
            if length == 15:
                if ip >= iend - 15:
                    return fail()
                while True:
                    s = src[ip]; ip += 1; length += s
                    if ip >= iend - 15 or s != 255:
                        break
            cpy = op + length
            if cpy > oend - MFLIMIT or ip + length > iend - (2 + 1 + LASTLITERALS):
                if ip + length != iend or cpy > oend:
                    return fail()
                lits(ip, length)
                return op + length, (None if whole else copies)
        lits(ip, length)
        ip += length; op += length
        offset = src[ip] | (src[ip + 1] << 8); ip += 2
        match = op - offset
        length = token & 15
        if shortcut and length != 15 and offset >= 8 and match >= low:
            copy_match(match, length + MINMATCH, offset)
            op += length + MINMATCH
            continue
        if length == 15:
            while True:
                s = src[ip]; ip += 1; length += s
                if ip >= iend - LASTLITERALS + 1:
                    return fail()
                if s != 255:
                    break
        length += MINMATCH
        if match < low:
            return fail()
        if op + length > oend - LASTLITERALS:
            return fail()
        copy_match(match, length, offset)
        op += length


def _run(out: bytearray, known: bytearray, base: int, recs) -> None:
    """Records copied at the same time (the lanes of one run, or one record by the whole warp): every byte any of
    them reads must be final before the first of them writes."""
    for op, length, offset in recs:
        lo = base + op - offset
        assert _final(known, lo, lo + min(length, offset)), "a replay run reads a byte that is not final yet"
    for op, length, offset in recs:
        _periodic(out, base + op, base + op - offset, length, offset)
        known[base + op:base + op + length] = b"\x01" * length


def _replay(out: bytearray, known: bytearray, base: int, cp, rules: Rules, st: Stats) -> None:
    """replay_block: phase A in groups of 32 (the short records together, then the long ones one by one), then
    phase B in windows of 32 that stop at the first lane that reads an earlier phase-B lane's destination or is long:
    the lanes before it together, then it alone, and the next window starts behind it."""
    nd = len(cp)
    src_hi = [op - offset + min(length, offset) for op, length, offset in cp]
    for k0 in range(0, nd, 32):
        grp = [cp[k] for k in range(k0, min(k0 + 32, nd)) if src_hi[k] <= rules.phase_a_hi]
        _run(out, known, base, [c for c in grp if c[1] <= rules.lane_copy])
        for c in grp:
            if c[1] > rules.lane_copy:
                _run(out, known, base, [c])
                st.phase_a_long += 1
        st.phase_a += len(grp)
    k, prev = 0, []
    while k < nd:
        lanes = [j for j in range(k, min(k + 32, nd))]
        b = [src_hi[j] > 0 for j in lanes]
        m, why, pairs = 32, None, []
        for lane, j in enumerate(lanes):
            if not b[lane]:
                continue
            op, length, offset = cp[j]
            lo, hi = op - offset, src_hi[j]
            deps = [i for i in range(31) if i + rules.dep_gap < lane and b[i] and cp[lanes[i]][0] < hi
                    and cp[lanes[i]][0] + cp[lanes[i]][1] > lo]
            st.cross_window += any(p_op < hi and p_op + p_len > lo for p_op, p_len, _ in prev)
            if deps or length > rules.lane_copy:
                m, why, pairs = lane, ("dep" if deps else "len"), deps
                break
        _run(out, known, base, [cp[lanes[i]] for i in range(min(m, len(lanes))) if b[i]])
        st.runs += 1
        if m < 32:
            _run(out, known, base, [cp[lanes[m]]])
            st.stop_lanes[m] += 1
            st.stops_dep += why == "dep"
            st.stops_len += why == "len"
            st.dep_pairs.update((i, m) for i in pairs)
            prev = [cp[lanes[i]] for i in range(m + 1) if b[i]]
            k += m + 1
        else:
            prev = [cp[lanes[i]] for i in range(len(lanes)) if b[i]]
            k += 32


def decode_streams(streams, budget: int = BUDGET, stats: Stats | None = None, rules: Rules = KERNEL):
    """streams: list of (history bytes, prefixLen, [(src, cap, raw)]).  -> list of (outLen list, decoded bytes of
    the stream's region up to its first failing entry)."""
    st = stats if stats is not None else Stats()
    res = []
    for hist, prefix, entries in streams:
        # pass 1: place
        sizes = []
        for src, cap, raw in entries:
            if raw:
                sizes.append(len(src) if 0 <= len(src) <= cap else 0)
            elif len(src) > 0 and cap > 0:
                w = walk(src)
                sizes.append(0 if w < 0 else min(w, cap))
            else:
                sizes.append(0)
        offs = [0]
        for z in sizes[:-1]:
            offs.append(offs[-1] + z)
        H = len(hist)
        total = sum(max(c, 0) for _, c, _ in entries)
        out = bytearray(hist) + bytearray(total + 16)
        known = bytearray(b"\x01" * H) + bytearray(total + 16)
        # pass 2: every block on its own
        r2, lists = [], []
        for k, (src, cap, raw) in enumerate(entries):
            base = H + offs[k]
            if raw:
                ok = 0 <= len(src) <= cap
                if ok:
                    out[base:base + len(src)] = src
                    known[base:base + len(src)] = b"\x01" * len(src)
                r2.append(len(src) if ok else -1); lists.append([])
            elif len(src) <= 0 or cap <= 0:
                r2.append(0 if cap == 0 and len(src) == 1 and src[0] == 0 else -1); lists.append([])
            else:
                r, cp = _deferred_decode(src, cap, prefix + offs[k], offs[k], out, known, base, budget, st)
                r2.append(r if r >= 0 else -1); lists.append(cp)
        # passes 3 and 4: verdicts and replay, in stream order
        outlen, failed = [], False
        for k, (src, cap, raw) in enumerate(entries):
            if failed or r2[k] < 0:
                st.whole_failed += not failed and lists[k] is None
                failed = True
                outlen.append(-1)
                continue
            base = H + offs[k]
            cp = lists[k]
            if cp is None:
                P = min(prefix + offs[k], 65535)
                assert _final(known, base - min(P, base), base)
                r, data = CR.decompress_prefix(src, cap, bytes(out[base - P:base]) if P else b"")
                assert r == r2[k]
                out[base:base + r] = data
                known[base:base + r] = b"\x01" * r
            else:
                _replay(out, known, base, cp, rules, st)
            assert _final(known, base, base + r2[k]), "a byte of an accepted block was never written"
            outlen.append(r2[k])
            if not raw:
                st.blocks += 1
                st.out_bytes += r2[k]
                if cp is None:
                    st.whole_blocks += 1
                    st.per_block.append(-1)
                else:
                    st.deferred_copies += len(cp)
                    st.deferred_bytes += sum(c[1] for c in cp)
                    st.max_copies = max(st.max_copies, len(cp))
                    st.per_block.append(len(cp))
        good = sum(r for r in outlen if r > 0)
        res.append((outlen, bytes(out[H:H + good])))
    return res


def step_reference(up: CR.Upstream, hist: bytes, prefix: int, entries):
    """Upstream stepped block by block behind the stream's history: -> (outLen list, decoded bytes up to the first
    failure).  A stored entry is copied as-is."""
    assert prefix == len(hist)
    seen = bytearray(hist)
    outlen, failed, got = [], False, bytearray()
    for src, cap, raw in entries:
        if failed:
            outlen.append(-1)
            continue
        if raw:
            r, data = (len(src), src) if 0 <= len(src) <= cap else (-1, b"")
        elif len(src) <= 0 or cap < 0:
            r, data = -1, b""
        else:
            h = bytes(seen[-min(len(seen), 65536):]) if seen else b""
            r, data = up.decode_prefix(src, cap, h)
        if r < 0:
            failed = True
            outlen.append(-1)
            continue
        outlen.append(r)
        seen += data
        got += data
    return outlen, bytes(got)
