"""Whole chained streams in one call (csrc/decode_stream.cuh) restated in Python, and the streams the tests use.

``decode_streams`` runs the four passes of k4lz4_decode_chain_streams over lists of blocks: place (the size walk
and the per-stream scan), the deferred decode of every block on its own (literals and final-source matches
written, the rest recorded on the block's deferred list, a block past the budget marked whole), the verdicts and
the replay in stream order (a block's records that read only earlier blocks first, then the rest in order).  Every
copy it makes asserts that the bytes it reads are already final, so the deferral rule and the replay's order are
checked, not only the end result.  ``step_reference`` is the authority: upstream's
LZ4_decompress_safe_continue stepped block by block (what k4lz4_decode_chain_batch does per call).
"""
from __future__ import annotations

import bisect
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
    whole_blocks: int = 0
    max_copies: int = 0
    per_block: list = field(default_factory=list)


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
                     budget: int):
    """decode_block_warp with DeferOut: -> (r, copies or None for whole).  Block byte x is out[base + x]; [base - off, base)
    are this call's earlier blocks."""
    n = len(src)
    low = -min(P, 65535)
    copies, spans = [], []                     # spans: [lo, hi) deferred intervals, increasing
    whole = False
    ip = op = 0
    iend, oend = n, cap
    shortiend, shortoend = iend - 16, oend - 32

    def copy_match(match: int, length: int, offset: int) -> None:
        nonlocal whole
        if whole:
            return
        lo, hi = match, match + min(length, offset)
        dep = offset != 0 and max(lo, -off) < min(hi, 0)
        if offset != 0 and not dep and hi > 0:
            qlo = max(lo, 0)
            k = bisect.bisect_left(spans, (hi, -1)) - 1
            dep = k >= 0 and spans[k][1] > qlo
        if not dep:
            assert offset == 0 or _final(known, base + lo, base + hi), "a final-source copy reads a deferred byte"
            _periodic(out, base + op, base + match, length, offset)
            known[base + op:base + op + length] = b"\x01" * length
            return
        if len(copies) == budget:
            whole = True
            return
        copies.append((op, length, offset))
        if spans and spans[-1][1] == op:
            spans[-1] = (spans[-1][0], op + length)
        else:
            spans.append((op, op + length))

    def lits(a: int, length: int) -> None:
        if not whole:
            out[base + op:base + op + length] = src[a:a + length]
            known[base + op:base + op + length] = b"\x01" * length

    while True:
        token = src[ip]; ip += 1
        length = token >> 4
        shortcut = length != 15 and ip < shortiend and op <= shortoend
        if not shortcut:
            if length == 15:
                if ip >= iend - 15:
                    return -1, None
                while True:
                    s = src[ip]; ip += 1; length += s
                    if ip >= iend - 15 or s != 255:
                        break
            cpy = op + length
            if cpy > oend - MFLIMIT or ip + length > iend - (2 + 1 + LASTLITERALS):
                if ip + length != iend or cpy > oend:
                    return -1, None
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
                    return -1, None
                if s != 255:
                    break
        length += MINMATCH
        if match < low:
            return -1, None
        if op + length > oend - LASTLITERALS:
            return -1, None
        copy_match(match, length, offset)
        op += length


def decode_streams(streams, budget: int = BUDGET, stats: Stats | None = None):
    """streams: list of (history bytes, prefixLen, [(src, cap, raw)]).  -> list of (outLen list, decoded bytes of
    the stream's region up to its first failing entry)."""
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
                r, cp = _deferred_decode(src, cap, prefix + offs[k], offs[k], out, known, base, budget)
                r2.append(r if r >= 0 else -1); lists.append(cp)
        # passes 3 and 4: verdicts and replay, in stream order
        outlen, failed = [], False
        for k, (src, cap, raw) in enumerate(entries):
            if failed or r2[k] < 0:
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
                # phase A: the records that read only earlier blocks; phase B: the rest, in order
                in_front = [op - offset + min(length, offset) <= 0 for op, length, offset in cp]
                for phase in (True, False):
                    for (op, length, offset), a in zip(cp, in_front):
                        if a != phase:
                            continue
                        assert _final(known, base + op - offset, base + op - offset + min(length, offset))
                        _periodic(out, base + op, base + op - offset, length, offset)
                        known[base + op:base + op + length] = b"\x01" * length
            assert _final(known, base, base + r2[k]), "a byte of an accepted block was never written"
            outlen.append(r2[k])
            if stats is not None and not raw:
                stats.blocks += 1
                stats.out_bytes += r2[k]
                if cp is None:
                    stats.whole_blocks += 1
                    stats.per_block.append(-1)
                else:
                    stats.deferred_copies += len(cp)
                    stats.deferred_bytes += sum(c[1] for c in cp)
                    stats.max_copies = max(stats.max_copies, len(cp))
                    stats.per_block.append(len(cp))
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
