"""Adversarial chained streams for k4lz4_decode_chain_streams (csrc/decode_stream.cuh, DESIGN 4.11).

Each family aims at one rule of the call's scheduling: where pass 2 draws the line between a final and a deferred
source, and how the replay partitions a block's deferred records (phase A in groups of 32, phase B in runs that stop
at a dependency or a long record, the whole-block path past the budget).  Blocks are built with
chain_ref.build_prefix_block from matches placed by their source position, so every boundary is exact.  The
sources that probe a boundary sit on bytes that are themselves deferred: pass 2 does not write those before the
replay, so a wrong verdict reads the destination's previous content (the GPU tests fill it with FILL) every time
instead of depending on a race.  No decoded byte equals FILL: literals and histories are drawn from 1..200.

``families()`` -> {name: Family}.  ``Family.target(stats)`` returns the coverage each family must reach in the
model's counters (tests/chain_stream_ref.Stats) as {what: bool}.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

from tests import block_mutants as BM
from tests import chain_ref as CR
from tests import lz4_blocks as LB

FILL = 0xCD
K4, K64 = 4096, 65536


def lits(rng, n: int) -> bytes:
    return rng.integers(1, 201, n, dtype=np.uint8).tobytes()


@dataclass
class Family:
    name: str
    streams: list                       # [(history, [(src, cap, raw)])]
    target: object                      # Stats -> {what: bool}
    zero_offset: bool = False           # content unspecified upstream: compare bytes with the model only


class Stream:
    """One chained stream under construction.  Matches are placed by their source position relative to the start of
    the block being built (negative: history or earlier blocks), so offset = op - src."""

    def __init__(self, rng, history: int | bytes = 0):
        self.rng = rng
        self.hist = history if isinstance(history, bytes) else lits(rng, history)
        self.content = bytearray(self.hist)
        self.entries = []
        self.starts = []                # each entry's first byte in the stream's content (history included)

    @property
    def at(self) -> int:
        return len(self.content)

    def block(self, items, last: int = 16, cap=None):
        """items: ("L", n) literals | ("M", src, ml) a match reading block position src | ("O", off, ml) a match by
        offset | ("Z", ml) a match with offset 0.  Returns the decoded size."""
        seqs, pend, op, zeros = [], b"", 0, []
        for it in items:
            if it[0] == "L":
                pend += lits(self.rng, it[1]); op += it[1]
            else:
                if it[0] == "Z":
                    off, ml = 1, it[1]
                    zeros.append(len(seqs))
                else:
                    off = op - it[1] if it[0] == "M" else it[1]
                    ml = it[2]
                seqs.append((pend, off, ml)); pend = b""; op += ml
        tail = pend + lits(self.rng, last)
        src, dec = CR.build_prefix_block(bytes(self.content[-K64:]), seqs, tail)
        if zeros:
            m, pos = bytearray(src), 0
            for i, (lt, off, ml) in enumerate(seqs):
                pos += 1 + _ext_len(len(lt)) + len(lt)
                if i in zeros:
                    m[pos:pos + 2] = b"\0\0"
                pos += 2 + _ext_len(ml - 4, 15)
            src = bytes(m)
            r, dec = CR.decompress_prefix(src, len(dec), bytes(self.content[-K64:]))
            assert r == len(dec)
        size = len(dec)
        c = size if cap is None else cap
        self.starts.append(self.at)
        self.entries.append((src, c, False))
        if c >= size:
            self.content += dec
        return size

    def stored(self, data: bytes, cap=None):
        self.starts.append(self.at)
        self.entries.append((data, len(data) if cap is None else cap, True))
        self.content += data

    def zero_size(self):
        self.starts.append(self.at)
        self.entries.append((b"\x00", 0, False))

    def rel(self, k: int, x: int = 0) -> int:
        """block position (of the block about to be built) of byte x of entry k"""
        return self.starts[k] + x - self.at

    def out(self):
        return self.hist, list(self.entries)


def _ext_len(v: int, lim: int = 15) -> int:
    return len(LB._ext(v - lim)) if v >= lim else 0


def _filler(s: Stream, size: int, items, last: int = 16):
    """items, then literals up to a decoded size of exactly `size`"""
    used = sum(it[1] if it[0] == "L" else it[-1] for it in items)
    return s.block(list(items) + [("L", size - used - last)], last=last)


# ---- families -------------------------------------------------------------------------------------------------

def history_boundary():
    """The caller's history against the call's first block: sources ending on the last history byte and one byte
    past it, sources spanning history, earlier blocks and the block's own literals, offset 65 535 once P passes
    the 65 535 clamp."""
    rng = np.random.default_rng(101)
    streams = []
    for P in (1, 4096, 65534, 65535, 65536):
        for B in (K4, K64):
            s = Stream(rng, P)
            # block 0 (short, so that block 1 reaches the history): a match on the last history byte and one
            # spanning history and its own literals
            span0 = min(P, 8)
            _filler(s, 1000, [("L", 20), ("M", -1, 4), ("M", -span0, span0 + 12)])
            h = s.rel(0)                                                 # the history boundary, from block 1
            # block 1: bytes 0 .. 39 deferred (from block 0)
            b1 = [("M", h + 100, 40), ("L", 8),
                  ("M", h - 4, 4) if P >= 4 else ("M", h - 1, 4),       # ends on the last history byte: final
                  ("M", h - 3, 4) if P >= 3 else ("M", h - 1, 5),       # one byte past it: deferred
                  ("M", h - min(P, 10), min(P, 10) - h + 60),           # history + block 0 + own bytes
                  ("M", h - min(P, 10), min(P, 10) - h + 30)]
            if P >= 65534:
                b1.append(("O", 65535, 6))                               # P = prefixLen + 1000 > 65 535
            _filler(s, B, b1)
            # block 2: sources across both earlier blocks, and offset 65 535 from deep inside the window
            b2 = [("M", s.rel(0, 50) if B == K4 else s.rel(1, 10), 50), ("L", 4), ("M", s.rel(1, 60), 16)]
            if B == K4:
                b2.append(("M", s.rel(0) - min(P, 5), min(P, 5) - s.rel(0) + 40))
            if P + 1000 + B > 65535:
                b2.append(("O", 65535, 8))
            _filler(s, B if B == K64 else 2 * B, b2)
            streams.append(s.out())

    def target(st):
        return {"earlier-block decisions": st.dec_earlier >= 20, "phase A": st.phase_a >= 10,
                "phase B": st.runs >= 10, "nothing whole": st.whole_blocks == 0}
    return Family("history", streams, target)


def depth():
    """4 KiB blocks whose matches read 1 .. 16 blocks back, onto bytes the replay writes; zero-size entries, empty
    stored entries and stored entries that later blocks copy in between."""
    rng = np.random.default_rng(102)
    streams, reached = [], set()
    for variant in range(3):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64)])
        for j in range(1, 21):
            if variant == 1 and j % 5 == 2:
                s.zero_size()
            if variant == 1 and j % 7 == 3:
                s.stored(b"")
            if variant == 2 and j % 4 == 1:
                s.stored(lits(rng, 1000 + 37 * j))
                continue
            items = [("M", -48, 32), ("L", 8)]      # bytes 0..31: deferred (the block before)
            blocks = [k for k in range(len(s.entries)) if not s.entries[k][2] and s.entries[k][1] > 0]
            for d in range(1, 17):
                if d > len(blocks):
                    break
                k = blocks[-d]
                src = s.rel(k, 4)                   # onto the deferred head of entry k
                op = sum(it[1] if it[0] == "L" else it[-1] for it in items)
                if op - src > 65535:
                    src = s.rel(k, K4 - 40)         # the tail of a 16-back block (literals up to the end)
                if op - src > 65535:
                    continue
                items.append(("M", src, 12))
                reached.add(d)
            stored = [k for k in range(len(s.entries)) if s.entries[k][2] and len(s.entries[k][0]) > 100]
            if stored:
                op = sum(it[1] if it[0] == "L" else it[-1] for it in items)
                src = s.rel(stored[-1], 50)
                if op - src <= 65535:
                    items.append(("M", src, 40))
            items.append(("M", -8, 24))             # straddles into the block's own deferred head: phase B
            _filler(s, K4, items)
        streams.append(s.out())

    def target(st):
        return {"reads 1 .. 16 blocks back": reached == set(range(1, 17)), "earlier-block decisions": st.dec_earlier >= 300,
                "phase B": st.runs >= 40}
    return Family("depth", streams, target)


def own_intervals():
    """Sources inside the block that overlap only an older deferred interval (the binary search), a gap between two
    intervals, an interval's first or last byte exactly and one byte off, and adjacent intervals."""
    rng = np.random.default_rng(103)
    streams = []
    for rep in range(4):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64)])
        # deferred intervals D1 [0, 20), D2 [30, 50), D3 [60, 80), D4 [80, 100): gaps [20, 30), [50, 60)
        items = [("M", -100, 20), ("L", 10), ("M", -200, 20), ("L", 10), ("M", -300, 20), ("M", -400, 20),
                 ("L", 30)]

        def probe(src, ml):
            items.append(("M", -500 - 8 * len(items), 8))     # a fresh interval: the last one is above the probe
            items.append(("M", src, ml))
        probe(5, 8)          # only D1: the search
        probe(20, 10)        # the gap [20, 30): written in pass 2
        probe(30, 4)         # D2's first byte
        probe(26, 4)         # ends one byte before D2: gap
        probe(27, 4)         # enters D2 by one byte
        probe(49, 4)         # D2's last byte
        probe(50, 4)         # one byte behind D2: gap
        probe(78, 4)         # across D3 | D4
        probe(100, 20)       # literals only
        probe(0, 4)          # D1's first byte, the lowest record
        last = sum(it[1] if it[0] == "L" else it[-1] for it in items)
        items.append(("M", last - 8, 4))                        # only the last interval
        items += [("L", 3), ("M", last - 6, 8)]
        _filler(s, K4, items)
        _filler(s, K4, [("M", -K4 + 2, 60), ("L", 5), ("M", -K4 + 25, 30)])
        streams.append(s.out())

    def target(st):
        return {"binary search found a record": st.dec_search >= 4 * 5,
                "binary search found a gap": st.dec_gap >= 4 * 3,
                "last interval": st.dec_last >= 4, "earlier block": st.dec_earlier >= 4 * 10}
    return Family("own-intervals", streams, target)


def phase_a():
    """More than 32 phase-A records per block, lengths 63 / 64 / 65 / 300 with several long ones in one group, and
    a source ending exactly at the block's start (phase A) beside one ending a byte into it (phase B) while byte 0
    is itself deferred."""
    rng = np.random.default_rng(104)
    streams = []
    for rep in range(3):
        s = Stream(rng, 0)
        _filler(s, K64 // 4, [("L", 64)])
        lens = [4, 63, 64, 65, 300, 7, 65, 300, 12]
        items = [("M", -50, 10)]                                # byte 0 .. 9: deferred, phase A
        items += [("M", -10, 10), ("M", -9, 10)]                # hi == 0 (phase A) and hi == 1 (phase B)
        for k in range(90):
            items.append(("M", -int(rng.integers(400, 16000)), lens[(k + rep) % len(lens)]))
            if k % 11 == 5:
                items.append(("L", 1))
        _filler(s, 12000, items)
        streams.append(s.out())

    def target(st):
        return {"phase-A records": st.phase_a >= 3 * 90, "long phase-A records": st.phase_a_long >= 3 * 30,
                "a phase-B record at hi == 1": st.runs >= 3}
    return Family("phase-a", streams, target)


def phase_b_runs():
    """Phase-B windows aligned by independent records, then dependencies at lane pairs (0,1), (0,31), (30,31),
    (31,32) across a window boundary, lane 20 reading lane 3, sources ending one byte before / entering an earlier
    record's destination by one byte, long records at window positions 0 and 31."""
    rng = np.random.default_rng(105)
    streams = []
    for rep in range(3):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64)])
        items = [("L", 16)]                      # final bytes for the independent records to straddle onto
        ops = []                                 # destination of each record, in record order

        def rec(src, ml=8):
            op = sum(it[1] if it[0] == "L" else it[-1] for it in items)
            items.append(("M", src, ml))
            ops.append(op)

        def ind(n=1):                            # independent: [-4, 4), the block before and own literals
            for _ in range(n):
                rec(-4)

        def dep(k):                              # reads record k's destination
            rec(ops[k])
        # window at record 0: (0, 1)
        ind(); dep(0)
        # window at 2: (0, 31)
        ind(31); dep(2)
        # window at 34: (30, 31)
        ind(31); dep(34 + 30)
        # window at 66: no stop; window at 98 starts with a record reading lane 31 of the one before: (31, 32)
        ind(32); dep(97)
        # the same window: lane 20 reads lane 3
        ind(19); dep(98 + 3)
        # window at 119: a long record at lane 0
        rec(-4, 100)
        # window at 120: 31 independent, a long record at lane 31
        ind(31); rec(-4, 100)
        # window at 152: one byte before lane 0's destination (independent), then one byte into it
        ind()
        rec(ops[152] - 8)
        rec(ops[152] - 7)
        if rep:
            ind(int(rng.integers(0, 40)))
        _filler(s, 2000, items)
        _filler(s, K4, [("M", -2000 + 17, 600), ("L", 3), ("M", -100, 90)])
        streams.append(s.out())

    def target(st):
        return {"pair (0,1)": st.dep_pairs[(0, 1)] >= 3, "pair (0,31)": st.dep_pairs[(0, 31)] >= 3,
                "pair (30,31)": st.dep_pairs[(30, 31)] >= 3, "pair (3,20)": st.dep_pairs[(3, 20)] >= 3,
                "pair (0,2)": st.dep_pairs[(0, 2)] >= 3, "across a window": st.cross_window >= 3,
                "stop at lane 0": st.stop_lanes[0] >= 3, "stop at lane 30 or 31": st.stop_lanes[31] >= 9,
                "length stops": st.stops_len >= 6, "dependency stops": st.stops_dep >= 15}
    return Family("phase-b-runs", streams, target)


def periodic():
    """Overlapping (periodic) copies, offset < length: offsets 1, 2, 3, 31, 32, 33, 511, 512, 513, lengths 64, 65,
    511, 512, 513 and 5 000, the source in the block before (phase A) or straddling into the block (phase B)."""
    rng = np.random.default_rng(106)
    streams = []
    for off in (1, 2, 3, 31, 32, 33, 511, 512, 513):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64)])
        for ml in (64, 65, 511, 512, 513, 5000):
            if off >= ml:
                continue
            s.block([("M", -off, ml)])                           # op 0: the period lies in the block before
            if off >= 2:
                h = off // 2
                s.block([("L", h), ("M", h - off, ml)])          # straddles: phase B
        streams.append(s.out())

    def target(st):
        return {"phase-A periodic": st.phase_a_long >= 36, "phase-B periodic": st.stops_len >= 31}
    return Family("periodic", streams, target)


def zero_offset():
    """Offset-0 matches (accepted; the kernel writes zeros at once) between deferred records and in a block with
    nothing deferred, and later records that read them."""
    rng = np.random.default_rng(107)
    streams = []
    for rep in range(3):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64), ("Z", 20), ("L", 12), ("M", 70, 10)])
        _filler(s, K4, [("M", -100, 30), ("Z", 16), ("M", -200, 20), ("L", 4), ("M", 30, 12), ("M", 20, 40),
                        ("Z", 5 + rep)])
        _filler(s, K4, [("M", -K4 + 64, 20), ("M", -K4 + 30, 20), ("L", 12)])
        streams.append(s.out())

    def target(st):
        return {"phase A": st.phase_a >= 6, "phase B": st.runs >= 3}
    return Family("zero-offset", streams, target, zero_offset=True)


def _budget_block(s: Stream, n: int, pre: int = 0, cap_delta: int = 0, ml: int = 4):
    """A block of `n` deferred 4-byte matches into the block before (after `pre` literal bytes); cap_delta < 0
    makes it fail at its end."""
    prev = s.at - s.starts[-1]
    items = [("L", pre)] if pre else []
    for k in range(n):
        items.append(("M", -ml - (k * 7919) % (prev - ml), ml))
    size_of = pre + n * ml + 16
    return s.block(items, cap=size_of + cap_delta)


def budget():
    """Blocks of exactly 2 047, 2 048 and 2 049 deferred records (only 2 049 is whole); whole blocks first, in the
    middle and followed by blocks whose phase-A and phase-B records read them; a whole block that fails and one that
    fills its capacity exactly; many whole blocks across many streams in one call."""
    rng = np.random.default_rng(108)
    streams = []
    for n in (2047, 2048, 2049):
        s = Stream(rng, 0)
        _filler(s, K4, [("L", 64)])
        _budget_block(s, n)
        streams.append(s.out())
    # whole first (behind a stored entry), whole in the middle, then blocks that read it
    s = Stream(rng, 0)
    s.stored(lits(rng, K4))
    _budget_block(s, 2049)
    _filler(s, K4, [("M", -5000, 40), ("L", 8), ("M", -300, 200), ("M", -10, 30), ("M", -6, 20)])
    _budget_block(s, 2100, pre=100)                             # pass 2 wrote its first 100 bytes
    _filler(s, K4, [("M", -8000, 64), ("M", -8, 24), ("L", 2), ("M", -4, 100)])
    _filler(s, K4, [("M", -K4 - 9000, 50), ("M", -K4 - 3, 9)])
    streams.append(s.out())
    # a whole block that fails: the stream is -1 from there on
    s = Stream(rng, 0)
    _filler(s, K4, [("L", 64)])
    _filler(s, K4, [("M", -100, 60)])
    _budget_block(s, 2049, pre=7, cap_delta=-1)
    _filler(s, K4, [("M", -100, 60)])
    _filler(s, K4, [("L", 64)])
    streams.append(s.out())
    # many streams, each with two whole blocks
    for t in range(40):
        s = Stream(rng, int(rng.integers(0, 3000)))
        _filler(s, K4, [("L", 64)])
        _budget_block(s, 2049 + t, pre=t % 3)
        _budget_block(s, 2049)
        _filler(s, K4, [("M", -300, 80), ("L", 4), ("M", -5, 9)])
        streams.append(s.out())

    def target(st):
        return {"2047 and 2048 fit": {2047, 2048} <= set(st.per_block), "2049 is whole": st.whole_blocks >= 1 + 2 + 80,
                "a whole block fails": st.whole_failed >= 1, "whole after pass-2 writes": st.whole_prewritten >= 28,
                "phase A reads a whole block": st.phase_a >= 100}
    return Family("budget", streams, target)


@functools.lru_cache(maxsize=None)
def _datagen_chain(block: int, nblocks: int, seed: int):
    import oracle
    data = oracle.Port().datagen(block * nblocks, 0.63, 0.0, seed).tobytes()
    return data, CR.Upstream().encode_chain(data, block)


def mutants():
    """Valid content mutants (offset, match length and literal rewrites) of a middle block of datagen streams, so
    that the blocks behind it decode against changed history."""
    rng = np.random.default_rng(109)
    streams = []
    for seed in (1, 2):
        data, blocks = _datagen_chain(K4, 12, 200 + seed)
        k = 6
        pa = BM.parsed(blocks[k])
        op = pa.op()
        for i in (1, pa.N // 2, pa.N - 2):
            op_lit = int(op[i] + pa.lit[i])
            for v in (max(1, int(pa.off[i]) - 1), min(65535, op_lit + k * K4), 8, op_lit + 1):
                if not 1 <= v <= min(65535, op_lit + k * K4):
                    continue
                m, size = BM.set_offset(blocks[k], i, v)
                es = [(b, K4, False) for b in blocks]
                es[k] = (m, size, False)
                streams.append((b"", es))
            for ml in (int(pa.ml[i]) + 1, max(4, int(pa.ml[i]) - 1)):
                try:
                    m, size = BM.set_match_len(blocks[k], i, ml)
                except ValueError:
                    continue
                es = [(b, K4, False) for b in blocks]
                es[k] = (m, size, False)
                streams.append((b"", es))
            if pa.lit[i]:
                m, size = BM.set_literals(blocks[k], i, lits(rng, int(pa.lit[i])))
                es = [(b, K4, False) for b in blocks]
                es[k] = (m, size, False)
                streams.append((b"", es))

    def target(st):
        return {"streams decoded": st.blocks >= 12 * 20, "phase B": st.runs >= 100}
    return Family("mutants", streams, target)


FAMILIES = (history_boundary, depth, own_intervals, phase_a, phase_b_runs, periodic, zero_offset, budget, mutants)


@functools.lru_cache(maxsize=None)
def families() -> dict:
    return {f.name: f for f in (g() for g in FAMILIES)}
