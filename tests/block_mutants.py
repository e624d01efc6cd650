"""Mutants of real full-size LZ4 blocks, for pinning the block decoders against the oracle (test infrastructure).

Every byte a frame decode, a chain decoder group or a frame reader group returns passes through the tile kernel
(csrc/decode_tile.cuh) or the exact warp-per-block engine (csrc/decode_generic.cuh).  Hand-built blocks pin their
mechanisms; this module rewrites fields of real 64 KiB blocks so that the same mechanisms meet real data:

* Layout-preserving rewrites (``set_offset``, ``set_match_len``, ``set_literals``) keep the stream's length and
  every token position.  The block stays a well-formed token chain, so it stays on the tile path and decodes to
  *different* content.  An offset rewritten to exactly the accept boundary ``op + lit (+ P)``, or one past it, pins
  the accept test at any sequence (``offset_targets``).
* Chain-breaking mutations (``chain_breaking``: length nibbles and bytes, whole tokens, truncation, appended bytes,
  ``inputs.mutate``) mostly go to the exact engine; the tile path must hand them over untouched.
* End-rule tails (``end_rule_tails``) put the block's last sequence in a later step, at varied lanes, with its last
  match and last literal run around ``cap - LASTLITERALS`` and ``cap - MFLIMIT``, where the reference's verdict
  depends on the capacity's slack.
* ``parse`` / ``route`` restate ``lz4_blocks.parse`` and ``tile_route`` / ``chain_ref.tile_route_p`` over numpy
  arrays and reuse the base block's parse: one list-form parse of a 64 KiB block costs 10-30 ms, so thousands of
  mutants could not be routed otherwise.  tests/test_block_mutants_model.py holds them against the list forms.

Base blocks are 64 KiB blocks of the library's own encoder (``oracle.Port``) and blocks k >= 1 of upstream's chained
encoder.  Everything comes from fixed seeds; base blocks and their parses are memoised.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

from tests import chain_ref as CR
from tests import inputs
from tests import lz4_blocks as LB

K64 = 65536
MINMATCH, MFLIMIT, LASTLITERALS = LB.MINMATCH, LB.MFLIMIT, LB.LASTLITERALS
DT_K = LB.DT_K
FIXED_SEQS = (0, 1, 31, 32, 511, 512, 513, 1023, 1024)     # plus N/2, N - 3, N - 2
TAIL_SLACK = (0, 1, 4, 5, 6, 11, 12, 13, 32)               # end-rule tails: cap = exact + slack
CAP_SLACK = (0, 1, 5, 13, 32, "64k", -1)                   # mutants: exact + slack, 65 536, exact - 1
HISTORY_P = (0, 1, 7, 4096, 65534, 65535, 65536, 131072)


# ---- parse and routing over arrays ------------------------------------------------------------------------------

class Parsed:
    """lz4_blocks.parse as int64 arrays, one entry per sequence (terminal included)."""
    FIELDS = ("tp", "lit", "lit_pos", "off", "ml", "nxt", "flags")

    def __init__(self, tp, lit, lit_pos, off, ml, nxt, flags):
        self.tp, self.lit, self.lit_pos, self.off = tp, lit, lit_pos, off
        self.ml, self.nxt, self.flags = ml, nxt, flags

    @classmethod
    def from_seqs(cls, seqs) -> "Parsed":
        a = np.array([(s.tp, s.lit, s.lit_pos, s.off, s.ml, s.next, s.flags) for s in seqs],
                     dtype=np.int64).reshape(-1, 7)
        return cls(*(a[:, k].copy() for k in range(7)))

    @property
    def N(self) -> int:
        return len(self.tp)

    @property
    def size(self) -> int:
        return int(self.lit.sum() + self.ml.sum())

    def op(self) -> np.ndarray:
        """output position where each sequence's literals begin"""
        o = np.zeros(self.N, dtype=np.int64)
        np.cumsum((self.lit + self.ml)[:-1], out=o[1:])
        return o

    def with_seq(self, i: int, off: int | None = None, ml: int | None = None) -> "Parsed":
        """The parse after a layout-preserving rewrite of sequence i (unchanged arrays are shared)."""
        o, m = self.off, self.ml
        if off is not None:
            o = o.copy(); o[i] = off
        if ml is not None:
            m = m.copy(); m[i] = ml
        return Parsed(self.tp, self.lit, self.lit_pos, o, m, self.nxt, self.flags)

    def seqs(self) -> list:
        return [LB.Seq(*(int(getattr(self, f)[k]) for f in self.FIELDS)) for k in range(self.N)]


_PARSES: dict[bytes, Parsed] = {}


def parsed(stream: bytes) -> Parsed:
    """The memoised parse of a base block (or of any stream the mutators are given)."""
    p = _PARSES.get(stream)
    if p is None:
        p = _PARSES[stream] = Parsed.from_seqs(LB.parse(stream))
    return p


def parse(stream: bytes, like: tuple[bytes, Parsed] | None = None) -> Parsed:
    """lz4_blocks.parse(stream).  With like = (base stream, its parse), the base's sequences that end at least 16
    bytes before both the first byte that differs and either end are reused: seq_header reads only [tp, next) and
    looks at the end only within 15 bytes of it, so they parse the same; the rest is parsed again."""
    if like is None:
        return Parsed.from_seqs(LB.parse(stream))
    s0, p0 = like
    n, n0 = len(stream), len(s0)
    m = min(n, n0)
    diff = np.flatnonzero(np.frombuffer(stream, np.uint8, m) != np.frombuffer(s0, np.uint8, m))
    d = int(diff[0]) if len(diff) else m
    k = int(np.searchsorted(p0.nxt, min(d, n - 16, n0 - 16), side="right"))
    p, tail = (int(p0.nxt[k - 1]) if k else 0), []
    while p < n:
        sq = LB.seq_header(stream, p)
        tail.append(sq)
        p = sq.next
    t = Parsed.from_seqs(tail)
    return Parsed(*(np.concatenate([getattr(p0, f)[:k], getattr(t, f)]) for f in Parsed.FIELDS))


def route(pa: Parsed, n: int, cap: int, src_phase: int = 0, P: int = 0) -> str:
    """lz4_blocks.tile_route(stream, cap, src_phase).engine for P = 0, chain_ref.tile_route_p(stream, cap, P,
    src_phase) otherwise (decode_tile.cuh:707-711, :460-471, :549-553), on the stream's parse."""
    if n <= 0 or cap <= 0:
        return "trivial"
    if n > LB.DT_MAX_SRC:
        return "generic"
    big = src_phase + n + 16 > LB.STAGE_SMALL
    fl = pa.flags
    if (fl & LB.SQ_BAD).any():
        return "generic"
    N, O = pa.N, pa.size
    if N > LB.DT_NMAX or O <= 0 or O > LB.TILE_BYTES or O > cap:
        return "generic"
    if (fl & LB.SQ_EDGE).any():
        return "generic"
    op, last = pa.op(), N - 1
    if not fl[last] & LB.SQ_LAST or op[last] + pa.lit[last] > cap:
        return "generic"
    h = slice(0, last)
    d = op[h] + pa.lit[h]
    off = pa.off[h]
    bad = ((fl[h] & LB.SQ_LAST) != 0) | (pa.lit_pos[h] + pa.lit[h] > n - 8) | (d > cap - MFLIMIT) | (off == 0) | \
        (off > d + min(P, 65535)) | (d + pa.ml[h] > cap - LASTLITERALS)
    if bad.any():
        return "generic"
    return "tile_big" if big else "tile"


def is_near(pa: Parsed, i: int) -> bool:
    """lz4_blocks.near_flags(stream)[i]: does match i read a source that ends behind its step's first output byte?"""
    op = pa.op()
    Sr = int(op[i // DT_K * DT_K])
    d = int(op[i] + pa.lit[i])
    a = d - int(pa.off[i])
    return int(pa.ml[i]) > 0 and min(a + int(pa.ml[i]), d) > Sr


# ---- layout-preserving rewrites -------------------------------------------------------------------------------------

def set_offset(stream: bytes, i: int, v: int) -> tuple[bytes, int]:
    """Sequence i's offset becomes v (0..65535).  -> (mutant, exact decoded size)."""
    pa = parsed(stream)
    if not (0 <= i < pa.N - 1 and 0 <= v <= 65535):
        raise ValueError((i, v))
    p = int(pa.lit_pos[i] + pa.lit[i])
    m = bytearray(stream)
    m[p:p + 2] = v.to_bytes(2, "little")
    return bytes(m), pa.size


def set_match_len(stream: bytes, i: int, ml: int) -> tuple[bytes, int]:
    """Sequence i's match length (MINMATCH included) becomes ml: through the token's nibble when the old and the new
    value are both below 15 + MINMATCH, else through the last length-extension byte, which stays below 255."""
    pa = parsed(stream)
    if not 0 <= i < pa.N - 1:
        raise ValueError(i)
    old = int(pa.ml[i])
    M0, M = old - MINMATCH, ml - MINMATCH
    m = bytearray(stream)
    tp = int(pa.tp[i])
    if M0 < 15 and 0 <= M < 15:
        m[tp] = (m[tp] & 0xF0) | M
    elif M0 >= 15 and 0 <= m[int(pa.nxt[i]) - 1] + M - M0 < 255:
        m[int(pa.nxt[i]) - 1] += M - M0
    else:
        raise ValueError((i, old, ml))
    return bytes(m), pa.size - old + ml


def set_literals(stream: bytes, i: int, lits: bytes) -> tuple[bytes, int]:
    """Sequence i's literal bytes become `lits` (same length)."""
    pa = parsed(stream)
    L, p = int(pa.lit[i]), int(pa.lit_pos[i])
    if len(lits) != L:
        raise ValueError((i, L, len(lits)))
    m = bytearray(stream)
    m[p:p + L] = lits
    return bytes(m), pa.size


# ---- base blocks ------------------------------------------------------------------------------------------------------

@dataclass(eq=False)
class Base:
    name: str
    stream: bytes
    history: bytes          # the stream's content in front of the block (b"" for an independent block)
    pa: Parsed

    @property
    def size(self) -> int:
        return self.pa.size


@functools.lru_cache(maxsize=None)
def independent_bases() -> tuple[Base, ...]:
    """64 KiB blocks of the library's encoder: datagen 0.55 / 0.63, text2, lowent, runs, lorem; lowent and
    literal-heavy blocks whose compressed size needs the big stage (> 40 KiB)."""
    import oracle
    port = oracle.Port()
    raws = [("datagen0.55", port.datagen(K64, 0.55, 0.0, 55).tobytes()),
            ("datagen0.63", port.datagen(K64, 0.63, 0.0, 63).tobytes())]
    raws += [(k, inputs.gen(k, K64, 5)) for k in ("text2", "lowent", "runs", "lorem")]
    raws += [("lowent-b", inputs.gen("lowent", K64, 6)),
             ("literal-heavy", inputs.gen("random", 40000, 7) + inputs.gen("text2", K64 - 40000, 7)),
             ("literal-heavy-b", inputs.gen("random", 30000, 8) + inputs.gen("lowent", K64 - 30000, 8))]
    out = []
    for name, raw in raws:
        r, c = port.encode(raw)
        assert r > 0
        out.append(Base(name, c, b"", parsed(c)))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def chained_bases() -> tuple[Base, ...]:
    """Blocks 2 and 3 of upstream's chained encoder (LZ4_compress_fast_continue) over datagen 0.63 / 0.55 and over
    blocks of 20 000 random bytes and lowent (compressed > 40 KiB: the big stage); each carries the 128 / 192 KiB of
    content in front of it."""
    import oracle
    up = CR.Upstream()
    port = oracle.Port()
    datas = [("chain-datagen0.63", port.datagen(4 * K64, 0.63, 0.0, 163).tobytes()),
             ("chain-datagen0.55", port.datagen(4 * K64, 0.55, 0.0, 155).tobytes()),
             ("chain-literal-heavy", b"".join(inputs.gen("random", 20000, 20 + k) + inputs.gen("lowent", K64 - 20000, 30 + k)
                                              for k in range(4)))]
    out = []
    for name, data in datas:
        blocks = up.encode_chain(data)
        for k in (2, 3):
            out.append(Base(f"{name}#{k}", blocks[k], data[:k * K64], parsed(blocks[k])))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def clamped(base: Base, P: int) -> Base:
    """`base` with every offset that reaches further back than the P bytes of history rewritten (layout-preserving)
    to a seeded value in range, so that the block is valid behind exactly P bytes: otherwise a block of upstream's
    chained encoder behind a short history fails at its first far match, whatever the mutation."""
    if P >= 65535:
        return base
    pa = base.pa
    d = pa.op()[:-1] + pa.lit[:-1]
    far = np.flatnonzero(pa.off[:-1] > d + P)
    if not len(far):
        return base
    rng = np.random.default_rng(P + 7)
    m = bytearray(base.stream)
    off = pa.off.copy()
    for i in far:
        reach = int(d[i]) + P
        v = int(rng.integers(1, reach + 1)) if reach > 0 else 1     # d = P = 0: no offset is valid, keep it failing
        p = int(pa.lit_pos[i] + pa.lit[i])
        m[p:p + 2] = v.to_bytes(2, "little")
        off[i] = v
    s = bytes(m)
    pc = Parsed(pa.tp, pa.lit, pa.lit_pos, off, pa.ml, pa.nxt, pa.flags)
    _PARSES[s] = pc
    return Base(f"{base.name}@P{P}", s, base.history, pc)


# ---- which sequences, which values ------------------------------------------------------------------------------------

def target_seqs(pa: Parsed, n: int, per_segment: int = 2) -> list[int]:
    """Sequences with a match to rewrite: FIXED_SEQS, N/2, N - 3, N - 2, and sequences whose token sits at a parse
    segment's first or last byte (80 bytes per lane on the small stage, 128 on the big one)."""
    N = pa.N
    idx = {i for i in FIXED_SEQS + (N // 2, N - 3, N - 2) if 0 <= i <= N - 2}
    seg = LB.SEG_SMALL if n + 16 <= LB.STAGE_SMALL else LB.SEG_BIG
    for r in (0, seg - 1):
        hits = np.flatnonzero(pa.tp[:-1] % seg == r)
        idx.update(int(x) for x in hits[::max(len(hits) // per_segment, 1)][:per_segment])
    return sorted(i for i in idx if pa.ml[i] > 0)


def offset_targets(pa: Parsed, i: int, P: int, rng, n_random: int = 4, full: bool = True) -> list[tuple[str, int]]:
    """(tag, offset) rewrites of match i behind P bytes of history: the accept boundary op + lit + P and one past
    it, 0, 1..7 (below the copy shortcut's offset >= 8), 8, 15, 16, ml - 1 .. ml + 1 (the overlap threshold), a value
    that turns a far match near or a near one far, and random values in range -- with a history, half of them
    reaching into it."""
    op = pa.op()
    d, ml = int(op[i] + pa.lit[i]), int(pa.ml[i])
    reach = min(d + min(P, 65535), 65535)
    out = []
    if 1 <= d + P <= 65535:
        out.append(("boundary", d + P))
    if d + P + 1 <= 65535:
        out.append(("boundary+1", d + P + 1))
    out.append(("zero", 0))
    small = range(1, 8) if full else (1, 3, 7)
    out += [("below8", v) for v in small]
    out += [("8/15/16", v) for v in ((8, 15, 16) if full else (8,))]
    out += [("overlap", v) for v in (ml - 1, ml, ml + 1) if v >= 1]
    Sr = int(op[i // DT_K * DT_K])
    if is_near(pa, i):
        v = d - Sr + ml                                      # source ends exactly at Sr: far
        if v <= reach:
            out.append(("near->far", v))
    elif d > Sr:
        out.append(("far->near", d - Sr + ml - 1))          # source ends at Sr + 1: near
    for k in range(n_random):
        if P > 0 and reach > d and k % 2 == 0:
            out.append(("random-history", int(rng.integers(d + 1, reach + 1))))
        elif reach >= 1:
            out.append(("random", int(rng.integers(1, reach + 1))))
    return [(t, v) for t, v in out if 0 <= v <= 65535]


def ml_targets(pa: Parsed, stream: bytes, i: int) -> list[int]:
    """Match lengths reachable by set_match_len: shorter and longer by one, the shortest, and a longer one."""
    ml = int(pa.ml[i])
    M = ml - MINMATCH
    if M < 15:
        vals = {MINMATCH, ml - 1, ml + 1, MINMATCH + 14}
        return sorted(v for v in vals if MINMATCH <= v < MINMATCH + 15 and v != ml)
    b = stream[int(pa.nxt[i]) - 1]
    return sorted({ml + k for k in (-1, 1, -b, 254 - b) if 0 <= b + k <= 254 and k != 0})


# ---- mutants ----------------------------------------------------------------------------------------------------------

@dataclass
class Mutant:
    base: Base
    stream: bytes
    size: int                   # exact decoded size of the token chain (for chain-breaking mutants: the base's)
    kind: str
    seq: int = -1               # the rewritten sequence, -1 for none
    pa: Parsed | None = None    # None: parsed on demand against the base

    def parse(self) -> Parsed:
        if self.pa is None:
            self.pa = parse(self.stream, (self.base.stream, self.base.pa))
        return self.pa


def layout_mutants(base: Base, rng, P: int = 0, full: bool = True) -> list[Mutant]:
    """Offset, match-length and literal rewrites of the target sequences, and the terminal run's literals."""
    pa, s = base.pa, base.stream
    out = []
    for i in target_seqs(pa, len(s)):
        for tag, v in offset_targets(pa, i, P, rng, full=full):
            m, z = set_offset(s, i, v)
            out.append(Mutant(base, m, z, "offset:" + tag, i, pa.with_seq(i, off=v)))
        for ml in ml_targets(pa, s, i)[:3 if full else 1]:
            m, z = set_match_len(s, i, ml)
            out.append(Mutant(base, m, z, "ml", i, pa.with_seq(i, ml=ml)))
        if pa.lit[i] > 0:
            m, z = set_literals(s, i, LB._rb(rng, int(pa.lit[i])))
            out.append(Mutant(base, m, z, "literals", i, pa))
    last = pa.N - 1
    if pa.lit[last] > 0:
        m, z = set_literals(s, last, LB._rb(rng, int(pa.lit[last])))
        out.append(Mutant(base, m, z, "literals", last, pa))
    return out


def _ext_bytes(pa: Parsed, s: bytes) -> list[int]:
    """positions of length-extension bytes equal to 254 or 255"""
    pos = []
    for i in np.flatnonzero((pa.lit >= 15) | (pa.ml >= 15 + MINMATCH)):
        lo, hi = int(pa.tp[i]) + 1, int(pa.lit_pos[i])
        pos += [p for p in range(lo, hi) if s[p] in (254, 255)]
        if pa.ml[i] >= 15 + MINMATCH:
            lo = int(pa.lit_pos[i] + pa.lit[i]) + 2
            pos += [p for p in range(lo, int(pa.nxt[i])) if s[p] in (254, 255)]
    return pos


def chain_breaking(base: Base, rng, n_mutate: int = 12) -> list[Mutant]:
    """Mutations that move tokens: the literal nibble +-1, a length-extension byte 254 <-> 255, the token set to
    0x00 / 0x0F / 0xF0 / 0xFF, truncation at each of the last 64 positions and at step boundaries, 1..8 bytes
    appended, inputs.mutate."""
    pa, s = base.pa, base.stream
    n, N = len(s), pa.N
    out = []

    def add(m, kind, i=-1):
        out.append(Mutant(base, bytes(m), base.size, kind, i))

    for i in sorted({i for i in (0, 1, 511, 512, 513, N // 2, N - 2, N - 1) if 0 <= i < N}):
        tp = int(pa.tp[i])
        L = s[tp] >> 4
        for dl in (-1, 1):
            if L < 15 and 0 <= L + dl < 15:
                m = bytearray(s); m[tp] += 16 * dl
                add(m, "lit-nibble", i)
        for t in (0x00, 0x0F, 0xF0, 0xFF):
            if s[tp] != t:
                m = bytearray(s); m[tp] = t
                add(m, "token", i)
    ext = _ext_bytes(pa, s)
    for p in ext[::max(len(ext) // 6, 1)][:6]:
        m = bytearray(s); m[p] ^= 1                          # 254 <-> 255
        add(m, "ext-254-255")
    for c in range(n - 64, n):
        add(s[:c], "truncate-end")
    for k in range(DT_K, N, DT_K):
        tp = int(pa.tp[k])
        add(s[:tp], "truncate-step", k)
        add(s[:tp + 1], "truncate-step", k)
    for k in range(1, 9):
        add(s + LB._rb(rng, k), "append")
    for _ in range(n_mutate):
        add(inputs.mutate(s, rng), "mutate")
    return out


# ---- end-rule tails ---------------------------------------------------------------------------------------------------

LAST_LANES = (512, 513, 543, 544, 1023, 1024, 1100, 1535)   # index of the terminal sequence


def end_rule_tails(rng, history: bytes = b"", lanes=LAST_LANES, terms=range(14)) -> list[tuple[bytes, int, str]]:
    """Blocks whose terminal sequence sits at `lanes` (steps 1 and 2, varied lanes) behind short filler sequences,
    with t = 0..13 terminal literals: with caps exact + TAIL_SLACK the last match ends at cap - LASTLITERALS +- 1 and
    the last literal run starts at cap - MFLIMIT +- 1; t = 0 ends on a match with an empty terminal run.  The same
    block without its terminal token ends on a match with no terminal sequence at all.  With a history, half of
    the filler matches reach into it.  -> [(stream, exact decoded size, tag)]."""
    P = len(history)
    out = []
    for j, last in enumerate(lanes):
        seqs, op = [(LB._rb(rng, 48), 7, 8)], 56
        for _ in range(last - 2):
            lit = LB._rb(rng, 1)
            reach = min(op + 1 + P, 65535)
            off = int(rng.integers(op + 2, reach + 1)) if P and reach > op + 1 and rng.random() < 0.5 \
                else int(rng.integers(5, 40))
            ml = int(rng.integers(4, 9))
            seqs.append((lit, off, ml))
            op += 1 + ml
        lm = (LB._rb(rng, j % 3), 3, 40) if j % 2 else (LB._rb(rng, j % 3), 1000 + j, 19)   # periodic near / far
        for t in terms:
            s, dec = CR.build_prefix_block(history, seqs + [lm], LB._rb(rng, t))
            out.append((s, len(dec), f"tail lane{last} t{t}"))
        s, dec = CR.build_prefix_block(history, seqs + [lm], b"")
        out.append((s[:-1], len(dec), f"tail lane{last} no terminal"))
    return out


# ---- the case lists the model and GPU tests share ---------------------------------------------------------------------

def _cap(size: int, slack) -> int:
    return K64 if slack == "64k" else size + slack


def independent_cases(seed: int = 2026) -> list[tuple[Mutant, int, int]]:
    """Every independent-block case: (mutant, cap, source phase).  Each layout-preserving mutant is decoded at two
    caps of CAP_SLACK in turn, each chain-breaking one at one; each end-rule tail at every TAIL_SLACK."""
    rng = np.random.default_rng(seed)
    out, k = [], 0
    for base in independent_bases():
        for m in layout_mutants(base, rng):
            for _ in range(2):
                out.append((m, _cap(m.size, CAP_SLACK[k % len(CAP_SLACK)]), int(rng.integers(0, 16))))
                k += 1
        for m in chain_breaking(base, rng):
            out.append((m, _cap(m.size, CAP_SLACK[k % len(CAP_SLACK)]), int(rng.integers(0, 16))))
            k += 1
    for s, z, tag in end_rule_tails(rng):
        pa = parse(s)
        b = Base(tag, s, b"", pa)
        for sl in TAIL_SLACK:
            out.append((Mutant(b, s, z, "tail", pa.N - 1, pa), z + sl, int(rng.integers(0, 16))))
    return out


def chained_cases(seed: int = 2027) -> list[tuple[Mutant, int, bytes]]:
    """Every chained-block case: (mutant, cap, history).  Upstream's chained blocks behind each history length of
    HISTORY_P (the block's real content in front of it), offset-rewritten; end-rule tails behind 1, 7, 4 096 and
    65 536 bytes of history."""
    rng = np.random.default_rng(seed)
    out, k = [], 0
    for P in HISTORY_P:
        for base in chained_bases():
            b = clamped(base, P)
            h = b.history[len(b.history) - P:]
            pa = b.pa
            for i in target_seqs(pa, len(b.stream), per_segment=1)[::2 if P in (65534, 131072) else 1]:
                for tag, v in offset_targets(pa, i, P, rng, full=False):
                    m, z = set_offset(b.stream, i, v)
                    cap = _cap(z, CAP_SLACK[k % 3])          # exact, + 1, + 5
                    k += 1
                    out.append((Mutant(b, m, z, "offset:" + tag, i, pa.with_seq(i, off=v)), cap, h))
    for P in (1, 7, 4096, 65536):
        hist = rng.integers(0, 256, P, dtype=np.uint8).tobytes()
        for s, z, tag in end_rule_tails(rng, hist, lanes=(513, 1024, 1100), terms=(0, 4, 5, 6, 7, 11, 12, 13)):
            pa = parse(s)
            b = Base(tag, s, hist, pa)
            for sl in (0, 1, 5, 6, 12):
                out.append((Mutant(b, s, z, "tail", pa.N - 1, pa), z + sl, hist))
    return out
