"""Hand-assembled LZ4 blocks and a model of the tile decoder's routing (test infrastructure).

* ``build_block(seqs, last)`` writes a raw LZ4 block from a list of sequences
  ``(literals, offset, match_len)`` plus a terminal literal run, with correct length-extension chains,
  and returns it together with the bytes it decodes to.  It does not check the end-of-block rules of the
  format; whether a block is acceptable is the oracle's verdict.
* ``tile_route(stream, cap, src_phase)`` / ``expected_engine(...)`` restate which engine of
  ``csrc/decode_tile.cuh`` decodes a block: ``"trivial"`` (empty input or no room, no kernel work),
  ``"tile"`` (small-stage tile kernel), ``"tile_big"`` (big-stage tile kernel) or ``"generic"`` (the exact
  warp-per-block decoder).  Each test cites the kernel line it restates.
* The helpers below them generate the block families the GPU edge tests run (dense blocks, near-match
  chains, copy-form grids, literal runs across parse segments, stage thresholds) and the adversarial
  encoder inputs (probe-step boundaries, hash / tag collisions).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

MINMATCH, MFLIMIT, LASTLITERALS = 4, 12, 5
TILE_BYTES, TILE_PAD = 65536, 32            # decode_tile.cuh:50-51
STAGE_SMALL = 40 * 1024                     # :72
DT_NMAX, DT_MAX_SRC, DT_K = 16384, 65535, 512   # :74-75, :57
SEG_SMALL, SEG_BIG = 80, 128                # parse segment per lane, :97-100
ENC_HASH_MUL = 2654435761


# ---- builder ---------------------------------------------------------------------------------------

def _ext(v: int) -> bytes:
    """length-extension chain for a nibble of 15 and `v` more (v >= 0)"""
    return b"\xFF" * (v // 255) + bytes([v % 255])


def _append_match(dec: bytearray, off: int, ml: int) -> None:
    if off >= ml:
        s = len(dec) - off
        dec += dec[s:s + ml]
    else:                                   # overlapping copy: periodic with period `off`
        pat = bytes(dec[len(dec) - off:])
        dec += (pat * (ml // off + 1))[:ml]


def build_block(seqs, last: bytes = b"") -> tuple[bytes, bytes]:
    """seqs: iterable of (literals: bytes, offset: 1..65535, match_len >= 4); `last`: terminal literals.
    -> (stream, decoded bytes)."""
    out, dec = bytearray(), bytearray()
    for lits, off, ml in seqs:
        L, M = len(lits), ml - MINMATCH
        if M < 0 or not 1 <= off <= 65535:
            raise ValueError((off, ml))
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out += _ext(L - 15)
        out += lits
        dec += lits
        if off > len(dec):
            raise ValueError(f"offset {off} reaches before the block start at {len(dec)}")
        out += bytes([off & 0xFF, off >> 8])
        if M >= 15:
            out += _ext(M - 15)
        _append_match(dec, off, ml)
    L = len(last)
    out.append(min(L, 15) << 4)
    if L >= 15:
        out += _ext(L - 15)
    out += last
    dec += last
    return bytes(out), bytes(dec)


# ---- the routing model ---------------------------------------------------------------------------------

SQ_LAST, SQ_BAD, SQ_EDGE = 1, 2, 4


@dataclass
class Seq:
    tp: int         # token position
    lit: int
    lit_pos: int
    off: int
    ml: int         # includes MINMATCH, 0 for the terminal sequence
    next: int
    flags: int


def seq_header(s: bytes, p: int) -> Seq:
    """seq_header<EXACT=true> (decode_tile.cuh:186-222) on a stream with nothing behind its end: a length
    chain that runs past the end makes the sequence terminal and bad there too (litEnd > n / q2 >= n), so the
    bytes the kernel reads behind the stream cannot change the verdict."""
    n = len(s)
    tok = s[p]
    q, lit, flags = p + 1, tok >> 4, 0
    if lit == 15:
        while True:
            if q >= n:
                return Seq(p, lit, q, 0, 0, n, SQ_LAST | SQ_BAD)
            b = s[q]; q += 1; lit += b
            if b != 255:
                break
        if q - 1 >= n - 15:                                  # :203
            flags |= SQ_EDGE
    lit_end = q + lit
    if lit_end + 2 > n:                                      # :206, :221
        return Seq(p, lit, q, 0, 0, n, flags | SQ_LAST | (SQ_BAD if lit_end != n else 0))
    off = s[lit_end] | (s[lit_end + 1] << 8)
    q2, m = lit_end + 2, tok & 15
    if m == 15:
        while True:
            if q2 >= n:
                return Seq(p, lit, q, off, 0, n, flags | SQ_BAD)
            b = s[q2]; q2 += 1; m += b
            if b != 255:
                break
        if q2 >= n - 4:                                      # :217
            flags |= SQ_EDGE
    return Seq(p, lit, q, off, m + MINMATCH, min(q2, n), flags | (SQ_BAD if q2 >= n else 0))


def parse(stream: bytes) -> list[Seq]:
    """The token chain from position 0 (what the segmented parse converges to, :408-448)."""
    out, p = [], 0
    while p < len(stream):
        sq = seq_header(stream, p)
        out.append(sq)
        p = sq.next
    return out


@dataclass
class Route:
    engine: str
    n_seq: int = 0
    out: int = 0
    stage: str = ""             # "small" / "big"
    table_intact: bool = False  # pass 2 walks the jump table (:477) rather than seq_next
    why: str = ""


def tile_route(stream: bytes, cap: int, src_phase: int = 0) -> Route:
    n = len(stream)
    if n <= 0 or cap <= 0:                                   # :707, decode_trivial :691-695
        return Route("trivial", why="n <= 0 or cap <= 0")
    if n > DT_MAX_SRC:                                       # :710
        return Route("generic", why="n > 65535")
    stage = "small" if src_phase + n + 16 <= STAGE_SMALL else "big"   # :711
    seqs = parse(stream)
    N = len(seqs)
    O = sum(s.lit + s.ml for s in seqs)
    r = Route("generic", N, O, stage, src_phase + n + 4 + 4 * N <= TILE_BYTES + TILE_PAD)
    if any(s.flags & SQ_BAD for s in seqs):                  # anyBad, :460,471
        r.why = "malformed"
        return r
    if N > DT_NMAX or O <= 0 or O > TILE_BYTES or O > cap:   # :471
        r.why = "N/O/cap"
        return r
    op = 0
    for i, s in enumerate(seqs):                             # per-sequence accept tests, :524-532
        bad = bool(s.flags & (SQ_EDGE | SQ_BAD))
        if i == N - 1:
            bad |= not (s.flags & SQ_LAST) or op + s.lit > cap                      # :527
        else:
            bad |= bool(s.flags & SQ_LAST) or s.lit_pos + s.lit > n - 8 or op + s.lit > cap - MFLIMIT   # :529
            bad |= s.off == 0 or s.off > op + s.lit or op + s.lit + s.ml > cap - LASTLITERALS      # :530
        if bad:
            r.why = f"sequence {i}"
            return r
        op += s.lit + s.ml
    r.engine = "tile" if stage == "small" else "tile_big"
    return r


def expected_engine(stream: bytes, cap: int, src_phase: int = 0) -> str:
    return tile_route(stream, cap, src_phase).engine


def near_flags(stream: bytes) -> list[bool]:
    """Per sequence: is its match `near` in the step scheduler (:536-541), i.e. does the source it reads from
    outside the match itself end behind the output position where its step of 512 sequences begins?"""
    seqs = parse(stream)
    out, op, Sr = [], 0, 0
    for i, s in enumerate(seqs):
        if i % DT_K == 0:
            Sr = op
        d = op + s.lit
        a = d - s.off
        src_end = min(a + s.ml, d)
        out.append(s.ml > 0 and src_end > Sr)
        op = d + s.ml
    return out


# ---- block families ---------------------------------------------------------------------------------------

def _rb(rng, k: int) -> bytes:
    return rng.integers(0, 256, k, dtype=np.uint8).tobytes()


def dense_block(n_seq: int, rng, term: int = 8, first_lit: int = 1):
    """n_seq sequences (terminal included) of 3 stream bytes each where possible: no literals, 4-byte matches
    at random distances.  Decoded size 4 * (n_seq - 1) + first_lit + term."""
    seqs, op = [(_rb(rng, first_lit), 1, 4)], first_lit + 4
    offs = rng.integers(1, 1 << 16, n_seq)
    for i in range(n_seq - 2):
        seqs.append((b"", int(min(offs[i], op, 65535)), 4))
        op += 4
    return build_block(seqs, _rb(rng, term))


def densest_tile_n(cap_slack: bool = True) -> int:
    """The largest sequence count a clean tile block can have.  Every non-terminal sequence decodes to >= 4
    bytes, the first needs >= 1 literal (offset <= op + lit, :530), and the terminal run is >= 5 bytes: the
    last match ends <= n - 8 in the stream (:529) -- or, with a match-length byte, <= n - 5 (:217), which
    costs 15 match bytes to save one literal.  So O >= 4 N + 2 <= 65 536 gives N <= 16 383 (< DT_NMAX).
    With cap == O the last match must also start <= cap - 12 (:529): the terminal run is >= 8, N <= 16 382."""
    return 16383 if cap_slack else 16382


def chain_block(rng, n_seq: int, skip: int = 0, lit0: int = 64):
    """Each sequence copies from the match of the one before it (a dependency chain through the whole step);
    the first `skip` sequences after the opening literal run are independent far copies, so the chain
    starts at lane `skip` of its step."""
    seqs = [(_rb(rng, lit0), 1 + int(rng.integers(0, lit0)), 4 + int(rng.integers(0, 8)))]
    op = lit0 + seqs[0][2]
    prev_d, prev_ml = lit0, seqs[0][2]
    for i in range(1, n_seq - 1):
        if i <= skip:
            lit, ml = 0, 4 + int(rng.integers(0, 8))
            off = op                                             # reads output byte 0..: long before the step
            seqs.append((b"", off, ml))
            prev_d, prev_ml = op, ml
            op += ml
            continue
        lit = int(rng.integers(0, 3))
        ml = 4 + int(rng.integers(0, 36))
        d = op + lit
        a = prev_d + int(rng.integers(0, prev_ml))               # inside the previous match
        seqs.append((_rb(rng, lit), d - a, ml))
        prev_d, prev_ml = d, ml
        op = d + ml
    return build_block(seqs, _rb(rng, 8))


def wide_source_block(rng, k_near: int = 30, steps: int = 3):
    """Per step: k_near short near matches, then one long match whose source spans all of them."""
    seqs = [(_rb(rng, 300), 7, 20)]
    op = 320
    while len(seqs) < steps * DT_K:
        start = op
        for _ in range(k_near):
            lit = int(rng.integers(1, 3))
            seqs.append((_rb(rng, lit), int(rng.integers(1, 4)), 4 + int(rng.integers(0, 4))))
            op += lit + seqs[-1][2]
        ml = 600
        seqs.append((b"", op - start, ml))
        op += ml
        for _ in range(int(rng.integers(0, 40))):              # filler: far copies
            seqs.append((_rb(rng, 1), op - 10, 4))
            op += 5
    return build_block(seqs, _rb(rng, 9))


def step_boundary_block(rng, delta: int, steps: int = 6):
    """The first sequences of every step read sources that end at Sr + delta (delta in -1, 0, +1): exactly at
    the far/near boundary of the scheduler (:540).  The first sequence of a step has no literals."""
    seqs = [(_rb(rng, 2000), 1000, 8)]
    op, i = 2008, 1
    for r in range(steps):
        while i % DT_K:                                          # filler up to the step start
            lit = int(rng.integers(0, 3))
            seqs.append((_rb(rng, lit), int(rng.integers(8, 1500)), 4 + int(rng.integers(0, 6))))
            op += lit + seqs[-1][2]; i += 1
        Sr = op
        for j in range(4):
            lit = 0 if j == 0 else int(rng.integers(0, 3))
            ml = 8 + 4 * j
            d = op + lit
            target = Sr + (delta if j else min(delta, 0))        # srcEnd can never pass d
            off = d - (target - ml)                              # a + ml == target, off >= ml
            seqs.append((_rb(rng, lit), off, ml))
            op = d + ml; i += 1
    return build_block(seqs, _rb(rng, 8))


COPY_LENS = list(range(4, 34)) + [127, 128, 129, 159, 160, 161, 600]


def copy_grid_blocks(rng, offsets=range(1, 201), lens=COPY_LENS, max_out: int = 60000):
    """Overlapping and plain matches for every (offset, length) pair, literal runs cycling through 0..40
    (and 31..34 around the lane/warp copy threshold).  Apart from the first sequence of a step (which has
    no literals here), matches with offset < length are near."""
    lit_cycle = list(range(0, 41)) + [31, 32, 33, 34]
    blocks, seqs, op, k = [], [], 0, 0
    pairs = [(o, m) for o in offsets for m in lens]
    first = _rb(rng, 256)
    for off, ml in pairs:
        if not seqs:
            seqs, op = [(first, 1, 4)], 260
        lit = 0 if len(seqs) % DT_K == 0 else lit_cycle[k % len(lit_cycle)]
        k += 1
        seqs.append((_rb(rng, lit), off, ml))
        op += lit + ml
        if op > max_out:
            blocks.append(build_block(seqs, _rb(rng, 8)))
            seqs = []
    if seqs:
        blocks.append(build_block(seqs, _rb(rng, 8)))
    return blocks


def far_overlap_blocks(rng, offsets, lens):
    """Overlapping matches as FAR copies: only the first sequence of a step, with no literals, reads a
    source that ends at the step start; everything else in the block is filler."""
    blocks, seqs, op = [], [], 0
    for off, ml in [(o, m) for o in offsets for m in lens if o < m]:
        if not seqs:
            seqs, op = [(_rb(rng, 256), 1, 4)], 260
        while len(seqs) % DT_K:
            seqs.append((b"", int(rng.integers(5, 200)), 4))
            op += 4
        seqs.append((b"", off, ml))
        op += ml
        if op > 60000 - 4 * DT_K:
            blocks.append(build_block(seqs, _rb(rng, 8)))
            seqs = []
    if seqs:
        blocks.append(build_block(seqs, _rb(rng, 8)))
    return blocks


def literal_run_block(rng, run: int, fill: int | None, n_runs: int = 3):
    """Literal runs of `run` bytes (random, or every byte = `fill`) between short matches: the speculative
    parse walks into them from arbitrary bytes."""
    lits = (lambda: bytes([fill]) * run) if fill is not None else (lambda: _rb(rng, run))
    seqs = [(_rb(rng, 16), 3, 5)]
    for _ in range(n_runs):
        seqs.append((lits(), int(rng.integers(1, 16)), 4 + int(rng.integers(0, 30))))
    return build_block(seqs, _rb(rng, 8))


def sized_block(rng, n: int, fill: int | None = None):
    """A clean literal-heavy block whose compressed size is exactly n (>= 20): one long literal run, a
    4-byte match, a terminal run of 8..10 literals (the last match
    starts >= 12 bytes before the end, so cap == decoded size is accepted)."""
    for term in (8, 9, 10):
        for L in range(n - 4 - term, max(n - 400, 7), -1):
            ext = 0 if L < 15 else (L - 15) // 255 + 1
            if 1 + ext + L + 2 + 1 + term == n:
                lits = bytes([fill]) * L if fill is not None else _rb(rng, L)
                s, d = build_block([(lits, 1 + int(rng.integers(0, 8)), 4)], _rb(rng, term))
                assert len(s) == n
                return s, d
    raise ValueError(n)


# ---- encoder inputs ------------------------------------------------------------------------------------------

def probe_advance(q: int) -> int:
    """Distance of search probe q from probe 0 of its run (encode_tile.cuh:47-52, LL64.fast.cs:159-170)."""
    if q <= 64:
        return q
    c = 63 + q
    k = c >> 6
    return 1 + 32 * k * (k - 1) + (c - 64 * k) * k


PROBE_TARGETS = [63, 64, 65, 127, 128, 129, 191, 192, 193, 40, 41]


def probe_step_input(rng, n: int = 65536, tail: int = 13, collide: bool = False) -> bytes:
    """Random bytes with copies of recently probed windows planted so that the first hit of each search run
    lands at probe index 64k - 1, 64k, 64k + 1 (where probe_advance changes its step), and a last match at
    n - `tail`.  With `collide`, the first probes of every run also see 4-byte words that share the hash -- and
    partly the 16-bit tag of the global-table encoder -- with a word probed a few positions earlier, while the
    bytes differ: v' = v + k * inv(2654435761) gives the product prod + k."""
    buf = bytearray(_rb(rng, n))
    inv = pow(ENC_HASH_MUL, -1, 1 << 32)
    base, t = 1, 0
    while True:
        q = PROBE_TARGETS[t % len(PROBE_TARGETS)]
        t += 1
        P = base + probe_advance(q)
        L = 4 + int(rng.integers(0, 20))
        if P + L + 300 > n - tail:
            break
        if collide:
            for j in range(0, 24, 8):
                x = base + j
                v = int.from_bytes(buf[x:x + 4], "little")
                prod = (v * ENC_HASH_MUL) & 0xFFFFFFFF
                k = int(rng.integers(1, 8)) if (prod & 7) == 7 else int(rng.integers(1, 8 - (prod & 7)))
                if j == 16:
                    k *= 8                                       # same hash, different tag
                v2 = (v + k * inv) & 0xFFFFFFFF
                buf[x + 4:x + 8] = v2.to_bytes(4, "little")
        src = base + probe_advance(q - 8 - int(rng.integers(0, 8)))   # a position probed shortly before P
        for i in range(L):
            buf[P + i] = buf[src + i]
        base = P + L + 1
    # close the run with a match that ends so that the last run starts 20 bytes before n - tail, then the last
    # match: a copy of the window of that run's probe 10, found by its probe 20 at n - tail
    end = n - tail - 20
    q2 = 0
    while base + probe_advance(q2 + 1) <= end - 5:
        q2 += 1
    P2 = base + probe_advance(q2)
    src2 = base + probe_advance(q2 - 8)
    for i in range(end - 1 - P2):
        buf[P2 + i] = buf[src2 + i]
    P = n - tail
    for i in range(min(8, tail)):
        buf[P + i] = buf[end + 10 + i]
    return bytes(buf)
