"""Inputs built for the batches of the chained and dictionary encoders' match search (chain_search_warp,
csrc/encode_chain.cuh).  Data only: every case is checked against upstream by tests/test_chain_windows_model.py,
which also counts that the cases reach what they are built for, and run on the GPU by
tests/test_gpu_chain_windows.py.

The search runs 32 consecutive probes at once.  The block's first run has no post-match lane: its probe q sits
at lane q % 32.  Every later run follows the post-match probe, which takes lane 0 of its first batch: its probe q
sits at lane (q + 1) % 32, so its batch edges fall between q = 30/31 and 62/63.

A case is ``Case(name, family, ext, h4, before, src, state, cap)``:
  * prefix mode (ext False): `before` is the history directly in front of the source and `state` the stream's
    K4LZ4_CHAIN_STATE_BYTES record before the block (planted, or what upstream left after encoding `before`);
  * extDict mode (ext True): `before` is a dictionary in a buffer of its own, loaded by LZ4_loadDict (hash5 only;
    `state` is None).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from tests import chain_enc_ref as CE
from tests import dict_enc_ref as DR
from tests.lz4_blocks import probe_advance

K5 = 889523592379                      # prime5bytes: hash5 = bits 28..39 of (low 40 bits of the word) * K5
K5_INV = pow(K5, -1, 1 << 40)
K4 = 2654435761                        # hash4 = bits 20..31 of word * K4
K4_INV = pow(K4, -1, 1 << 32)
M40 = (1 << 40) - 1

TARGETS = (0, 29, 30, 31, 32, 33, 61, 62, 63, 64, 65, 127, 128, 129, 191, 192, 193)
DICT_SIZES = (8, 9, 4096, 4097, 65535, 65536, 200000)


def hash5_12(b8: bytes) -> int:
    """hash5 at 12 bits (the 64-bit engine's byU32 hash, test_gpu_chain_encode._hash5)."""
    v = int.from_bytes(bytes(b8[:8]).ljust(8, b"\0"), "little")
    return (((v << 24) * K5) & ((1 << 64) - 1)) >> 52


def hash4_12(b4: bytes) -> int:
    """hash4 at 12 bits (the 32-bit engine's, enforce32_ref.hash4)."""
    return ((int.from_bytes(bytes(b4[:4]), "little") * K4) & 0xFFFFFFFF) >> 20


def probe_lane(q: int, post: bool) -> int:
    """The lane of search probe q: q % 32 in the block's first run, (q + 1) % 32 in a run behind a match."""
    return (q + (1 if post else 0)) % 32


@dataclass
class Case:
    name: str
    family: str
    ext: bool
    h4: bool
    before: bytes
    src: bytes
    state: np.ndarray | None
    cap: int

    @property
    def n(self) -> int:
        return len(self.src)


def bound(n: int) -> int:
    return n + n // 255 + 16


# ---- collisions -----------------------------------------------------------------------------------------------

def collide(buf: bytearray, x: int, y: int, rng, h4: bool) -> None:
    """Rewrite the word at x so that it has the 12-bit hash of the word at y but other first 4 bytes.  hash5
    rewrites 5 bytes (bits 0..27 of y = x * K5 mod 2^40 change), which changes the words at x - 4 .. x + 4 too;
    hash4 rewrites 4 bytes (bits 0..19 of word * K4 change)."""
    if h4:
        v = int.from_bytes(buf[y:y + 4], "little")
        p = (v * K4) & 0xFFFFFFFF
        while True:
            p2 = (p & 0xFFF00000) | int(rng.integers(0, 1 << 20))
            v2 = (p2 * K4_INV) & 0xFFFFFFFF
            if v2 != v:
                break
        buf[x:x + 4] = v2.to_bytes(4, "little")
        return
    v = int.from_bytes(buf[y:y + 5], "little")
    p = (v * K5) & M40
    while True:
        p2 = (p & ~((1 << 28) - 1) & M40) | int(rng.integers(0, 1 << 28))
        v2 = (p2 * K5_INV) & M40
        if (v2 & 0xFFFFFFFF) != (v & 0xFFFFFFFF):
            break
    buf[x:x + 5] = v2.to_bytes(5, "little")


def _copy(buf: bytearray, at: int, frm, L: int) -> None:
    """buf[at + i] = frm(i) in increasing i (an overlapping copy repeats), then a byte that ends the match."""
    for i in range(L):
        buf[at + i] = frm(i)
    if frm(L) is not None and buf[at + L] == frm(L):
        buf[at + L] ^= 0x5A


class Planter:
    """Runs planted one after another into random bytes.  rd(p) for p < 0 reads the history or dictionary."""

    def __init__(self, rng, n: int, h4: bool, before: bytes = b""):
        self.rng, self.h4, self.before = rng, h4, before
        self.buf = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())

    def rd(self, p: int):
        if p >= len(self.buf):
            return None
        return self.buf[p] if p >= 0 else self.before[len(self.before) + p]

    def length(self) -> int:
        return (4 if self.h4 else 5) + int(self.rng.integers(0, 12))

    def hit(self, base: int, q: int, post: bool, frm: int | None = None, L: int | None = None) -> int:
        """Make probe q of the run at `base` hit a copy of the bytes at `frm` (by default an earlier probe of the
        same run, or for q = 0 the position before `base`: the post probe, or position 0).  -> the match's end."""
        P = base + probe_advance(q)
        if frm is None:
            frm = base - 1 if q == 0 else base + probe_advance(q - 1 - int(self.rng.integers(0, min(q, 8))))
        L = L or self.length()
        _copy(self.buf, P, lambda i: self.rd(frm + i), L)
        return P + L

    def offset2(self, E: int) -> int:
        """An offset-2 repeat at the match end E: the post probe hits put(ip-2) with no literal."""
        L = 5 + int(self.rng.integers(0, 8))
        _copy(self.buf, E, lambda i: self.buf[E - 2 + i] if E + i < len(self.buf) else None, L)
        return E + L


def _runs(pl: Planter, base: int, post: bool, targets, stop: int, extra=None) -> tuple[int, bool]:
    """Plant runs from `base`, the t-th hitting at probe targets[t % len]; extra(pl, base, q, post, t) may plant
    more before each hit and return a replacement end.  -> (the next run's base, post) once a run would pass stop."""
    t = 0
    while True:
        q = targets[t % len(targets)]
        if base + probe_advance(q) + 40 > stop:
            return base, post
        E = extra(pl, base, q, post, t) if extra else None
        if E is None:
            E = pl.hit(base, q, post)
        base, post, t = E + 1, True, t + 1


def _finish(pl: Planter, n: int) -> bytes:
    return bytes(pl.buf[:n])


# ---- the families -----------------------------------------------------------------------------------------------

def hit_src(rng, h4: bool, q_first: int, n: int = 6000, before: bytes = b"") -> bytes:
    """The block's first run hits at q_first; every later run (behind a match) cycles through TARGETS."""
    pl = Planter(rng, n, h4, before)
    E = pl.hit(1, q_first, False)
    k = TARGETS.index(q_first)
    _runs(pl, E + 1, True, TARGETS[k:] + TARGETS[:k], n - 40)
    return _finish(pl, n)


def split_src(rng, h4: bool, post_first: bool, n: int = 8000, before: bytes = b"") -> bytes:
    """Runs whose probes share slots with earlier probes of their batch (pairs and three-way), on both sides of
    each batch edge, before their first hit at q = 70..193."""
    def extra(pl, base, q, post, t):
        edges = [e for e in ((31, 63, 95) if post else (32, 64, 96)) if e + 3 < q - 4]
        for e in edges:
            sel = t % 3
            if sel == 0:        # a pair inside the batch below the edge and a pair across it
                pairs = [(e - 6, e - 1), (e - 3, e + 2)]
            elif sel == 1:      # three probes of one batch on one slot
                pairs = [(e - 15, e - 10), (e - 15, e - 5)]
            else:               # the last lane of a batch and the first of the next on one slot
                pairs = [(e - 6, e - 1), (e - 6, e)]
            for a, b in pairs:
                pa, pb = base + probe_advance(a), base + probe_advance(b)
                if pb - pa >= 5 and a >= 0:
                    collide(pl.buf, pb, pa, pl.rng, pl.h4)
        return None
    pl = Planter(rng, n, h4, before)
    base, post = (1, False) if post_first else (pl.hit(1, 3, False) + 1, True)
    _runs(pl, base, post, (70, 100, 129, 160, 193), n - 40, extra)
    return _finish(pl, n)


def post_src(rng, h4: bool, n: int = 8000, before: bytes = b"") -> bytes:
    """Behind every match one of: an offset-2 repeat (the post lane hits through put(ip-2), h(ip) == h(ip-2));
    a later lane of the post batch on put(ip-2)'s slot and then a copy of put(ip-2)'s word, which must find that
    lane's store (the GPU drops put(ip-2)); or a lane copying put(ip-2)'s word, which finds it."""
    def extra(pl, base, q, post, t):
        if not post or q < 12:
            return None
        ip = base - 1
        kind = t % 4
        if kind == 0:                                  # the post lane hits, then the next match is planted
            E2 = pl.offset2(ip)
            return pl.hit(E2 + 1, q, True)
        j = 1 + int(pl.rng.integers(0, 6))             # lane j + 1 holds the colliding word
        if kind in (1, 2):
            collide(pl.buf, base + j, ip - 2, pl.rng, pl.h4)
            k = j + 5 + (int(pl.rng.integers(0, 4)) if kind == 1 else 31)   # same batch, or the next one
            if k < q:
                _copy(pl.buf, base + probe_advance(k), lambda i: pl.rd(ip - 2 + i), 4 if pl.h4 else 5)
            return None
        return pl.hit(base, j, True, frm=ip - 2)       # kind 3: probe j finds put(ip-2)
    pl = Planter(rng, n, h4, before)
    _runs(pl, pl.hit(1, 2, False) + 1, True, (20, 33, 40, 64, 70, 100), n - 40, extra)
    return _finish(pl, n)


def end_src(rng, h4: bool, lane: int, post: bool, second: bool, before: bytes = b"") -> bytes:
    """The last run ends at `lane` of its first (second False) or second batch, after a pair and a triple of
    probes of that batch share slots.  `post`: the run is behind a match; else it is the block's first."""
    n_max = 4000
    pl = Planter(rng, n_max, h4, before)
    if post:
        base, post_ = _runs(pl, pl.hit(1, 5, False) + 1, True, (10, 33, 64), 1500)
    else:
        base, post_ = 1, False
    q_end = (lane - (1 if post_ else 0)) + (32 if second else 0)
    if q_end < 0:
        q_end += 32
    first_q = q_end - probe_lane(q_end, post_)                  # the probe at lane 0 of the last batch
    lanes = [q for q in range(max(first_q, 0), q_end)]
    if len(lanes) >= 11:                                        # a pair and a triple before the end
        a = lanes[0]
        for b in (a + 5, a + 10):
            collide(pl.buf, base + probe_advance(b), base + probe_advance(a), pl.rng, h4)
    if len(lanes) >= 17:
        collide(pl.buf, base + probe_advance(lanes[-1]), base + probe_advance(lanes[-7]), pl.rng, h4)
    n = base + probe_advance(q_end) + 11
    return _finish(pl, n)


def tight_caps(block: bytes) -> dict:
    """From a block's token walk: a capacity at which each limitedOutput check fails first, where one exists.
    -> {"lit": [caps], "match": [caps], "last": [caps]}.  A sequence of zero literals may be a post-match hit,
    which skips the literal check; its match check then fails at the same capacities with the same state."""
    seqs, p = [], 0
    while p < len(block):
        tok = block[p]; op = p; p += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = block[p]; p += 1; lit += b
                if b != 255:
                    break
        p += lit
        if p >= len(block):
            break
        p += 2
        mc = tok & 15
        if mc == 15:
            while True:
                b = block[p]; p += 1; mc += b
                if b != 255:
                    break
        seqs.append((op, lit, mc, p))
    out = {"lit": [], "match": [], "last": []}
    need = 0
    for op, lit, mc, end in seqs:
        c_lit = op + 1 + lit + 8 + lit // 255
        hdr = 1 + (0 if lit < 15 else (lit - 15) // 255 + 1)
        c_match = op + hdr + lit + 2 + 6 + (mc + 240) // 255
        if lit and c_lit - 1 >= need:
            out["lit"].append(c_lit - 1)
        if c_match - 1 >= max(need, c_lit if lit else 0):
            out["match"].append(c_match - 1)
        need = max(need, c_lit if lit else 0, c_match)
    if len(block) - 1 >= need:
        out["last"].append(len(block) - 1)
    return out


# ---- history: prefix-mode states and extDict dictionaries -------------------------------------------------------

def _history_table(rng, st: int, d: int, hist: bytes, h4: bool, n_slots: int = 3000) -> np.ndarray:
    """A planted table: random slots hold indices of history positions (some beyond 65 535 back)."""
    table = np.zeros(4096, dtype=np.uint32)
    H, unit = (hash4_12, 4) if h4 else (hash5_12, 8)
    for p in rng.integers(0, d - unit, n_slots):
        table[H(hist[p:p + unit])] = st - d + int(p)
    return table


def history_cases(rng, h4: bool) -> list:
    """Prefix-mode cases on planted states: a candidate 65 535 back (accepted) and 65 536 back (rejected) at a
    lane >= 1 of a batch whose later lane hits; a stale history slot that a same-hash lane of the batch forwards
    over; a candidate below startIndex - d under dictSmall mid-batch; catch-ups that cross into the history and
    stop at -d."""
    H, unit = (hash4_12, 4) if h4 else (hash5_12, 8)
    cases = []
    # distances, in the first run and in a run behind a match
    hist = rng.integers(0, 256, 70000, dtype=np.uint8).tobytes()
    st = 300000
    for dist in (65535, 65536):
        for lane in (1, 7, 30, 31):
            for post in (False, True):
                table = _history_table(rng, st, len(hist), hist, h4)
                pl = Planter(rng, 3000, h4, hist)
                base, pst = (1, False) if not post else (pl.hit(1, 4, False) + 1, True)
                q = lane - (1 if pst else 0) + 32
                P = base + probe_advance(q)
                frm = P - dist
                pl.hit(base, q, pst, frm=frm, L=12)
                table[H(pl.buf[P:P + unit])] = st + frm
                E = pl.hit(base, q + 13, pst)           # past the 12 copied bytes
                _runs(pl, E + 1, True, (5, 40), 2960)
                s = CE.make_state(table, st, len(hist))
                cases.append(Case(f"dist{dist}-lane{lane}-{'post' if post else 'first'}", "history", False, h4,
                                  hist, _finish(pl, 3000), s, bound(3000)))
    # a stale slot of the planted state, forwarded over by an earlier lane of the same batch with its hash
    for lane_a, lane_b in ((3, 9), (30, 31), (0, 31), (20, 25)):
        table = _history_table(rng, st, len(hist), hist, h4)
        pl = Planter(rng, 3000, h4, hist)
        pa, pb = 1 + lane_a + 64, 1 + lane_b + 64
        t = -int(rng.integers(100, 60000))
        _copy(pl.buf, pb, lambda i: pl.rd(t + i), 12)
        table[H(pl.buf[pb:pb + unit])] = st + t
        if pb - pa >= 5:
            collide(pl.buf, pa, pb, rng, h4)
        else:
            table[H(pl.buf[pb:pb + unit])] = st + t
        E = pl.hit(1, lane_b + 64 + 20, False)
        _runs(pl, E + 1, True, (30, 64), 2960)
        cases.append(Case(f"stale-{lane_a}-{lane_b}", "history", False, h4, hist, _finish(pl, 3000),
                          CE.make_state(table, st, len(hist)), bound(3000)))
    # dictSmall: d = 2000 < 65 536 and < startIndex; slots point below startIndex - d mid-batch
    small = rng.integers(0, 256, 2000, dtype=np.uint8).tobytes()
    for lane in (5, 17, 31):
        st2 = 100000
        table = _history_table(rng, st2, len(small), small, h4, 500)
        pl = Planter(rng, 3000, h4, small)
        P = 1 + lane + 32
        table[H(pl.buf[P:P + unit])] = st2 - 2000 - int(rng.integers(1, 3000))   # below the window, < 65 535 back
        q_hit = lane + 32 + 2 + int(rng.integers(0, 10))
        frm = -int(rng.integers(50, 1900))                                        # a hit in the window after it
        pl.hit(1, q_hit, False, frm=frm, L=10)
        Pq = 1 + probe_advance(q_hit)
        table[H(pl.buf[Pq:Pq + unit])] = st2 + frm
        cases.append(Case(f"dictsmall-{lane}", "history", False, h4, small, _finish(pl, 3000),
                          CE.make_state(table, st2, len(small)), bound(3000)))
    # catch-ups into the history, stopped at -d (the history's first byte) with literals still in front
    for d in (100, 3000, 40000):
        hist2 = rng.integers(0, 256, d, dtype=np.uint8).tobytes()
        for k in (1, 7, 30, 60):
            st3 = 500000
            table = _history_table(rng, st3, d, hist2, h4, 200)
            pl = Planter(rng, 3000, h4, hist2)
            q = 40 + k
            P = 1 + probe_advance(q)
            for i in range(k):                       # the bytes before the hit equal the history's first k
                pl.buf[P - k + i] = hist2[i]
            _copy(pl.buf, P, lambda i: hist2[k + i], 12)
            table[H(hist2[k:k + unit])] = st3 - d + k
            _runs(pl, P + 13, True, (10, 33), 2960)
            cases.append(Case(f"floor-d{d}-k{k}", "history", False, h4, hist2, _finish(pl, 3000),
                              CE.make_state(table, st3, d), bound(3000)))
    return cases


def _loaded_positions(dictionary: bytes) -> dict:
    """{kept-dictionary position: slot} of the positions LZ4_loadDict's table still holds."""
    d = DR.kept(len(dictionary))
    table = DR.load_table(dictionary).view(np.uint32)[:4096]
    tail = dictionary[len(dictionary) - d:]
    out = {}
    for p in range(0, d - 7, 3):
        h = hash5_12(tail[p:p + 8])
        if int(table[h]) == 65536 - d + p:
            out[p] = h
    return out


def ext_cases(rng) -> list:
    """extDict cases: matches into the dictionary whose count crosses its end into src[0] (the candidate 0..7
    positions before the last possible one, the match running 0..8 bytes into the source), for every size in
    DICT_SIZES; dictionary matches whose catch-up stops at the dictionary's start; a source match whose catch-up
    stops at the source's start although the dictionary's last byte would match; and the families' content."""
    cases = []
    for dn in DICT_SIZES:
        dic = rng.integers(0, 256, dn, dtype=np.uint8).tobytes()
        d = DR.kept(dn)
        tail = dic[dn - d:]
        held = _loaded_positions(dic)
        ends = sorted((p for p in held if p >= d - 8 - 7), reverse=True)   # the last loaded positions
        for rep in range(2):
            pl = Planter(rng, 2500, False, tail)
            base, post = 1, False
            for j, p in enumerate(ends):
                into = (j + 3 * rep) % 9
                q = 20 + 7 * j
                P = base + probe_advance(q)
                L = d - p                              # to the dictionary's end, then `into` bytes of src[0..]
                seg = tail[p:] + bytes(pl.buf[:into])
                # the copy ends where src[into] would have continued the match
                _copy(pl.buf, P, lambda i: seg[i] if i < len(seg) else pl.buf[into], len(seg))
                base, post = P + len(seg) + 1, True
            _runs(pl, base, post, (20, 64), 2460)
            cases.append(Case(f"straddle-d{dn}-{rep}", "straddle", True, False, dic, _finish(pl, 2500), None,
                              bound(2500)))
        if d >= 64:                                    # catch-up down to the dictionary's start
            for k in sorted(p for p in held if 0 < p <= 300)[:3]:
                pl = Planter(rng, 2000 + 2 * k, False, tail)
                q = 30 + k
                P = 1 + probe_advance(q)
                for i in range(k):
                    pl.buf[P - k + i] = tail[i]
                _copy(pl.buf, P, lambda i: tail[k + i], 10)
                _runs(pl, P + 11, True, (10, 40), len(pl.buf) - 40)
                cases.append(Case(f"dictfloor-d{dn}-k{k}", "history", True, False, dic, bytes(pl.buf), None,
                                  bound(len(pl.buf))))
    for seed in range(3):                              # the source's start bounds a source match
        src, dic = DR.catchup_input(seed + 5)
        cases.append(Case(f"srcfloor-{seed}", "history", True, False, dic, src, None, bound(len(src))))
    return cases


# ---- all cases ----------------------------------------------------------------------------------------------

def _prefix_state(up, rng, kind: int, hist: bytes) -> np.ndarray:
    """The state in front of a block: upstream's after encoding `hist` as a stream's block, or a planted one."""
    if kind == 0:
        st = up.lib.LZ4_createStream()
        try:
            a = np.frombuffer(hist, dtype=np.uint8)
            up.compress(st, a.ctypes.data, len(hist), bound(len(hist)))
            return up.state_of(st)
        finally:
            up.lib.LZ4_freeStream(st)
    s = 1 << 20
    return CE.make_state(_history_table(rng, s, len(hist), hist, False), s, len(hist))


def family_cases(up, up32, seed: int = 7) -> list:
    """Every family in every mode.  `up` is chain_enc_ref.EncUpstream (it makes the prefix states of hash5
    cases), `up32` the 32-bit engine's (hash4)."""
    rng = np.random.default_rng(seed)
    cases = []
    for h4 in (False, True):
        eng = up32 if h4 else up
        tag = "h4" if h4 else "h5"

        def pre(name, fam, make, k):
            hist = rng.integers(0, 256, (5000, 70000)[k % 2], dtype=np.uint8).tobytes() if k % 3 else b""
            st = _prefix_state(eng, rng, k % 2, hist) if hist else CE.make_state()
            if hist and k % 2 and h4:
                st = _prefix_state(eng, rng, 0, hist)
            src = make(hist)
            cases.append(Case(f"{fam}-{tag}-{name}", fam, False, h4, hist, src, st, bound(len(src))))
        for i, q in enumerate(TARGETS):
            pre(f"q{q}", "hit", lambda hist, q=q: hit_src(rng, h4, q, before=hist), i)
        for i in range(4):
            pre(f"{i}", "split", lambda hist, i=i: split_src(rng, h4, i % 2 == 0, before=hist), i)
            pre(f"{i}", "post", lambda hist: post_src(rng, h4, before=hist), i)
        for lane in range(32):
            for j, (post, second) in enumerate(((False, False), (False, True), (True, False), (True, True))):
                pre(f"e{lane}-{int(post)}{int(second)}", "end",
                    lambda hist, lane=lane, post=post, second=second: end_src(rng, h4, lane, post, second, hist),
                    lane + j)
        for c in history_cases(rng, h4):
            c.name = f"{c.name}-{tag}"
            cases.append(c)
    # extDict: the hash5 families over dictionaries, and the dictionary-only cases
    for i, q in enumerate(TARGETS):
        dic = rng.integers(0, 256, DICT_SIZES[i % len(DICT_SIZES)], dtype=np.uint8).tobytes()
        cases.append(Case(f"hit-ext-q{q}", "hit", True, False, dic, hit_src(rng, False, q), None, bound(6000)))
    for i in range(4):
        dic = rng.integers(0, 256, 4096 << (i % 3), dtype=np.uint8).tobytes()
        cases.append(Case(f"split-ext-{i}", "split", True, False, dic, split_src(rng, False, i % 2 == 0), None,
                          bound(8000)))
        cases.append(Case(f"post-ext-{i}", "post", True, False, dic, post_src(rng, False), None, bound(8000)))
    for lane in range(0, 32, 3):
        dic = rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()
        src = end_src(rng, False, lane, lane % 2 == 0, lane % 4 < 2)
        cases.append(Case(f"end-ext-e{lane}", "end", True, False, dic, src, None, bound(len(src))))
    cases += ext_cases(rng)
    return cases


def tight_cases(cases: list, want: dict, every: int = 3) -> list:
    """Cases of `cases` (every `every`-th) again with each capacity tight_caps finds in the block `want[name]`
    (upstream's at the bound): the first, a middle and the last sequence of each check."""
    out = []
    for c in cases[::every]:
        caps = tight_caps(want[c.name])
        for check, cs in caps.items():
            for cap in sorted({cs[0], cs[len(cs) // 2], cs[-1]} if cs else ()):
                out.append(Case(f"{c.name}-{check}{cap}", "tight", c.ext, c.h4, c.before, c.src, c.state, cap))
    return out
