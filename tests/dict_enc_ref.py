"""Encoding against an external dictionary: test infrastructure for k4lz4_encode_dict_batch.

* ``load_table`` restates LZ4_loadDict (orig/lib/lz4.c:1475-1514, 64-bit: HASH_UNIT 8, hash5) in numpy: the last
  writer per slot, which is the largest position.
* ``DictUpstream`` drives upstream's own engine (oracle/_ref/libk4ref.so): ``encode`` is the oracle of one block,
  LZ4_loadDict on the dictionary in a buffer of its own followed by LZ4_compress_fast_continue (the usingExtDict
  branch); ``encode_prefix`` loads the same bytes directly in front of the source, so that the same call takes the
  prefix branch instead; ``loaded`` is the state LZ4_loadDict leaves, as a K4LZ4_CHAIN_STATE_BYTES record.
* ``records`` makes seeded JSON-like records that share a vocabulary, the content dictionaries are made for.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from tests import chain_enc_ref as CE

K64 = 65536
PRIME5 = np.uint64(889523592379)


def kept(n: int) -> int:
    """The dictionary bytes LZ4_loadDict keeps: the last min(n, 65 536), none below 8."""
    return 0 if n < 8 else min(n, K64)


def load_table(dictionary: bytes) -> np.ndarray:
    """The K4LZ4_CHAIN_STATE_BYTES record LZ4_loadDict leaves (currentOffset 65 536, dictSize = kept bytes)."""
    d = kept(len(dictionary))
    table = np.zeros(4096, dtype=np.uint32)
    if d:
        tail = np.frombuffer(dictionary[len(dictionary) - d:], dtype=np.uint8)
        pos = np.arange(0, d - 8 + 1, 3, dtype=np.int64)
        words = np.zeros(len(pos), dtype=np.uint64)
        for k in range(8):
            words |= tail[pos + k].astype(np.uint64) << np.uint64(8 * k)
        with np.errstate(over="ignore"):
            h = (((words << np.uint64(24)) * PRIME5) >> np.uint64(52)).astype(np.int64)
        vals = (K64 - d + pos).astype(np.uint32)
        table[h] = vals                              # numpy: for repeated indices the last assignment wins
    return CE.make_state(table, K64, d)


class DictUpstream(CE.EncUpstream):
    def __init__(self):
        super().__init__()
        L = self.lib
        L.LZ4_loadDict.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.LZ4_loadDict.restype = C.c_int

    def loaded(self, dictionary: bytes) -> np.ndarray:
        dic = np.frombuffer(bytes(dictionary) + b"\0", dtype=np.uint8)
        st = self.lib.LZ4_createStream()
        try:
            self.lib.LZ4_loadDict(st, dic.ctypes.data, len(dictionary))
            return self.state_of(st)
        finally:
            self.lib.LZ4_freeStream(st)

    def encode(self, src: bytes, dictionary: bytes, cap: int | None = None) -> tuple[int, bytes]:
        """-> (upstream's result, bytes) with the dictionary in a buffer of its own (extDict)."""
        cap = len(src) + len(src) // 255 + 16 if cap is None else cap
        dic = np.frombuffer(bytes(dictionary) + b"\0" * 8, dtype=np.uint8)
        s = np.frombuffer(bytes(src) + b"\0" * 8, dtype=np.uint8)
        st = self.lib.LZ4_createStream()
        try:
            self.lib.LZ4_loadDict(st, dic.ctypes.data, len(dictionary))
            return self.compress(st, s.ctypes.data, len(src), cap)
        finally:
            self.lib.LZ4_freeStream(st)

    def encode_prefix(self, src: bytes, dictionary: bytes, cap: int | None = None) -> tuple[int, bytes]:
        """The same load, the dictionary directly in front of the source: the prefix branch."""
        cap = len(src) + len(src) // 255 + 16 if cap is None else cap
        buf = np.frombuffer(bytes(dictionary) + bytes(src) + b"\0" * 8, dtype=np.uint8)
        st = self.lib.LZ4_createStream()
        try:
            self.lib.LZ4_loadDict(st, buf.ctypes.data, len(dictionary))
            return self.compress(st, buf.ctypes.data + len(dictionary), len(src), cap)
        finally:
            self.lib.LZ4_freeStream(st)

    def decode(self, block: bytes, n: int, dictionary: bytes) -> tuple[int, bytes]:
        """LZ4_decompress_safe_usingDict with the dictionary in a buffer of its own."""
        dic = np.frombuffer(bytes(dictionary) + b"\0", dtype=np.uint8)
        s = np.frombuffer(bytes(block) + b"\0", dtype=np.uint8)
        out = np.zeros(max(n, 1), dtype=np.uint8)
        r = int(self.lib.LZ4_decompress_safe_usingDict(s.ctypes.data, out.ctypes.data, len(block), n,
                                                       dic.ctypes.data, len(dictionary)))
        return r, out[:max(r, 0)].tobytes()


_WORDS = ["user", "id", "name", "email", "created_at", "status", "active", "pending", "score", "tags", "items",
          "price", "quantity", "currency", "EUR", "USD", "country", "city", "Berlin", "Paris", "Tokyo", "true",
          "false", "null", "session", "token", "version", "platform", "android", "ios", "web", "event", "click"]


def records(n_bytes: int, seed: int) -> bytes:
    """Seeded JSON-like records of a shared vocabulary, n_bytes long."""
    rng = np.random.default_rng(seed)
    out, total = [], 0
    while total < n_bytes:
        k = int(rng.integers(3, 8))
        fields = []
        for _ in range(k):
            key = _WORDS[int(rng.integers(len(_WORDS)))]
            if rng.random() < 0.5:
                val = str(int(rng.integers(0, 100000)))
            else:
                val = '"' + _WORDS[int(rng.integers(len(_WORDS)))] + '"'
            fields.append(f'"{key}":{val}')
        r = "{" + ",".join(fields) + "}\n"
        out.append(r)
        total += len(r)
    return "".join(out).encode()[:n_bytes]


def catchup_input(seed: int = 5) -> tuple[bytes, bytes]:
    """(source, dictionary) where the source's second copy of its first 16 bytes is preceded by the dictionary's
    last 6 bytes: the match found in the source would catch up into the dictionary in the prefix mode only."""
    rng = np.random.default_rng(seed)
    dictionary = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
    head = rng.integers(0, 256, 16, dtype=np.uint8).tobytes()
    gap = rng.integers(0, 256, 40, dtype=np.uint8).tobytes()
    tail = rng.integers(0, 256, 200, dtype=np.uint8).tobytes()
    return head + gap + dictionary[-6:] + head + tail, dictionary
