"""Generates the committed golden fixtures.  Run in the build container (needs /root/reference):

    python tests/golden/make_golden.py

1. issue64_block0.{lz4,bin}: the reference's own golden DECODE vector -- block #0 of
   /root/reference/assets/issue64/input.dat (a "bv41" container: 12-byte header at byte 20,
   14 505 compressed bytes -> 65 536 bytes == output.dat[0:65536]); exercised by the
   reference's Issue64.cs:16-55.  issue64_block1.{lz4,bin}: block #1 of the same file (366 -> 3 034
   bytes), which only decodes with block #0's output as external dictionary.
2. encode_rows.json: known-answer rows for LZ4Codec.Encode at L00_FAST in the style of the
   reference's ChecksumBlockTests.cs:185-216 (exact length, Adler-32 of the compressed bytes,
   first 60 compressed bytes base64) over the deterministic inputs of tests/inputs.py,
   produced -- like the reference's own rows (playground/SharedSources/app.cpp:94-97) -- by the
   upstream C engine orig/lib/lz4.c compiled as-is (oracle/_ref/libk4ref.so), including
   limited-output capacities and the expected return codes.
3. ref_digests.json: for each differential test of tests/test_oracle.py, the SHA-256 of the reference
   engine's results over that test's cases; the tests compare the restatement with it where
   oracle/_ref is not built.
"""
import base64
import hashlib
import json
import os
import struct
import sys
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from tests import inputs  # noqa: E402

REF = "/root/reference"


def main():
    oracle.build()
    R = oracle.Ref()
    # 1. issue64
    blob = open(os.path.join(REF, "assets/issue64/input.dat"), "rb").read()
    expect = open(os.path.join(REF, "assets/issue64/output.dat"), "rb").read()
    assert blob[20:24] == b"bv41"
    usize, csize = struct.unpack("<II", blob[24:32])
    comp = blob[32:32 + csize]
    r, out = R.decode(comp, usize)
    assert r == usize == 65536 and out == expect[:usize]
    open(os.path.join(HERE, "issue64_block0.lz4"), "wb").write(comp)
    open(os.path.join(HERE, "issue64_block0.bin"), "wb").write(expect[:usize])
    # block #1 needs block #0's output as its dictionary (Issue64.cs:39-49)
    pos1 = 32 + csize
    assert blob[pos1:pos1 + 4] == b"bv41"
    usize1, csize1 = struct.unpack("<II", blob[pos1 + 4:pos1 + 12])
    comp1 = blob[pos1 + 12:pos1 + 12 + csize1]
    r1, out1 = R.decode_dict(comp1, usize1, expect[:usize])
    assert r1 == usize1 == 3034 and csize1 == 366 and out1 == expect[usize:usize + usize1]
    assert blob[pos1 + 12 + csize1:pos1 + 16 + csize1] == b"bv4$"
    open(os.path.join(HERE, "issue64_block1.lz4"), "wb").write(comp1)
    open(os.path.join(HERE, "issue64_block1.bin"), "wb").write(out1)

    # 2. encode rows
    rows = []
    sizes = inputs.THRESHOLD_SIZES + inputs.BIG_SIZES
    for kind in inputs.KINDS:
        for n in sizes:
            if kind.startswith("synth") and n < 13:
                continue
            seed = 0xAA if kind == "repeat" else (n * 7 + 1) & 0xFFFF
            data = inputs.gen(kind, n, seed)
            r, c = R.encode(data)
            row = {"kind": kind, "size": n, "seed": seed, "len": r,
                   "adler32": zlib.adler32(c) & 0xFFFFFFFF,
                   "sha256": hashlib.sha256(c).hexdigest(),
                   "head60": base64.b64encode(c[:60]).decode()}
            caps = sorted({c_ for c_ in (n, 1024, r, r - 1, r + 1, max(r // 2, 1), n + n // 255 + 15)
                           if c_ > 0})
            row["limited"] = [[cap, R.encode(data, cap)[0]] for cap in caps]
            rows.append(row)
    json.dump({"engine": "orig/lib/lz4.c LZ4_compress_fast(src,dst,n,cap,1)",
               "lz4_version": R.version(), "rows": rows},
              open(os.path.join(HERE, "encode_rows.json"), "w"), indent=0)
    print(len(rows), "encode rows; issue64 ok")

    # 3. ref_digests.json: one digest per differential test of tests/test_oracle.py over the reference
    # engine's results, so that those tests also run where oracle/_ref cannot be built
    from tests import test_oracle as T
    digests = {}

    def record(name, port, results_of):
        digests[name] = T._digest(results_of(R))
    T._pin, saved = record, T._pin
    try:
        port = oracle.Port()
        for fn in (T.test_port_equals_reference_engine, T.test_malformed_decode_matches_reference_engine,
                   T.test_datagen_port_matches_reference_generator, T.test_dictionary_decode_matches_reference_engine,
                   T.test_partial_decode_matches_reference_engine, T.test_xxh32_restatement_matches_upstream):
            fn(port)
    finally:
        T._pin = saved
    json.dump(digests, open(os.path.join(HERE, "ref_digests.json"), "w"), indent=1, sort_keys=True)
    print(len(digests), "reference digests")


if __name__ == "__main__":
    main()
