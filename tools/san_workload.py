"""tools/san_workload.py -- a small pass over every kernel of libk4lz4 for compute-sanitizer
(memcheck / racecheck / synccheck); results are checked against the oracle so that a sanitizer-clean
run is also a correct run.  Sized for the ~50x slowdown of the tools.
    compute-sanitizer --tool memcheck python tools/san_workload.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import oracle
import k4os.compression.lz4_b200 as k4
if len(sys.argv) > 2 and sys.argv[1] == "--lib":       # another build of the library (e.g. -DK4_DT_NEARSPIN=0)
    from k4os.compression.lz4_b200 import _native as _N
    _N.SO_PATH = os.path.abspath(sys.argv[2])
from tests import inputs

port = oracle.Port()
bs = 65536
raw = port.datagen(6 * bs, 0.63, 0.0, 1234)
blocks = [raw[i * bs:(i + 1) * bs].tobytes() for i in range(6)]
blocks += [inputs.gen("text2", 20000, 1), inputs.gen("runs", 65536, 2), inputs.gen("lorem", 65536, 3),
           inputs.gen("random", 65536, 4), inputs.gen("random", 45000, 5) + b"\x07" * 20000, inputs.gen("text2", 100000, 6),
           b"abc", b""]
enc, lens = k4.batch.encode_batch_host(blocks)
for b, e, n in zip(blocks, enc, lens):
    assert (int(n), e) == port.encode(b), len(b)
dec, dl = k4.batch.decode_batch_host(enc, [len(b) for b in blocks])
assert dec == blocks
# more blocks than one round of the shared-memory-table encoder kernel: the global-table kernel takes part
many = [raw[(i * 37) % (5 * bs):(i * 37) % (5 * bs) + 40 + (i * 13) % 900].tobytes() for i in range(1400)]
me, ml = k4.batch.encode_batch_host(many)
for b, e, n in zip(many, me, ml):
    assert (int(n), e) == port.encode(b), len(b)
rng = np.random.default_rng(1)
bad = [inputs.mutate(enc[i % 7], rng) for i in range(40)]
caps = [len(blocks[i % 7]) for i in range(40)]
got = k4.batch.decode_batch_host(bad, caps)[1]
assert got.tolist() == [port.decode(c, cap)[0] for c, cap in zip(bad, caps)]
msgs = [inputs.gen("text2", n, n) for n in (1, 100, 300, 1024, 1025, 4096)]
pk, _ = k4.batch.pickle_batch_host(msgs)
assert pk == [port.pickle(m) for m in msgs]
assert k4.batch.unpickle_batch_host(pk)[0] == msgs
pw, _ = k4.batch.pickle_writer_batch_host(msgs)
assert pw == [port.pickle_writer(m) for m in msgs]
dic = blocks[0]
dd, dr = k4.batch.decode_dict_batch_host(enc[:3], [bs] * 3, [dic] * 3)
assert dd == blocks[:3]
pd, pr = k4.batch.partial_decode_batch_host(enc[:3], [1000, 65536, 5])
assert pd == [blocks[0][:1000], blocks[1], blocks[2][:5]]
cr, cd = k4.batch.decode_chain_blocks_host(enc[:3], [b"", blocks[5], blocks[6][:100]], [bs] * 3)
assert cd == blocks[:3]
from k4os.compression.lz4_b200 import frame
xs = frame.xxh32_batch(raw, [0, bs, 7], [bs, 100, 0])
assert xs.tolist() == [port.xxh32(raw[:bs].tobytes()), port.xxh32(raw[bs:bs + 100].tobytes()), port.xxh32(b"")]
print("san workload ok:", k4.batch.decode_stats(0))
