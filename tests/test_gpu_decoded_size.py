"""k4lz4_decoded_size_batch on the GPU: the warp walk of csrc/size_walk.cuh against the serial walk
(test_frame_model.walk) and the oracle decoder, in host and device memory, with its argument checks and the
2^31 - 1 limit; a device-memory call records into a CUDA graph (it never waits on the host)."""
import numpy as np
import pytest

from tests import block_mutants as BM
from tests import lz4_blocks as LB
from tests.test_frame_model import walk

pytestmark = pytest.mark.gpu
LIMIT = 0x7FFFFFFF


@pytest.fixture(scope="module")
def k4(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    return k


def _device(k4, blocks):
    import torch
    from k4os.compression.lz4_b200 import batch as B
    src, so, sl = B._pack(blocks)
    d = torch.device("cuda", 0)
    ts, tso, tsl = (torch.from_numpy(x.copy()).to(d) for x in (src, so, sl))
    out = torch.full((len(blocks),), -7, dtype=torch.int32, device=d)
    B.decoded_size_batch_device(ts.data_ptr(), tso.data_ptr(), tsl.data_ptr(), out.data_ptr(), len(blocks),
                                torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _both(k4, blocks):
    """-> sizes; host and device memory must agree"""
    h = k4.batch.decoded_size_batch_host(blocks)
    d = _device(k4, blocks)
    assert np.array_equal(h, d), np.flatnonzero(h != d)[:8]
    return h


def test_oracle_blocks_give_their_raw_length(k4, port):
    raws = [b""] + [port.datagen(n, 0.63, 0.0, n).tobytes() for n in (1, 12, 13, 65536, 65547, 1 << 20, 4 << 20)]
    blocks = [b""] + [port.encode(r)[1] for r in raws[1:]]
    assert list(_both(k4, blocks)) == [len(r) for r in raws]


def test_mutants_tails_and_hand_built_chains(k4, port):
    rng = np.random.default_rng(12)
    streams = []
    for base in BM.independent_bases():
        streams += [m.stream for m in BM.chain_breaking(base, rng)]
        streams += [m.stream for m in BM.layout_mutants(base, rng)[::11]]
        streams += [base.stream[:c] for c in range(len(base.stream) - 20, len(base.stream) + 1)]
    rb = lambda k: bytes(rng.integers(0, 256, k, dtype=np.uint8))
    for L in (14, 15, 270, 255 * 64 + 15, 255 * 130 + 3):
        for lead in range(0, 64, 9):
            seqs = [(rb(lead + 1), 1, 4), (rb(L), 1, L + 4), (rb(3), 2, 4), (rb(L // 3), 7, L // 2 + 4)]
            streams.append(LB.build_block(seqs, rb(int(rng.integers(0, 40))))[0])
    streams += [b"\x00", b"\x10a", b"\xf0" + b"\xff" * 3, b"\x0f\x01\x00\xff\x00", b"\x0f\x01\x00\xff\x00\x00"]
    got = _both(k4, streams)
    accepted = 0
    for s, g in zip(streams, got):
        w = walk(s)
        assert int(g) == (w if 0 <= w <= LIMIT else -1), (len(s), int(g), w)
        r, _ = port.decode(s, 1 << 24)
        if r > 0:
            accepted += 1
            assert int(g) == r
    assert len(streams) > 1500 and accepted > 100


def test_length_limit_on_the_device(k4):
    """A match whose 0xFF extension run makes the walk 2^31 - 1 + 128 gives -1; one 255 shorter is exact."""
    import torch
    from k4os.compression.lz4_b200 import batch as B
    d = torch.device("cuda", 0)
    K = (LIMIT - 19) // 255 + 1                       # 15 + 255 K + 4 > 2^31 - 1
    head = torch.tensor([0x0F, 1, 0], dtype=torch.uint8, device=d)
    tail = torch.tensor([0, 0], dtype=torch.uint8, device=d)
    over = torch.cat([head, torch.full((K,), 0xFF, dtype=torch.uint8, device=d), tail])
    under = torch.cat([head, torch.full((K - 1,), 0xFF, dtype=torch.uint8, device=d), tail])
    src = torch.cat([over, under])
    so = torch.tensor([0, over.numel()], dtype=torch.int64, device=d)
    sl = torch.tensor([over.numel(), under.numel()], dtype=torch.int32, device=d)
    out = torch.full((2,), -7, dtype=torch.int32, device=d)
    B.decoded_size_batch_device(src.data_ptr(), so.data_ptr(), sl.data_ptr(), out.data_ptr(), 2,
                                torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert 15 + 255 * K + 4 > LIMIT >= 15 + 255 * (K - 1) + 4
    assert out.cpu().tolist() == [-1, 15 + 255 * (K - 1) + 4]


def test_argument_errors_in_header_order(k4, native):
    from k4os.compression.lz4_b200 import _native as N
    f = native.k4lz4_decoded_size_batch
    keep = [np.zeros(16, dtype=np.int64) for _ in range(4)]
    p = [a.ctypes.data for a in keep]
    assert f(*p, 1, 7, None, 0) == N.E_ARG                       # unknown memKind first
    assert f(None, None, None, None, -1, N.MEM_HOST, None, 0) == N.E_ARG
    assert f(p[0], p[1], p[2], None, 1, N.MEM_HOST, None, 0) == N.E_ARG
    assert f(None, None, None, None, 0, N.MEM_DEVICE, None, 0) == N.OK
    assert f(*p, 1, N.MEM_HOST, None, native.k4lz4_device_count()) == N.E_ARG
    keep[3][:] = -1
    assert f(*p, 1, N.MEM_HOST, None, N.ALL_DEVICES) == N.OK    # zeroed source arrays: one empty block
    assert int(keep[3].view(np.int32)[0]) == 0


def test_device_call_records_into_a_cuda_graph(k4, port):
    import torch
    from k4os.compression.lz4_b200 import batch as B
    raws = [port.datagen(65536, 0.63, 0.0, 70 + i).tobytes() for i in range(64)]
    src, so, sl = B._pack([port.encode(r)[1] for r in raws])
    d = torch.device("cuda", 0)
    ts, tso, tsl = (torch.from_numpy(x.copy()).to(d) for x in (src, so, sl))
    out = torch.zeros(64, dtype=torch.int32, device=d)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        B.decoded_size_batch_device(ts.data_ptr(), tso.data_ptr(), tsl.data_ptr(), out.data_ptr(), 64, s.cuda_stream)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        B.decoded_size_batch_device(ts.data_ptr(), tso.data_ptr(), tsl.data_ptr(), out.data_ptr(), 64, s.cuda_stream)
    out.fill_(-7)
    g.replay()
    torch.cuda.synchronize()
    assert out.cpu().tolist() == [65536] * 64
