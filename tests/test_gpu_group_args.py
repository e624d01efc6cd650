"""The argument checks of every resident group's exports (k4lz4_chain_group_*, k4lz4_frame_writer_group_*,
k4lz4_frame_reader_group_*) on real groups, in host and device memory: the codes k4lz4.h gives for each argument
error, and the calls that must succeed (a reset listing a stream twice, n = 0 with null pointers)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
S = 4
OK, E_ARG = 0, -102
MEM_HOST, MEM_DEVICE = 0, 1

# each call's pointer arguments after the group, by role
ROLES = {
    "chain_encode": ["streams", "src", "off", "len", "dst", "off", "cap", "out"],
    "chain_decode": ["streams", "src", "off", "len", "dst", "off", "cap", "out"],
    "chain_inject": ["streams", "src", "off", "len"],
    "writer_write": ["streams", "src", "off", "len", "dst", "off", "cap", "out"],
    "writer_close": ["streams", "dst", "off", "cap", "out"],
    "reader_read": ["streams", "src", "off", "len", "used", "dst", "off", "cap", "out", "ended"],
    "reader_end": ["streams", "out"],
}
EXPORT = {
    "chain_encode": "k4lz4_chain_group_encode", "chain_decode": "k4lz4_chain_group_decode",
    "chain_inject": "k4lz4_chain_group_inject", "writer_write": "k4lz4_frame_writer_group_write",
    "writer_close": "k4lz4_frame_writer_group_close", "reader_read": "k4lz4_frame_reader_group_read",
    "reader_end": "k4lz4_frame_reader_group_end",
}
RESET = {"chain_enc": "k4lz4_chain_group_reset", "chain_dec": "k4lz4_chain_group_reset",
         "writer": "k4lz4_frame_writer_group_reset", "reader": "k4lz4_frame_reader_group_reset"}
GROUP_OF = {"chain_encode": "chain_enc", "chain_decode": "chain_dec", "chain_inject": "chain_dec",
            "writer_write": "writer", "writer_close": "writer", "reader_read": "reader", "reader_end": "reader"}


@pytest.fixture(scope="module")
def groups(native):
    import k4os.compression.lz4_b200 as k
    if native.k4lz4_device_count() <= 0:
        pytest.fail("no CUDA device: GPU tests must run on an H100")
    gs = {"chain_enc": k.ChainEncoderGroup(S, 1024), "chain_dec": k.ChainDecoderGroup(S, 1024),
          "writer": k.FrameWriterGroup(S), "reader": k.FrameReaderGroup(S)}
    yield gs
    for name, g in gs.items():
        (g.close if name.startswith("chain") else g.free)()


class Args:
    """Two entries' worth of every role in host or device memory, kept alive by the object."""

    def __init__(self, mem, streams=(0, 1), lens=(3, 3)):
        import torch
        host = {"streams": np.array(streams, np.int32), "src": np.zeros(64, np.uint8),
                "off": np.zeros(2, np.int64), "len": np.array(lens, np.int32),
                "dst": np.zeros(64, np.uint8), "cap": np.full(2, 64, np.int32), "out": np.zeros(2, np.int32),
                "used": np.zeros(2, np.int32), "ended": np.zeros(2, np.int32)}
        if mem == MEM_HOST:
            self.keep = host
            self.ptr = {r: a.ctypes.data for r, a in host.items()}
        else:
            self.keep = {r: torch.from_numpy(a).cuda() for r, a in host.items()}
            self.ptr = {r: t.data_ptr() for r, t in self.keep.items()}

    def call(self, L, call, g, n, mem, null=None, level=0):
        ps = [None if r == null else self.ptr[r] for r in ROLES[call]]
        fn = getattr(L, EXPORT[call])
        if call == "chain_encode":
            return fn(g, *ps, n, level, mem, None)
        return fn(g, *ps, n, mem, None)


def _sync():
    import torch
    torch.cuda.synchronize()


@pytest.mark.parametrize("mem", [MEM_HOST, MEM_DEVICE])
@pytest.mark.parametrize("call", list(ROLES))
def test_step_call_arguments(native, groups, call, mem):
    L = native
    g = groups[GROUP_OF[call]].handle
    a = Args(mem)
    assert a.call(L, call, None, 2, mem) == E_ARG                 # no group
    assert a.call(L, call, g, 2, 5) == E_ARG                      # unknown memKind
    assert a.call(L, call, g, 0, 5) == E_ARG                      # ... before n == 0 is done
    assert a.call(L, call, g, -1, mem) == E_ARG
    for role in sorted(set(ROLES[call])):                         # each required pointer null in turn
        assert a.call(L, call, g, 2, mem, null=role) == E_ARG, role
    nulls = Args(mem)
    nulls.ptr = {r: None for r in nulls.ptr}
    assert nulls.call(L, call, g, 0, mem) == OK                   # n == 0: no pointer is needed
    if mem == MEM_HOST:
        assert Args(mem, streams=(0, S)).call(L, call, g, 2, mem) == E_ARG     # out of range
        assert Args(mem, streams=(-1, 0)).call(L, call, g, 2, mem) == E_ARG
        assert Args(mem, streams=(1, 1)).call(L, call, g, 2, mem) == E_ARG     # listed twice
    _sync()


@pytest.mark.parametrize("mem", [MEM_HOST, MEM_DEVICE])
def test_chain_kind_and_level(native, groups, mem):
    L = native
    enc, dec = groups["chain_enc"].handle, groups["chain_dec"].handle
    a = Args(mem)
    assert a.call(L, "chain_encode", dec, 2, mem) == E_ARG        # a group of the other kind
    assert a.call(L, "chain_decode", enc, 2, mem) == E_ARG
    assert a.call(L, "chain_inject", enc, 2, mem) == E_ARG
    assert a.call(L, "chain_encode", dec, 0, mem) == E_ARG
    for level in (256, -1):
        assert a.call(L, "chain_encode", enc, 2, mem, level=level) == E_ARG
        assert a.call(L, "chain_encode", enc, 0, mem, level=level) == E_ARG
    _sync()


def test_writer_bound_overflow(native, groups):
    """A host-memory write whose bound exceeds 2^31 - 1 is refused before anything is read, at any entry."""
    L = native
    g = groups["writer"].handle
    for lens in ((3, 2**31 - 64), (2**31 - 1, 3)):
        assert Args(MEM_HOST, lens=lens).call(L, "writer_write", g, 2, MEM_HOST) == E_ARG, lens
    assert Args(MEM_HOST, streams=(1, 1), lens=(3, 2**31 - 64)).call(L, "writer_write", g, 2, MEM_HOST) == E_ARG


@pytest.mark.parametrize("mem", [MEM_HOST, MEM_DEVICE])
@pytest.mark.parametrize("kind", list(RESET))
def test_reset_arguments(native, groups, kind, mem):
    L = native
    fn = getattr(L, RESET[kind])
    g = groups[kind].handle
    a = Args(mem)
    assert fn(None, a.ptr["streams"], 2, mem, None) == E_ARG
    assert fn(g, a.ptr["streams"], 2, 5, None) == E_ARG
    assert fn(g, None, 0, 5, None) == E_ARG
    assert fn(g, a.ptr["streams"], -1, mem, None) == E_ARG
    assert fn(g, None, 2, mem, None) == E_ARG
    assert fn(g, None, 0, mem, None) == OK                         # n == 0 with null streams
    twice = Args(mem, streams=(1, 1))                              # kept alive until the reset has run
    assert fn(g, twice.ptr["streams"], 2, mem, None) == OK         # a stream listed twice is fine
    if mem == MEM_HOST:
        assert fn(g, Args(mem, streams=(0, S)).ptr["streams"], 2, mem, None) == E_ARG
        assert fn(g, Args(mem, streams=(-1, 0)).ptr["streams"], 2, mem, None) == E_ARG
    _sync()
