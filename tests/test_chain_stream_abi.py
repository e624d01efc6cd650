"""k4lz4_decode_chain_streams: argument errors come first (E_ARG with or without a GPU), then the machine
(E_NODEVICE without a GPU), then an empty call (OK).  No case reaches a device."""
import numpy as np
import pytest

from tests.conftest import has_gpu


def _call(native, n, m, mem, es=None, pre=None, null=False, device=0):
    from k4os.compression.lz4_b200 import _native as N
    keep = [np.zeros(16, dtype=np.int64) for _ in range(8)]
    es = np.ascontiguousarray(es if es is not None else [0] * (max(m, 0) + 1), dtype=np.int32)
    pre = np.ascontiguousarray(pre if pre is not None else [0] * max(m, 1), dtype=np.int32)
    p = (lambda i: None) if null else (lambda i: keep[i].ctypes.data)
    mk = {"host": N.MEM_HOST, "device": N.MEM_DEVICE, "unknown": 7}[mem]
    return native.k4lz4_decode_chain_streams(p(0), p(1), p(2), None, p(3), p(4), n,
                                             None if null else es.ctypes.data, p(5), p(6),
                                             None if null else pre.ctypes.data, m, mk, None, device)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_argument_errors(native, mem):
    from k4os.compression.lz4_b200 import _native as N
    assert _call(native, 1, 1, "unknown", es=[0, 1]) == N.E_ARG
    assert _call(native, -1, 1, mem) == N.E_ARG
    assert _call(native, 1, -1, mem) == N.E_ARG
    assert _call(native, 2, 0, mem) == N.E_ARG                       # entries without a stream
    assert _call(native, 1, 1, mem, null=True) == N.E_ARG


def test_host_stream_table_checks(native):
    """With host memory the stream table is checked: it runs from 0 to the entry count without decreasing, and no
    prefix length is negative."""
    from k4os.compression.lz4_b200 import _native as N
    assert _call(native, 2, 2, "host", es=[1, 1, 2]) == N.E_ARG
    assert _call(native, 2, 2, "host", es=[0, 1, 1]) == N.E_ARG
    assert _call(native, 2, 2, "host", es=[0, 2, 1]) == N.E_ARG
    assert _call(native, 2, 2, "host", es=[0, 1, 2], pre=[0, -1]) == N.E_ARG
    want = N.E_ARG if has_gpu() else N.E_NODEVICE
    ndev = native.k4lz4_device_count()
    assert _call(native, 2, 2, "host", es=[0, 1, 2], pre=[0, 5], device=ndev) == want


def test_empty_call(native):
    from k4os.compression.lz4_b200 import _native as N
    want = N.OK if has_gpu() else N.E_NODEVICE
    assert _call(native, 0, 0, "host", null=True) == want
    assert _call(native, 0, 3, "device") == want
