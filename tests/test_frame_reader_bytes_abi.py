"""k4lz4_frame_reader_group_read_bytes without a GPU: its argument errors come in _read's order, the flags check
last (a group exists only on a device, so every call here stops at the null group), and a group cannot be created
without a device."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import has_gpu

E_ARG, E_NODEVICE = -102, -100


def test_read_bytes_without_group(native):
    L = native
    s = np.zeros(4, np.int32)
    o = np.zeros(4, np.int64)
    n = np.zeros(4, np.int32)
    b = np.zeros(16, np.uint8)
    p = [s.ctypes.data, b.ctypes.data, o.ctypes.data, n.ctypes.data, n.ctypes.data, b.ctypes.data, o.ctypes.data,
         n.ctypes.data, n.ctypes.data, n.ctypes.data]
    for mem in (0, 1, 5):
        for flags in (0, 1, 2, -1):
            for count in (1, 0, -1):
                assert L.k4lz4_frame_reader_group_read_bytes(None, *p, count, flags, mem, None) == E_ARG
            assert L.k4lz4_frame_reader_group_read_bytes(None, *([None] * 10), 1, flags, mem, None) == E_ARG


def test_no_device(native):
    if has_gpu():
        pytest.skip("for a machine without a GPU")
    g = C.c_void_p()
    assert native.k4lz4_frame_reader_group_create(4, 65536, 0, C.byref(g)) == E_NODEVICE and g.value is None
    from k4os.compression.lz4_b200 import FrameReaderGroup, _native
    with pytest.raises(_native.K4Error) as e:
        FrameReaderGroup(4)
    assert e.value.code == E_NODEVICE
