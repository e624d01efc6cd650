"""The k4lz4_frame_reader_group_* exports without a GPU: argument errors in the documented order, maxBlockSize
validation and K4LZ4_E_NODEVICE."""
import ctypes as C

import numpy as np
import pytest

from tests.conftest import has_gpu

E_ARG, E_NODEVICE = -102, -100


def test_create_arguments(native):
    L = native
    g = C.c_void_p()
    for args in ((0, 65536), (-1, 65536), (4, 0), (4, 65535), (4, 65537), (4, 100000), (4, 1 << 17), (4, 8 << 20)):
        assert L.k4lz4_frame_reader_group_create(*args, 0, C.byref(g)) == E_ARG, args
        assert g.value is None
    assert L.k4lz4_frame_reader_group_create(4, 65536, 0, None) == E_ARG
    if has_gpu():
        pytest.skip("the rest is for a machine without a GPU")
    for mb in (1 << 16, 1 << 18, 1 << 20, 1 << 22):
        assert L.k4lz4_frame_reader_group_create(4, mb, 0, C.byref(g)) == E_NODEVICE and g.value is None


def test_calls_without_group(native):
    L = native
    s = np.zeros(4, np.int32)
    o = np.zeros(4, np.int64)
    n = np.zeros(4, np.int32)
    b = np.zeros(16, np.uint8)
    p = [s.ctypes.data, b.ctypes.data, o.ctypes.data, n.ctypes.data, n.ctypes.data, b.ctypes.data, o.ctypes.data,
         n.ctypes.data, n.ctypes.data, n.ctypes.data]
    for mem in (0, 1, 5):
        assert L.k4lz4_frame_reader_group_read(None, *p, 1, mem, None) == E_ARG
        assert L.k4lz4_frame_reader_group_end(None, s.ctypes.data, n.ctypes.data, 1, mem, None) == E_ARG
        assert L.k4lz4_frame_reader_group_reset(None, s.ctypes.data, 1, mem, None) == E_ARG
    assert L.k4lz4_frame_reader_group_destroy(None) == 0


def test_python_mirror_arguments(native):
    from k4os.compression.lz4_b200 import FrameReaderGroup, _native
    with pytest.raises(_native.K4Error) as e:
        FrameReaderGroup(4, 100000)
    assert e.value.code == E_ARG
    if not has_gpu():
        with pytest.raises(_native.K4Error) as e:
            FrameReaderGroup(4)
        assert e.value.code == E_NODEVICE
