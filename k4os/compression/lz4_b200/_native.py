"""ctypes binding of libk4lz4.so (include/k4lz4.h).  Fails loudly: there is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libk4lz4.so")

OK = 0
E_NODEVICE, E_CUDA, E_ARG, E_NOMEM = -100, -101, -102, -103
R_DELEGATE = -2
R_CORRUPT = -1000
R_DST_SMALL = -1001                       # K4LZ4_R_DST_SMALL (frame decode)
FRAME_INDEPENDENT, FRAME_BLOCK_CHECKSUM, FRAME_CONTENT_CHECKSUM = 1, 2, 4
MEM_HOST, MEM_DEVICE = 0, 1
ALL_DEVICES = -1
CHAIN_STATE_BYTES = 16400                 # K4LZ4_CHAIN_STATE_BYTES
CHAIN_ENCODER, CHAIN_DECODER = 0, 1       # K4LZ4_CHAIN_ENCODER / K4LZ4_CHAIN_DECODER
READ_INTERACTIVE = 1                      # K4LZ4_READ_INTERACTIVE

_vp, _i32, _i64, _u32, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64
_BATCH = [_vp] * 7                        # srcBase srcOff srcLen dstBase dstOff dstCap outLen
_CALL = [_i32, _vp, _i32]                 # memKind cudaStream device

# {symbol: (argtypes, restype)} for every symbol include/k4lz4.h declares (tests/test_abi.py checks the .so
# exports them all)
SIGNATURES = {
    "k4lz4_codec_version": ([], _i32),
    "k4lz4_device_count": ([], _i32),
    "k4lz4_last_error": ([], C.c_char_p),
    "k4lz4_launch_count": ([], _i64),
    "k4lz4_max_output_size": ([_i32], _i32),
    "k4lz4_pickle_bound": ([_i32], _i32),
    "k4lz4_pickle_writer_bound": ([_i32], _i32),
    "k4lz4_encode": ([_vp, _i32, _vp, _i32, _i32], _i32),
    "k4lz4_encode_x32": ([_vp, _i32, _vp, _i32, _i32], _i32),
    "k4lz4_decode": ([_vp, _i32, _vp, _i32], _i32),
    "k4lz4_decode_dict": ([_vp, _i32, _vp, _i32, _vp, _i32], _i32),
    "k4lz4_partial_decode": ([_vp, _i32, _vp, _i32], _i32),
    "k4lz4_encode_batch": (_BATCH + [_i32, _i32] + _CALL, _i32),
    "k4lz4_encode_batch_x32": (_BATCH + [_i32, _i32] + _CALL, _i32),
    "k4lz4_decode_batch": (_BATCH + [_i32] + _CALL, _i32),
    "k4lz4_decoded_size_batch": ([_vp] * 4 + [_i32] + _CALL, _i32),
    "k4lz4_partial_decode_batch": (_BATCH + [_i32] + _CALL, _i32),
    "k4lz4_decode_dict_batch": (_BATCH[:6] + [_vp] * 3 + [_vp, _i32] + _CALL, _i32),
    "k4lz4_decode_chain_batch": (_BATCH[:6] + [_vp, _vp, _i32] + _CALL, _i32),
    "k4lz4_encode_chain_batch": ([_vp] * 10 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_encode_chain_batch_x32": ([_vp] * 10 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_unpickle_batch": (_BATCH + [_i32] + _CALL, _i32),
    "k4lz4_pickle_batch": ([_vp] * 6 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_pickle_batch_x32": ([_vp] * 6 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_pickle_writer_batch": ([_vp] * 6 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_pickle_writer_batch_x32": ([_vp] * 6 + [_i32, _i32] + _CALL, _i32),
    "k4lz4_unpickled_size_batch": ([_vp] * 4 + [_i32] + _CALL, _i32),
    "k4lz4_xxh32": ([_vp, _i64, _u32], _u32),
    "k4lz4_xxh32_batch": ([_vp, _vp, _vp, _u32, _vp, _i32] + _CALL, _i32),
    "k4lz4_synth_host": ([_vp, _i64, _i32, _i32, _u64, _i64], _i32),
    "k4lz4_synth_device": ([_vp, _i64, _i32, _i32, _u64, _i64, _vp, _i32], _i32),
    "k4lz4_copy_blocks_device": ([_vp] * 5 + [_i32, _vp, _i32], _i32),
    "k4lz4_decode_stats": ([_i32, _vp, _i32], _i32),
    "k4lz4_encode_stats": ([_i32, _vp, _i32], _i32),
    "k4lz4_chain_group_create": ([_i32, _i32, _i32, _i32, _vp], _i32),
    "k4lz4_chain_group_destroy": ([_vp], _i32),
    "k4lz4_chain_group_reset": ([_vp, _vp, _i32, _i32, _vp], _i32),
    "k4lz4_chain_group_encode": ([_vp] * 9 + [_i32, _i32, _i32, _vp], _i32),
    "k4lz4_chain_group_encode_x32": ([_vp] * 9 + [_i32, _i32, _i32, _vp], _i32),
    "k4lz4_chain_group_decode": ([_vp] * 9 + [_i32, _i32, _vp], _i32),
    "k4lz4_chain_group_inject": ([_vp] * 5 + [_i32, _i32, _vp], _i32),
    "k4lz4_chain_group_state": ([_vp, _i32, _vp], _i32),
    "k4lz4_chain_group_history": ([_vp, _i32, _vp, _i32], _i32),
    "k4lz4_frame_bound": ([_i64, _i32, _i32], _i64),
    "k4lz4_frame_encode_batch": (_BATCH + [_i32, _i32, _i32, _i32] + _CALL, _i32),
    "k4lz4_frame_encode_batch_x32": (_BATCH + [_i32, _i32, _i32, _i32] + _CALL, _i32),
    "k4lz4_frame_content_size_batch": ([_vp] * 4 + [_i32] + _CALL, _i32),
    "k4lz4_frame_decode_batch": (_BATCH + [_i32] + _CALL, _i32),
    "k4lz4_frame_writer_group_create": ([_i32, _i32, _i32, _i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_group_destroy": ([_vp], _i32),
    "k4lz4_frame_writer_group_reset": ([_vp, _vp, _i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_group_write": ([_vp] * 9 + [_i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_group_write_x32": ([_vp] * 9 + [_i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_group_close": ([_vp] * 6 + [_i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_group_close_x32": ([_vp] * 6 + [_i32, _i32, _vp], _i32),
    "k4lz4_frame_writer_bound": ([_vp, _i64], _i64),
    "k4lz4_frame_writer_close_bound": ([_vp], _i64),
    "k4lz4_frame_reader_group_create": ([_i32, _i32, _i32, _vp], _i32),
    "k4lz4_frame_reader_group_destroy": ([_vp], _i32),
    "k4lz4_frame_reader_group_reset": ([_vp, _vp, _i32, _i32, _vp], _i32),
    "k4lz4_frame_reader_group_read": ([_vp] * 11 + [_i32, _i32, _vp], _i32),
    "k4lz4_frame_reader_group_read_bytes": ([_vp] * 11 + [_i32, _i32, _i32, _vp], _i32),
    "k4lz4_frame_reader_group_end": ([_vp] * 3 + [_i32, _i32, _vp], _i32),
}
SYMBOLS = list(SIGNATURES)


class NativeLibraryMissing(RuntimeError):
    pass


class K4Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libk4lz4 error {code}: {msg}")
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise NativeLibraryMissing(
            f"{SO_PATH} not found: build it with `python -m k4os.compression.lz4_b200.build` "
            "(or __graft_entry__.build()). There is no CPU fallback by design.")
    L = C.CDLL(SO_PATH)
    for name, (args, res) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = args, res
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != OK:
        raise K4Error(rc, lib().k4lz4_last_error().decode("utf-8", "replace"))
