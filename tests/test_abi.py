"""The C-ABI shared library: loads, exports every symbol include/k4lz4.h declares, and its
non-compute entry points behave.  CPU only -- no compute call is made without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

from tests.conftest import ROOT, has_gpu


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "k4lz4.h")).read()
    return sorted(set(re.findall(r"K4LZ4_API\s+[\w\s\*]+?\b(k4lz4_\w+)\s*\(", text)))


def test_header_symbols_all_exported(native):
    from k4os.compression.lz4_b200 import _native
    decl = _declared_symbols()
    assert len(decl) >= 15
    assert sorted(_native.SYMBOLS) == decl
    raw = ctypes.CDLL(_native.SO_PATH)
    for s in decl:
        assert hasattr(raw, s), s


def test_information_entry_points(native):
    assert native.k4lz4_codec_version() == 192          # LZ4Codec.cs:13
    assert native.k4lz4_device_count() >= 0
    assert native.k4lz4_max_output_size(65536) == 65809
    assert native.k4lz4_max_output_size(0) == 16
    assert native.k4lz4_max_output_size(0x7E000001) == 0
    assert native.k4lz4_pickle_bound(0) == 0 and native.k4lz4_pickle_bound(100) == 101


def test_no_device_fails_loudly(native):
    """Without a GPU the product refuses to run: no silent CPU fallback."""
    if has_gpu():
        return
    from k4os.compression.lz4_b200 import LZ4Codec, _native
    import pytest
    with pytest.raises(_native.K4Error) as e:
        LZ4Codec.Encode(b"some bytes some bytes some bytes", bytearray(100))
    assert e.value.code == _native.E_NODEVICE
    # reference semantics that need no device still hold
    assert LZ4Codec.Encode(b"", bytearray(10)) == 0
    assert LZ4Codec.Decode(b"", bytearray(10)) == 0


def test_synth_host_is_deterministic(native):
    from k4os.compression.lz4_b200.batch import synth_host
    a = synth_host(3, 4096, 525, seed=9)
    b = synth_host(3, 4096, 525, seed=9)
    c = synth_host(1, 4096, 525, seed=9, first_block=2)
    assert np.array_equal(a, b) and np.array_equal(a[8192:], c)
    assert not np.array_equal(a[:4096], a[4096:8192])


def test_library_holds_sm90a_code_only(native):
    """The shipped library is Hopper code: an sm_90a cubin, no other architecture."""
    import subprocess
    from k4os.compression.lz4_b200 import _native, build
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    out = subprocess.run([cuobjdump, "--list-elf", _native.SO_PATH], capture_output=True, text=True, check=True).stdout
    archs = set(re.findall(r"\.(sm_\w+)\.cubin", out))
    assert archs == {"sm_90a"}, out
    assert "arch=compute_90a,code=sm_90a" in build.NVCC_FLAGS


def test_product_never_imports_oracle():
    """The product package must not reference oracle/ (checked textually over its sources)."""
    pkg = os.path.join(ROOT, "k4os")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dp, f), errors="replace").read()
                assert "import oracle" not in text and "from oracle" not in text, f
                assert "k4lz4_oracle" not in text and "libk4ref" not in text, f


def test_cpp_mirror_header_compiles_and_links(native, tmp_path):
    """include/k4lz4.hpp (the compiled-language host mirror of LZ4Codec / LZ4Pickler) builds against
    the C ABI with a plain host compiler and resolves against libk4lz4.so."""
    import shutil
    import subprocess
    from k4os.compression.lz4_b200 import _native
    gxx = shutil.which("g++")
    if gxx is None:
        import pytest
        pytest.skip("no g++")
    src = tmp_path / "t.cpp"
    src.write_text(
        '#include "k4lz4.hpp"\n'
        'int main() {\n'
        '  using namespace k4lz4;\n'
        '  if (LZ4Codec::MaximumOutputSize(65536) != 65809) return 1;\n'
        '  if (LZ4Codec::Version != 192) return 2;\n'
        '  unsigned char b[4] = {0};\n'
        '  if (LZ4Codec::Encode(b, 0, b, 4) != 0) return 3;          // empty input -> 0, no device needed\n'
        '  if (LZ4Codec::Decode(b, 0, b, 4) != 0) return 4;\n'
        '  if (!LZ4Pickler::Pickle(b, 0).empty()) return 5;\n'
        '  return (int)LZ4Level::L12_MAX == 12 ? 0 : 6;\n'
        '}\n')
    exe = tmp_path / "t"
    libdir = os.path.dirname(_native.SO_PATH)
    subprocess.run([gxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-L", libdir, "-lk4lz4",
                    f"-Wl,-rpath,{libdir}", "-o", str(exe)], check=True, capture_output=True)
    assert subprocess.run([str(exe)]).returncode == 0


# Every batched export, called with its pointer arguments all null (`ptrs(None)`) or all pointing at
# zeroed host arrays (empty blocks, zero capacities and prefixes).
def _export_calls(L):
    return {
        "encode_batch": lambda p, n, mk, d: L.k4lz4_encode_batch(*p(7), n, 0, mk, None, d),
        "encode_batch_x32": lambda p, n, mk, d: L.k4lz4_encode_batch_x32(*p(7), n, 0, mk, None, d),
        "decode_batch": lambda p, n, mk, d: L.k4lz4_decode_batch(*p(7), n, mk, None, d),
        "pickle_batch": lambda p, n, mk, d: L.k4lz4_pickle_batch(*p(6), n, 0, mk, None, d),
        "pickle_writer_batch": lambda p, n, mk, d: L.k4lz4_pickle_writer_batch(*p(6), n, 0, mk, None, d),
        "unpickle_batch": lambda p, n, mk, d: L.k4lz4_unpickle_batch(*p(7), n, mk, None, d),
        "unpickled_size_batch": lambda p, n, mk, d: L.k4lz4_unpickled_size_batch(*p(4), n, mk, None, d),
        "decode_dict_batch": lambda p, n, mk, d: L.k4lz4_decode_dict_batch(*p(10), n, mk, None, d),
        "partial_decode_batch": lambda p, n, mk, d: L.k4lz4_partial_decode_batch(*p(7), n, mk, None, d),
        "decode_chain_batch": lambda p, n, mk, d: L.k4lz4_decode_chain_batch(*p(8), n, mk, None, d),
        "xxh32_batch": lambda p, n, mk, d: L.k4lz4_xxh32_batch(*p(3), 0, *p(1), n, mk, None, d),
    }


_EXPORTS = sorted(_export_calls(None))


@pytest.mark.parametrize("case", ["negative_count", "null_pointer", "empty_nulls", "device_out_of_range"])
@pytest.mark.parametrize("mem", ["host", "device", "unknown"])
@pytest.mark.parametrize("export", _EXPORTS)
def test_argument_error_matrix(native, export, mem, case):
    """One check for every batched export: argument errors first (E_ARG with or without a GPU), then the
    machine (E_NODEVICE without a GPU), then an empty batch (OK), then the device index.  No row reaches a
    device: the pointers are null or zeroed host arrays that are rejected before any copy or launch."""
    from k4os.compression.lz4_b200 import _native as N
    keep = [np.zeros(16, dtype=np.int64) for _ in range(10)]
    real = lambda k: [a.ctypes.data for a in keep[:k]]
    null = lambda k: [None] * k
    mk = {"host": N.MEM_HOST, "device": N.MEM_DEVICE, "unknown": 7}[mem]
    ndev = native.k4lz4_device_count()
    ptrs, n, dev = {"negative_count": (null, -1, 0), "null_pointer": (null, 1, 0), "empty_nulls": (null, 0, 0),
                    "device_out_of_range": (real, 1, ndev)}[case]
    rc = _export_calls(native)[export](ptrs, n, mk, dev)
    if mem == "unknown" or case in ("negative_count", "null_pointer"):
        want = N.E_ARG
    elif not has_gpu():
        want = N.E_NODEVICE
    else:
        want = N.OK if case == "empty_nulls" else N.E_ARG
    assert rc == want, (export, mem, case, rc, native.k4lz4_last_error())


def test_device_only_calls_check_arguments_first(native):
    """synth_device, copy_blocks_device and the two stats calls: argument errors are E_ARG with or without a
    GPU; a device index out of range is E_ARG on a GPU."""
    from k4os.compression.lz4_b200 import _native as N
    assert native.k4lz4_synth_device(None, 1, 4096, 500, 1, 0, None, 0) == N.E_ARG
    assert native.k4lz4_synth_device(None, -1, 4096, 500, 1, 0, None, 0) == N.E_ARG
    assert native.k4lz4_copy_blocks_device(None, None, None, None, None, 1, None, 0) == N.E_ARG
    assert native.k4lz4_copy_blocks_device(None, None, None, None, None, -1, None, 0) == N.E_ARG
    assert native.k4lz4_decode_stats(0, None, 0) == N.E_ARG
    assert native.k4lz4_encode_stats(0, None, 0) == N.E_ARG
    keep = np.zeros(16, dtype=np.int64)
    p, ndev = keep.ctypes.data, native.k4lz4_device_count()
    want = N.E_ARG if has_gpu() else N.E_NODEVICE
    assert native.k4lz4_synth_device(p, 1, 4096, 500, 1, 0, None, ndev) == want
    assert native.k4lz4_copy_blocks_device(p, p, p, p, p, 1, None, ndev) == want
    assert native.k4lz4_decode_stats(ndev, p, 0) == want
    assert native.k4lz4_encode_stats(ndev, p, 0) == want
