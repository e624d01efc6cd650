"""The C-ABI shared library: loads, exports every symbol include/k4lz4.h declares, and its
non-compute entry points behave.  CPU only -- no compute call is made without a GPU."""
import ctypes
import os
import re

import numpy as np

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
