"""The model of `lz4 -d` (tests/lz4f_dec_ref.py) against upstream's CLI itself (oracle/_ref/lz4) on every grid case:
exit code, the LZ4F error name, the output, and where reading stopped.  Then the grid's coverage: every CLI error
number and every LZ4F code the reader can raise, both names of a failed block among them."""
from __future__ import annotations

import os
import re
import subprocess
import tempfile

import pytest

import oracle

CLI = os.path.join(os.path.dirname(oracle.REF_SO), "lz4")
pytestmark = pytest.mark.skipif(not (oracle.have_ref() and os.path.exists(CLI)), reason="needs oracle/_ref")

NAMES = {1: "ERROR_GENERIC", 2: "ERROR_maxBlockSize_invalid", 6: "ERROR_headerVersion_wrong",
         7: "ERROR_blockChecksum_invalid", 8: "ERROR_reservedFlag_set", 14: "ERROR_frameSize_wrong",
         16: "ERROR_decompressionFailed", 17: "ERROR_headerChecksum_invalid", 18: "ERROR_contentChecksum_invalid"}


def cli(data: bytes, dictionary: bytes | None, tmp: str):
    """-> (exit code, stdout, stderr) of `lz4 -d -c -v [-D dict] input`."""
    src = os.path.join(tmp, "in.lz4")
    with open(src, "wb") as f:
        f.write(data)
    cmd = [CLI, "-d", "-c", "-v"]
    if dictionary is not None:
        dp = os.path.join(tmp, "dict")
        with open(dp, "wb") as f:
            f.write(dictionary)
        cmd += ["-D", dp]
    r = subprocess.run(cmd + [src], capture_output=True)
    return r.returncode, r.stdout, r.stderr.decode("latin-1")


@pytest.fixture(scope="module")
def results():
    from tests import lz4f_dec_ref as M
    model = M.CliModel()
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        for name, data, d in M.grid():
            out.append((name, data, d, model.run(data, d), cli(data, d, tmp)))
    return out


def test_model_matches_cli(results):
    bad = []
    for name, data, d, (content, e, code, end), (rc, stdout, stderr) in results:
        if rc != e:
            bad.append(f"{name}: exit {rc}, model {e}")
            continue
        if e == 66 and NAMES[code] not in stderr:
            bad.append(f"{name}: model {NAMES[code]}, cli {stderr.strip()[-120:]}")
        if e == 0:
            if stdout != content:
                bad.append(f"{name}: output differs ({len(stdout)} vs {len(content)} bytes)")
            m = re.search(r"undecodable data at position (\d+)", stderr)
            want = None if end == len(data) else end + 4
            if (int(m.group(1)) if m else None) != want:
                bad.append(f"{name}: trailing position {m.group(1) if m else None}, model end {end}")
    assert not bad, "\n".join(bad[:40])


def test_grid_coverage(results):
    from tests import lz4f_dec_ref as M
    errors = {e for *_, (_, e, _, _), _ in results}
    codes = {c for *_, (_, e, c, _), _ in results if e == 66}
    assert M.CLI_ERRORS <= errors, M.CLI_ERRORS - errors
    assert M.LZ4F_ERRORS <= codes, M.LZ4F_ERRORS - codes
    assert any(e == 0 and end < len(data) for _, data, _, (_, e, _, end), _ in results)
    names = {n for n, *_ in results}
    assert {"mut/indep-decodes-to-max+1", "cat/legacy+legacy+frame", "legacy/full", "skip/past-end"} <= names
