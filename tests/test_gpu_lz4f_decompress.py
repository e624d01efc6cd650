"""k4lz4_lz4f_decompress_batch and k4lz4_lz4f_decompressed_size_batch against the model of `lz4 -d`
(tests/lz4f_dec_ref.py), on the whole grid in a few large calls, in host and device memory: content, result, error
and end of every stream, with the bytes around every destination untouched."""
from __future__ import annotations

import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not oracle.have_ref(), reason="needs oracle/_ref")]

GAP = 64


@pytest.fixture(scope="module")
def expected():
    from tests import lz4f_dec_ref as M
    model = M.CliModel()
    cases = M.grid()
    return cases, [model.run(data, d) for _, data, d in cases]


def code_of(e, c):
    return (e << 8) | c if e else 0


def device_call(streams, dictionaries, caps):
    """k4lz4_lz4f_decompress_batch on device memory, destinations GAP bytes apart in a 0xCD buffer; -> (contents,
    out, err, end, whole buffer, offsets)."""
    import torch
    from k4os.compression.lz4_b200 import LZ4F
    dev = torch.device("cuda", 0)
    lens = [len(s) for s in streams]
    so = np.zeros(len(streams), dtype=np.int64)
    so[1:] = np.cumsum(lens[:-1])
    src = torch.from_numpy(np.frombuffer(b"".join(streams) + b"\0", dtype=np.uint8).copy()).to(dev)
    caps = np.asarray(caps, dtype=np.int64)
    do = np.zeros(len(streams), dtype=np.int64)
    do[1:] = np.cumsum(np.maximum(caps[:-1], 0) + GAP)
    do += GAP
    dst = torch.full((int(do[-1] + max(caps[-1], 0) + GAP),), 0xCD, dtype=torch.uint8, device=dev)
    t = lambda a, ty: torch.from_numpy(np.asarray(a, dtype=ty)).to(dev)               # noqa: E731
    args = dict()
    if dictionaries is not None:
        dl = [len(d) for d in dictionaries]
        dof = np.zeros(len(dl), dtype=np.int64)
        dof[1:] = np.cumsum(dl[:-1])
        args = dict(dict_base=torch.from_numpy(np.frombuffer(b"".join(dictionaries) + b"\0", dtype=np.uint8).copy())
                    .to(dev), dict_off=t(dof, np.int64), dict_len=t(dl, np.int32))
    out, err, end = (torch.zeros(len(streams), dtype=torch.int32, device=dev) for _ in range(3))
    LZ4F.decompress_many_device(src, t(so, np.int64), t(lens, np.int32), dst, t(do, np.int64),
                                t(caps, np.int32), out, err, end,
                                stream=torch.cuda.current_stream().cuda_stream, **args)
    torch.cuda.synchronize()
    o, e, n, buf = out.cpu().numpy(), err.cpu().numpy(), end.cpu().numpy(), dst.cpu().numpy()
    contents = [buf[do[i]:do[i] + o[i]].tobytes() if o[i] > 0 else b"" for i in range(len(o))]
    return contents, o, e, n, buf, do


def check(cases, want, got_out, got_err, got_end, contents, caps=None, full=None):
    """caps: the destinations, when some are below `full` (caps_of): a stream that does not fit gets
    K4LZ4_R_DST_SMALL, or an error found without decoding."""
    bad = []
    for i, ((name, data, _), (content, e, c, end)) in enumerate(zip(cases, want)):
        small = caps is not None and int(caps[i]) < int(full[i]) - 100
        if small:
            ok = (int(got_out[i]) == -1001 and int(got_err[i]) == 0) or (e != 0 and int(got_out[i]) == -1 and
                                                                           int(got_err[i]) != 0)
        elif e == 0:
            ok = int(got_out[i]) == len(content) and contents[i] == content and int(got_err[i]) == 0
        else:
            ok = int(got_out[i]) == -1 and int(got_err[i]) == code_of(e, c)
        ok = ok and int(got_end[i]) == end
        if not ok:
            bad.append(f"{name}: got ({int(got_out[i])}, {int(got_err[i]):#x}, {int(got_end[i])}), "
                       f"model ({len(content) if e == 0 else -1}, {code_of(e, c):#x}, {end})")
    assert not bad, "\n".join(bad[:40])


def caps_of(want, streams):
    """Room for every stream: its content, or where the model fails, the size call's length (a failed stream's
    partial output is no bound)."""
    from k4os.compression.lz4_b200 import LZ4F
    sizes = LZ4F.decompressed_sizes(streams)[0]
    return [(len(content) if e == 0 else max(int(s), 0)) + 100 for (content, e, *_), s in zip(want, sizes)]


def test_grid_host(expected):
    from k4os.compression.lz4_b200 import LZ4F
    cases, want = expected
    streams = [data for _, data, _ in cases]
    dicts = [d if d is not None else b"" for _, _, d in cases]
    has = [d is not None for _, _, d in cases]
    idx = [i for i in range(len(cases)) if has[i]]
    nodict = [i for i in range(len(cases)) if not has[i]]
    for sel, with_dict in ((nodict, False), (idx, True)):
        c = [cases[i] for i in sel]
        w = [want[i] for i in sel]
        sub = [streams[i] for i in sel]
        contents, out, err, end = LZ4F.decompress_many(sub, [dicts[i] for i in sel] if with_dict else None,
                                                       caps_of(w, sub))
        check(c, w, out, err, end, contents)


def test_grid_device_canaries(expected):
    cases, want = expected
    streams = [data for _, data, _ in cases]
    dicts = [d if d is not None else b"" for _, _, d in cases]
    caps = caps_of(want, streams)
    contents, out, err, end, buf, do = device_call(streams, dicts, caps)
    # an empty dictionary is no dictionary: the whole grid in one call
    check(cases, want, out, err, end, contents)
    for i in range(len(cases)):
        assert (buf[do[i] - GAP:do[i]] == 0xCD).all(), cases[i][0]
        assert (buf[do[i] + caps[i]:do[i] + caps[i] + GAP] == 0xCD).all(), cases[i][0]


def test_sizes_agree(expected):
    from k4os.compression.lz4_b200 import LZ4F
    cases, want = expected
    size, serr, send = LZ4F.decompressed_sizes([data for _, data, _ in cases])
    for i, ((name, data, _), (content, e, c, end)) in enumerate(zip(cases, want)):
        assert int(send[i]) == end, name
        if e == 0:
            assert int(size[i]) == len(content) and int(serr[i]) == 0, name
        elif int(serr[i]):                 # an error found without decoding: decompress fails too
            assert int(size[i]) == -1, name


def test_small_destinations(expected):
    cases, want = expected
    streams = [data for _, data, _ in cases]
    dicts = [d if d is not None else b"" for _, _, d in cases]
    rng = np.random.default_rng(3)
    full = caps_of(want, streams)
    caps = [int(rng.integers(0, c + 1)) for c in full]
    contents, out, err, end, buf, do = device_call(streams, dicts, caps)
    check(cases, want, out, err, end, contents, caps, full)
    for i in range(len(cases)):
        assert (buf[do[i] + caps[i]:do[i] + caps[i] + GAP] == 0xCD).all(), cases[i][0]


def test_cli_spot_check(expected):
    """A sample straight against upstream's CLI binary."""
    from k4os.compression.lz4_b200 import LZ4F
    cli = os.path.join(os.path.dirname(oracle.REF_SO), "lz4")
    if not os.path.exists(cli):
        pytest.skip("no oracle/_ref/lz4")
    cases, want = expected
    pick = [i for i in range(len(cases)) if i % 9 == 0 and cases[i][2] is None]
    sample = [cases[i] for i in pick]
    contents, out, err, _ = LZ4F.decompress_many([d for _, d, _ in sample], None,
                                                 caps_of([want[i] for i in pick], [d for _, d, _ in sample]))
    for i, (name, data, _) in enumerate(sample):
        with tempfile.NamedTemporaryFile(suffix=".lz4") as f:   # a file, not a pipe: the CLI seeks past skippables
            f.write(data)
            f.flush()
            r = subprocess.run([cli, "-d", "-c", f.name], capture_output=True)
        assert r.returncode == int(err[i]) >> 8, name
        if r.returncode == 0:
            assert r.stdout == contents[i], name


def test_mixed_legacy_and_small_frames():
    """One legacy stream with 8 MiB blocks beside thousands of small-frame streams: scratch slots are sized by each
    member's own capacity, so the call fits easily."""
    from k4os.compression.lz4_b200 import LZ4F
    from tests import lz4f_dec_ref as M, lz4f_ref as LR
    up = LR.Lz4fUpstream()
    big = LR.content("text", 3 * M.LEGACY_BLOCK, 0) + LR.content("text", 5000, 1)
    leg = M.legacy(up, big)
    small = [up.frame(LR.content("text", 300 + i % 700, i), 1 << 16, LR.flags_of(False, True, True, True))
             for i in range(6000)]
    contents, out, err, end = LZ4F.decompress_many([leg] + small)
    assert int(err.max()) == 0 and int(out[0]) == len(big) and contents[0] == big
    for i in range(0, 6000, 97):
        assert contents[1 + i] == LR.content("text", 300 + i % 700, i)


def test_linked_steps_per_member():
    """1 000 streams of 50 concatenated frames: the linked steps run over members, so their count is the largest block
    count of one member, not of one stream."""
    import torch
    from k4os.compression.lz4_b200 import _native as N
    from tests import lz4f_ref as LR
    up = LR.Lz4fUpstream()
    frames = [up.frame(LR.content("text", 65536 * 3 + 11 * i, i), 1 << 16, LR.flags_of(True, False, i % 2 == 0, False))
              for i in range(50)]
    one = b"".join(frames)
    want = b"".join(LR.content("text", 65536 * 3 + 11 * i, i) for i in range(50))
    streams = [one] * 1000
    caps = [len(want)] * 1000
    before = int(N.lib().k4lz4_launch_count())
    contents, out, err, end, _, _ = device_call(streams, None, caps)
    launches = int(N.lib().k4lz4_launch_count()) - before
    assert int(err.max()) == 0 and all(c == want for c in contents[::111])
    # 4 blocks per member at most: a step is prepare + copy + chain + commit + copy (at most 5 launches each);
    # a stream-wide walk would need 200 steps
    assert launches < 150, launches
    torch.cuda.synchronize()


def test_round_trips():
    """A 4 MiB-block frame from k4lz4_lz4f_compress_batch, and dictionary frames from k4lz4_frame_encode_dict_batch."""
    from k4os.compression.lz4_b200 import LZ4F, LZ4Frame
    from tests import lz4f_ref as LR
    data = LR.content("text", (4 << 20) * 2 + 12345, 9)
    frames, res = LZ4F.compress_many([data, data[:5000]], 1 << 22, True, True, True, True)
    assert (res > 0).all()
    contents, out, err, _ = LZ4F.decompress_many([frames[0], frames[1] + frames[0]])
    assert int(err.max()) == 0 and contents[0] == data and contents[1] == data[:5000] + data
    dic = LR.content("text", 50000, 77)
    body = LR.content("text", 200000, 3) + dic[1000:30000]
    for linked in (True, False):
        fr, r = LZ4Frame.EncodeManyWithDictionary([body], [dic], [9], 1 << 16, linked, True, True)
        assert int(r[0]) > 0
        contents, out, err, _ = LZ4F.decompress_many([fr[0] + fr[0]], [dic])
        assert int(err[0]) == 0 and contents[0] == body + body
