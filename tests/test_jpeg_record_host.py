"""The recording JPEG decode without a GPU: the host build of the entropy kernel's recording instantiation
(tests/emu/faa_emu_jpeg_record.cpp, the same faa_jpeg.cuh the kernels run).  On every file of the decoder grid, on the
restart-free hand-built streams and on corrupt files, its coefficients, pixels and status equal the decode without
recording; the points it records equal the index decode's (``jpeg_index_record``) byte for byte, and it writes none
outside the file's range.  Restart-interval files, short scans, corrupt files and files whose points were used get a
count of 0."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_index_cases as jic
from helpers import ROOT
from jpeg_cases import GRID, content, encode
from test_jpeg_host import MUTATIONS
from test_jpeg_index_host import FILES, GRID_CHUNKS, STREAMS, _mutated, grid_bytes, header

from fast_autoaugment_b200 import _lib

SYNC = jic.SYNC
GUARD = 64


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_record.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_record.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64 = C.c_void_p, C.c_int64
    lib.faa_emu_jpeg_decode_recording.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, vp, i64, vp, vp, i64]
    return lib


@pytest.fixture(scope="module")
def emu_index():
    return jic.load_emu_index()


def decode(lib, b, pts=None, record=True, cap=None):
    """(status, pixels, coefficients, count, recorded points) of the host build; ``cap``: the room given to the
    recording (default the file's capacity).  Guard bytes around the output, the coefficients and the point range
    must keep their value."""
    src = np.frombuffer(b, np.uint8).copy()
    hw = np.zeros(2, np.int32)
    st = np.zeros(1, np.int32)
    assert lib.faa_emu_jpeg_decode_recording(src.ctypes.data, src.size, None, 0, None, 0, st.ctypes.data,
                                             hw.ctypes.data, None, 0, None, None, 0) == 0
    h = header(b)
    n = int(hw[0]) * int(hw[1]) * 3
    blocks = int(h["mcu_x"]) * int(h["mcu_y"]) * (1 if int(h["ncomp"]) == 1 else int(h["hs"]) * int(h["vs"]) + 2)
    if cap is None:
        cap = _lib.lib.faa_jpeg_index_capacity(h.tobytes())
    out = np.full(n + 2 * GUARD, 0xA5, np.uint8)
    coef = np.full(blocks * 64 + 2 * GUARD, 0x5A5A, np.int16)
    rec = np.full((cap + 2 * GUARD) * 16, 0x3C, np.uint8)
    count = np.full(1, -7, np.int32)
    q = None if pts is None else np.ascontiguousarray(pts, SYNC).reshape(-1)
    assert lib.faa_emu_jpeg_decode_recording(
        src.ctypes.data, src.size, None if q is None or not len(q) else q.ctypes.data, 0 if q is None else len(q),
        out.ctypes.data + GUARD, n, st.ctypes.data, hw.ctypes.data, rec.ctypes.data + GUARD * 16 if record else None,
        cap, count.ctypes.data if record else None, coef.ctypes.data + 2 * GUARD, blocks * 64) == 0
    assert (out[:GUARD] == 0xA5).all() and (out[GUARD + n:] == 0xA5).all()
    assert (coef[:GUARD] == 0x5A5A).all() and (coef[GUARD + blocks * 64:] == 0x5A5A).all()
    assert (rec[:GUARD * 16] == 0x3C).all() and (rec[(GUARD + cap) * 16:] == 0x3C).all()
    c = int(count[0]) if record else 0
    assert 0 <= c <= cap
    pts_out = rec[GUARD * 16:(GUARD + c) * 16].view(SYNC).copy()
    return int(st[0]), out[GUARD:GUARD + n].reshape(int(hw[0]), int(hw[1]), 3), coef[GUARD:GUARD + blocks * 64], c, pts_out


def check_file(lib, emu_index, b, pts=None):
    """the recording decode equals the plain one, and its points jpeg_index_record's; returns (count, status)"""
    st0, px0, coef0, _, _ = decode(lib, b, pts, record=False)
    st, px, coef, n, got = decode(lib, b, pts)
    assert st == st0 and np.array_equal(px, px0) and np.array_equal(coef, coef0)
    want, st_idx, _ = jic.host_index(emu_index, b)
    h = header(b)
    if pts is None:
        if jic.parts(int(h["scan_len"]), int(h["restart"])):
            assert st_idx == st
        assert got.tobytes() == want.tobytes()
    if int(h["restart"]) or jic.parts(int(h["scan_len"]), 0) == 0 or st:
        assert n == 0
    return n, st


@pytest.mark.parametrize("k", range(len(GRID_CHUNKS)), ids=lambda k: GRID_CHUNKS[k][0][0])
def test_grid_recording_equals_plain_and_index_decodes(emu, emu_index, k):
    for case in GRID_CHUNKS[k]:
        b = grid_bytes(case)
        h = header(b)
        n, _ = check_file(emu, emu_index, b)
        assert (n > 0) == (int(h["restart"]) == 0 and int(h["scan_len"]) >= 2048), case[0]


@pytest.mark.parametrize("k", range(0, len(STREAMS), 16), ids=lambda k: STREAMS[k][0])
def test_streams_recording_equals_plain_and_index_decodes(emu, emu_index, k):
    for _, b in STREAMS[k:k + 16]:
        check_file(emu, emu_index, b)


def test_restart_files_short_scans_and_corrupt_files_get_count_0(emu, emu_index):
    a = content("photo", 375, 500, 1)
    for opts in ({"restart_marker_blocks": 4}, {"restart_marker_rows": 1}):
        b = encode(a, quality=90, **opts)
        assert int(header(b)["restart"]) > 0 and int(header(b)["scan_len"]) > 4096
        assert check_file(emu, emu_index, b)[0] == 0
        assert decode(emu, b, cap=64)[3] == 0                  # even when given room
    flat = encode(np.full((64, 64, 3), 100, np.uint8), quality=75)
    assert int(header(flat)["scan_len"]) < 2048
    assert check_file(emu, emu_index, flat)[0] == 0 and decode(emu, flat, cap=8)[3] == 0
    flagged = 0
    cases = [b for _, b, _ in MUTATIONS] + [m for _, good in FILES for _, m in _mutated(good, len(good))]
    for b in cases:
        n, st = check_file(emu, emu_index, b)
        flagged += st != 0
    assert flagged > 10


def test_capacity_exact_and_short(emu, emu_index):
    b = jic.big_file()
    h = header(b)
    cap = _lib.lib.faa_jpeg_index_capacity(h.tobytes())
    assert cap == 127
    full = jic.host_index(emu_index, b)[0]
    _, _, _, n, got = decode(emu, b)                            # exactly at capacity: 127 of 127
    assert n == 127 and got.tobytes() == full.tobytes()
    for c in (1, 3, 126):
        _, _, _, n, got = decode(emu, b, cap=c)
        assert n == c and got.tobytes() == jic.host_index(emu_index, b, cap=c)[0].tobytes()
    assert decode(emu, b, cap=0)[3] == 0


@pytest.mark.parametrize("k", range(len(FILES)), ids=[f[0] for f in FILES])
def test_points_used_give_count_0_and_failed_points_are_recorded_afresh(emu, emu_index, k):
    name, b = FILES[k]
    h = header(b)
    mcus = int(h["mcu_x"]) * int(h["mcu_y"])
    pts, _, scan = jic.host_index(emu_index, b)
    st0, px0, coef0, _, _ = decode(emu, b, record=False)
    st, px, coef, n, _ = decode(emu, b, pts)                   # the file's own points: used, nothing recorded
    assert (st, n) == (st0, 0) and np.array_equal(px, px0) and np.array_equal(coef, coef0)
    other = jic.host_index(emu_index, FILES[(k + 1) % len(FILES)][1])[0]
    for what, q in jic.fuzzed(pts, other, scan, mcus, b, jic.host_states(emu_index, b, mcus)):
        st, px, coef, n, got = decode(emu, b, q)
        assert st == st0 and np.array_equal(px, px0) and np.array_equal(coef, coef0), (name, what)
        if jic.linked(emu_index, b, q) == 1:
            assert n == 0, (name, what)
        else:
            assert got.tobytes() == pts.tobytes(), (name, what)
