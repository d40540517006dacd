"""The progressive JPEG decoder without a GPU: the host build (tests/emu/faa_emu_jpeg_progressive.cpp, the same
faa_jpeg.cuh the progressive kernel runs) on Pillow-written progressive files.  Pixels equal Pillow's byte for byte,
and the coefficients equal the baseline decoder's on the same image saved baseline with the same options (libjpeg
quantises the same way in both modes).  Waves equal a brute-force dependency model, refusals come with their reasons,
corrupt streams never write outside their buffers, and the Python parse takes progressive files only when asked."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_progressive_cases as jp
from helpers import ROOT

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.engine import EncodedImages, parse_jpeg_headers


@pytest.fixture(scope="module")
def emu():
    return jp.load_emu()


@pytest.fixture(scope="module")
def emu_baseline():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_record.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_record.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64 = C.c_void_p, C.c_int64
    lib.faa_emu_jpeg_decode_recording.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp, vp, i64, vp, vp, i64]
    return lib


def baseline_coefs(lib, b, blocks):
    src = np.frombuffer(b, np.uint8).copy()
    hw = np.zeros(2, np.int32)
    st = np.zeros(1, np.int32)
    assert lib.faa_emu_jpeg_decode_recording(src.ctypes.data, src.size, None, 0, None, 0, st.ctypes.data,
                                             hw.ctypes.data, None, 0, None, None, 0) == 0
    out = np.zeros(int(hw[0]) * int(hw[1]) * 3, np.uint8)
    coef = np.zeros(blocks * 64, np.int16)
    assert lib.faa_emu_jpeg_decode_recording(src.ctypes.data, src.size, None, 0, out.ctypes.data, out.size,
                                             st.ctypes.data, hw.ctypes.data, None, 0, None, coef.ctypes.data,
                                             coef.size) == 0
    assert st[0] == 0
    return coef.reshape(-1, 64)


@pytest.mark.parametrize("entry", jp.GRID, ids=[e[0] for e in jp.GRID])
def test_grid_matches_pillow_and_baseline_coefficients(emu, emu_baseline, entry):
    b = jp.grid_files(entry)
    st, px, coef = jp.decode(emu, b)
    assert st == 0
    assert np.array_equal(px, jp.pillow(b))
    # blocks that only an interleaved DC scan reaches hold no AC in either mode; compare every block
    base = baseline_coefs(emu_baseline, jp.grid_files(entry, progressive=False), len(coef))
    e, _, h, scans = jp.parse(emu, b)
    extent = np.zeros(len(coef), bool)          # blocks inside each component's own extent
    at = 0
    for c in range(int(h["ncomp"])):
        hc, vc = (int(h["hs"]), int(h["vs"])) if c == 0 else (1, 1)
        gw, gh = int(h["mcu_x"]) * hc, int(h["mcu_y"]) * vc
        cw = int(h["w"]) if c == 0 else -(-int(h["w"]) // int(h["hs"]))
        ch = int(h["h"]) if c == 0 else -(-int(h["h"]) // int(h["vs"]))
        m = np.zeros((gh, gw), bool)
        m[:-(-ch // 8), :-(-cw // 8)] = True
        extent[at:at + gw * gh] = m.reshape(-1)
        at += gw * gh
    assert np.array_equal(coef[extent], base[extent])
    assert np.array_equal(coef[~extent][:, 1:], np.zeros_like(coef[~extent][:, 1:]))
    assert [int(s["wave"]) for s in scans] == jp.brute_waves(scans)


def test_pillow_default_script_waves(emu):
    b = jp.encode(jp.content("photo", 64, 64, 1), progressive=True, quality=90, subsampling=2)
    _, _, _, scans = jp.parse(emu, b)
    bands = [(tuple(int(c) for c in s["comp"][:s["ns"]]), int(s["ss"]), int(s["se"]), int(s["ah"]), int(s["wave"]))
             for s in scans]
    # DC, Y 1-5, Cr, Cb, Y 6-63 | Y refine, DC refine, Cr, Cb refine | last luma refinement
    assert [w for *_, w in bands] == [0, 0, 0, 0, 0, 1, 1, 1, 1, 2]
    assert bands[0][:3] == ((0, 1, 2), 0, 0) and bands[-1][:4] == ((0,), 1, 63, 1)


def _sos_offsets(b):
    """offsets of the SOS markers of a file"""
    out, i = [], 2
    while i + 4 <= len(b):
        if b[i] != 0xFF:
            i += 1
            continue
        m = b[i + 1]
        if m == 0xDA:
            out.append(i)
        if m in (0x00, 0xFF) or 0xD0 <= m <= 0xD9:
            i += 2 if m != 0xFF else 1
            continue
        if m == 0xDA:
            i += 2 + (b[i + 2] << 8 | b[i + 3])
            continue
        i += 2 + (b[i + 2] << 8 | b[i + 3])
    return out


def _patch_sos(b, k, ss=None, se=None, ahal=None):
    b = bytearray(b)
    at = _sos_offsets(bytes(b))[k]
    ns = b[at + 4]
    q = at + 5 + 2 * ns
    if ss is not None:
        b[q] = ss
    if se is not None:
        b[q + 1] = se
    if ahal is not None:
        b[q + 2] = ahal
    return bytes(b)


def _refused_cases():
    """(name, file, the refusal's reason, whether Pillow raises OSError on it rather than giving pixels)"""
    import jpeg_progressive_streams as ps
    import jpeg_progressive_writer as pw
    a = jp.content("photo", 40, 56, 3)
    b = jp.encode(a, progressive=True, quality=80, subsampling=2)
    sos = _sos_offsets(b)
    sof = b.index(b"\xff\xc2")
    rng = np.random.default_rng(1)
    gray, s444 = [(1, 1)], [(1, 1)] * 3
    blk = ps._blocks(rng, 16, 24, gray, {0: ps.QA}, [0])
    ac_first = pw.write(16, 24, blk, {0: ps.QA}, pw.script([ps._sc([0], 1, 63), ps._sc([0], 0, 0)]))
    blk3 = ps._blocks(rng, 16, 24, s444, {0: ps.QA, 1: ps.QB}, [0, 1, 1])
    multi = pw.write(16, 24, blk3, {0: ps.QA, 1: ps.QB},
                     pw.script([ps._sc([0, 1, 2], 0, 0), ps._sc([0, 1], 1, 63), ps._sc([2], 1, 63)]))
    return [
        ("cut before the last scan", b[:sos[-1]] + b"\xff\xd9", "incomplete progression", False),
        ("progressive arithmetic", b[:sof] + b"\xff\xca" + b[sof + 2:], "progressive arithmetic coding", False),
        ("DC scan with AC", _patch_sos(b, 0, se=5), "bad progression", True),
        ("AC scan of several components", multi, "bad progression", True),
        ("Se above 63", _patch_sos(b, 1, se=64), "bad progression", True),
        ("Ss above Se", _patch_sos(b, 1, ss=6, se=5), "bad progression", True),
        ("Al above 13", _patch_sos(b, 0, ahal=0x0E), "bad progression", True),
        ("Ah not Al + 1", _patch_sos(b, 5, ahal=0x31), "bad progression", True),
        ("refinement at the wrong bit", _patch_sos(b, 5, ahal=0x32), "bad progression", False),
        ("second first pass", _patch_sos(b, 5, ahal=0x01), "bad progression", False),
        ("AC before the component's DC", ac_first, "AC before the component's first DC scan", False),
        ("baseline file", jp.encode(a, quality=80), "not a progressive frame", False),
    ]


@pytest.mark.parametrize("case", _refused_cases(), ids=lambda c: c[0])
def test_refusals_name_their_reason(emu, case):
    name, b, reason, pillow_raises = case
    e, why, _, _ = jp.parse(emu, b)
    assert e != 0 and reason in why, (name, why)
    hdr = np.zeros(1, _lib.JPEG_HEADER_DTYPE)
    scans = np.zeros(64, _lib.JPEG_SCAN_DTYPE)
    n = C.c_int(0)
    assert _lib.lib.faa_jpeg_parse_progressive(b, len(b), hdr.ctypes.data, scans.ctypes.data, 64, C.byref(n)) != 0
    assert reason in _lib.lib.faa_last_error().decode()
    # what Pillow does with the same file: libjpeg stops on some, and decodes the others (with a warning, or with
    # smoothing of an incomplete progression), which is why they stay with Pillow
    if pillow_raises:
        with pytest.raises(OSError):
            jp.pillow(b)
    else:
        px = jp.pillow(b)
        assert px.ndim == 3 and px.shape[2] == 3


def test_corrupt_streams_stay_in_their_buffers(emu):
    rng = np.random.default_rng(5)
    base = jp.encode(jp.content("photo", 48, 72, 2), progressive=True, quality=85, subsampling=2,
                     restart_marker_blocks=2)
    sos = _sos_offsets(base)
    seen = 0
    for k in range(200):
        b = bytearray(base)
        for _ in range(1 + k % 4):
            at = int(rng.integers(sos[0] + 12, len(b) - 2))
            b[at] = int(rng.integers(0, 256))
        b = bytes(b)
        e, _, _, _ = jp.parse(emu, b)
        if e != 0:
            continue
        st, _, _ = jp.decode(emu, b)       # guard bytes checked inside
        seen += st != 0
    assert seen > 0


def test_parse_headers_takes_progressive_files_only_when_asked(emu):
    a = jp.content("photo", 33, 47, 4)
    files = [jp.encode(a, quality=90), jp.encode(a, progressive=True, quality=90, subsampling=2),
             jp.encode(a, progressive=True, quality=60, subsampling=0, optimize=True)]
    headers, pool, refused = parse_jpeg_headers(files)
    assert [i for i, _ in refused] == [1, 2] and all("progressive coding" in r for _, r in refused)
    headers, pool, refused, scans, scan_first = parse_jpeg_headers(files, progressive=True)
    assert refused == []
    assert list(headers["reserved"]) == [0, 1, 1] and list(np.diff(scan_first)) == [0, 10, 10]
    assert (headers["pool"][1:, :3] >= 0).all() and (headers["pool"][1:, 3:] == -1).all()
    for s in scans:                              # every table a scan uses is in the pool, and only those
        used = [k for k in range(3) if s["ss"] == 0 and s["ah"] == 0 and k < s["ns"]] + ([3] if s["ss"] > 0 else [])
        assert all(0 <= s["pool"][k] < len(pool) for k in used)
        assert all(s["pool"][k] == -1 for k in range(6) if k not in used)
    assert len({p.tobytes() for p in pool}) == len(pool)
    for i in (1, 2):
        assert _lib.lib.faa_jpeg_index_capacity(headers[i:i + 1].ctypes.data) == 0
    with pytest.raises(ValueError, match="progressive coding"):
        EncodedImages.from_bytes(files, "cpu")
