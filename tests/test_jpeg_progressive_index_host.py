"""The scan index of progressive JPEG files without a GPU: the host build (tests/emu/faa_emu_jpeg_progressive_index.cpp,
the faa_jpeg.cuh the progressive kernel runs, split into waves, work items and whole-image redo as the kernel splits
it) on Pillow-written progressive files and hand-built streams.  Recorded points equal the placement rule computed a
second way, by chaining one-unit segments; decodes from any index, recorded, chosen or fuzzed, and from a corrupt
file's stale index, give the pixels and status of the decode without one and stay inside their guard bytes.  Also the
C ABI's capacity and refusals for scan-indexed headers, and the Python parse."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_progressive_cases as jp
import jpeg_progressive_writer as pw
from helpers import ROOT
from jpeg_writer import block_grid

from fast_autoaugment_b200 import _lib, engine

SYNC = _lib.JPEG_SYNC_DTYPE
GUARD = 64
INDEXED = _lib.JPEG_PROGRESSIVE | _lib.JPEG_SCAN_INDEXED


def load_emu():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_progressive_index.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_progressive_index.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    lib.faa_emu_jpi_header.argtypes = [vp, i64, i32, vp, vp]
    lib.faa_emu_jpi_decode.argtypes = [vp, i64, i32, vp, i64, vp, i64, vp, vp, i64, vp, i64, vp]
    lib.faa_emu_jpi_rule.argtypes = [vp, i64, vp, i64]
    lib.faa_emu_jpi_state.argtypes = [vp, i64, i32, i64, vp]
    return lib


@pytest.fixture(scope="module")
def emu():
    return load_emu()


def header(lib, b, indexed=1):
    src = np.frombuffer(b, np.uint8).copy()
    h = np.zeros(1, _lib.JPEG_HEADER_DTYPE)
    n = np.zeros(1, np.int32)
    assert lib.faa_emu_jpi_header(src.ctypes.data, src.size, indexed, h.ctypes.data, n.ctypes.data) == 0
    return h[0]


def parts(h):
    p = int(h["scan_len"]) // 1024
    return 0 if p < 2 else min(p, 128)


def decode(lib, b, pts=None, record=False, indexed=1):
    """(status, pixels, coefficients, recorded points or None) of the host build, every buffer inside guard bytes"""
    h = header(lib, b, indexed)
    H, W = int(h["h"]), int(h["w"])
    blocks = int(h["mcu_x"]) * int(h["mcu_y"]) * (1 if int(h["ncomp"]) == 1 else int(h["hs"]) * int(h["vs"]) + 2)
    src = np.frombuffer(b, np.uint8).copy()
    out = np.full(H * W * 3 + 2 * GUARD, 0xA5, np.uint8)
    coef = np.full(blocks * 64 + 2 * GUARD, 0x5A5A, np.int16)
    cap = 127
    rec = np.zeros(cap + 8, SYNC)
    rec.view(np.uint8)[:] = 0x77
    cnt = np.full(3, 0x7777, np.int32)
    st = np.zeros(1, np.int32)
    p = None if pts is None else np.ascontiguousarray(pts, SYNC)
    assert lib.faa_emu_jpi_decode(src.ctypes.data, src.size, indexed, None if p is None else p.ctypes.data,
                                  0 if p is None else len(p), rec[4:].ctypes.data if record else None, cap,
                                  cnt[1:].ctypes.data if record else None, out[GUARD:].ctypes.data, H * W * 3,
                                  coef[GUARD:].ctypes.data, blocks * 64, st.ctypes.data) == 0
    assert (out[:GUARD] == 0xA5).all() and (out[GUARD + H * W * 3:] == 0xA5).all()
    assert (coef[:GUARD] == 0x5A5A).all() and (coef[GUARD + blocks * 64:] == 0x5A5A).all()
    assert cnt[0] == 0x7777 and cnt[2] == 0x7777
    n = int(cnt[1]) if record else 0
    assert (rec.view(np.uint8)[:64] == 0x77).all() and (rec[4 + n:].view(np.uint8) == 0x77).all()
    return (int(st[0]), out[GUARD:GUARD + H * W * 3].reshape(H, W, 3), coef[GUARD:GUARD + blocks * 64],
            rec[4:4 + n].copy() if record else None)


def rule(lib, b):
    src = np.frombuffer(b, np.uint8).copy()
    at = np.zeros(127, SYNC)
    n = lib.faa_emu_jpi_rule(src.ctypes.data, src.size, at.ctypes.data, 127)
    return None if n < 0 else at[:n].copy()


# --------------------------------------------------------------------------------------------------------- inputs --
def _sc(comps, ss, se, ah=0, al=0, **kw):
    return dict(comps=list(comps), ss=ss, se=se, ah=ah, al=al, **kw)


EOB_HW = (2048, 1400)


def _streams():
    """hand-built streams big enough to get points: (name, bytes)"""
    rng = np.random.default_rng(77)
    qa = np.arange(1, 65, dtype=np.int64) % 5 + 1
    out = []
    # EOB runs that span points, up to 32767 blocks and across block rows: dense bands between empty ones.  Rows 20
    # .. 248 (39900 blocks) are empty: one run of 32767 blocks, then one of 7133
    h, w = EOB_HW
    rows, cols = block_grid(h, w, [(1, 1)], 0)
    b = np.zeros((rows, cols, 64), np.int16)
    b[..., 0] = rng.integers(-200, 200, (rows, cols))
    dense = np.zeros((rows, cols), bool)
    dense[:8], dense[12:20], dense[-8:] = True, True, True
    dense &= rng.random((rows, cols)) < 0.5
    ac = rng.integers(-40, 40, (rows, cols, 63)) * (rng.random((rows, cols, 63)) < 0.3)
    b[..., 1:] = np.where(dense[..., None], ac, 0)
    sc = [_sc([0], 0, 0), _sc([0], 1, 63, 0, 1), _sc([0], 1, 63, 1, 0)]
    out.append(("eobrun_span", pw.write(h, w, [b], {0: qa}, pw.script(sc), sampling=[(1, 1)], qsel=[0])))
    # interleaved DC with three predictors, restart-free and restart scans in one file, DHT redefined at every scan
    h, w = 320, 480
    samp = [(2, 2), (1, 1), (1, 1)]
    blocks = []
    for c in range(3):
        r, cc = block_grid(h, w, samp, c)
        x = np.zeros((r, cc, 64), np.int16)
        x[..., 0] = rng.integers(-300, 300, (r, cc))
        x[..., 1:] = rng.integers(-30, 30, (r, cc, 63)) * (rng.random((r, cc, 63)) < 0.25)
        er, ec = pw.extent(h, w, samp, c)
        x[er:, :, 1:] = 0
        x[:, ec:, 1:] = 0
        blocks.append(x)
    sc = [_sc([0, 1, 2], 0, 0, 0, 1), _sc([0], 1, 5, 0, 2, restart=0), _sc([1], 1, 63, 0, 1, restart=17),
          _sc([2], 1, 63, 0, 1, restart=0), _sc([0], 6, 63, 0, 2), _sc([0, 1, 2], 0, 0, 1, 0),
          _sc([0], 1, 63, 2, 1), _sc([0], 1, 63, 1, 0, restart=40), _sc([1], 1, 63, 1, 0, restart=0),
          _sc([2], 1, 63, 1, 0)]
    out.append(("dc3_mixed_restarts", pw.write(h, w, blocks, {0: qa, 1: qa[::-1].copy()}, pw.script(sc),
                                               sampling=samp, qsel=[0, 1, 1])))
    return out


STREAMS = _streams()
PILLOW = [e for e in jp.GRID if e[0].startswith("p") or e[0] == "big2048"]


def _pillow_files():
    return [(e[0], jp.grid_files(e)) for e in PILLOW]


FILES = STREAMS + _pillow_files()


# ---------------------------------------------------------------------------------------------------------- tests --
@pytest.mark.parametrize("name,b", FILES, ids=[f[0] for f in FILES])
def test_recorded_points_are_the_rule_and_the_indexed_decode_is_the_serial_one(emu, name, b):
    st0, px0, coef0, _ = decode(emu, b, indexed=0)
    st, px, coef, pts = decode(emu, b, record=True)
    assert st == st0 == 0 and np.array_equal(px, px0) and np.array_equal(coef, coef0)
    assert np.array_equal(px, jp.pillow(b))
    want = rule(emu, b)
    assert want is not None and pts.tobytes() == want.tobytes()
    h = header(emu, b)
    assert len(pts) <= max(parts(h) - 1, 0)
    if "rb1" in name or "rb3" in name or "rr1" in name:
        assert len(pts) == 0                               # every scan has a restart interval
    # the indexed decode: the serial decode's coefficients, pixels and status, the points used as they stand
    st2, px2, coef2, again = decode(emu, b, pts=pts, record=True)
    assert st2 == 0 and np.array_equal(coef2, coef0) and np.array_equal(px2, px0)
    assert len(again) == 0 or len(pts) == 0
    # a reserved-1 header takes no points and records none
    st3, px3, _, none = decode(emu, b, pts=pts, record=True, indexed=0)
    assert st3 == 0 and np.array_equal(px3, px0) and len(none) == 0


def test_streams_cover_what_points_must_carry(emu):
    """EOB runs (first pass and refinement) spanning points, up to 32767 blocks, DC points with three predictors,
    thresholds on the 00 of a stuffed pair"""
    eob = STREAMS[0][1]
    e, _, h, scans = jp.parse(jp.load_emu(), eob)
    pts = rule(emu, eob)
    axis = np.concatenate([[0], np.cumsum(scans["len"])])
    scan_of = np.searchsorted(axis, pts["byte"], side="right") - 1
    ac_first = [k for k, s in enumerate(scans) if s["ss"] > 0 and s["ah"] == 0]
    ac_ref = [k for k, s in enumerate(scans) if s["ss"] > 0 and s["ah"] > 0]
    assert (pts["pred"][np.isin(scan_of, ac_first), 0] > 0).any()
    assert (pts["pred"][np.isin(scan_of, ac_ref), 0] > 0).any()
    dc3 = STREAMS[1][1]
    _, _, _, scans = jp.parse(jp.load_emu(), dc3)
    pts = rule(emu, dc3)
    axis = np.concatenate([[0], np.cumsum(scans["len"])])
    scan_of = np.searchsorted(axis, pts["byte"], side="right") - 1
    dc = [k for k, s in enumerate(scans) if s["ss"] == 0 and s["ah"] == 0 and s["ns"] == 3]
    assert (np.count_nonzero(pts["pred"][np.isin(scan_of, dc)], axis=1) == 3).any()
    assert any(scans[k]["restart"] > 0 for k in range(len(scans))) and \
        any(scans[k]["restart"] == 0 for k in range(len(scans)))
    assert all(scans[k]["restart"] == 0 for k in scan_of)
    # thresholds on the 00 of a stuffed pair, across the files
    on00 = 0
    for _, b in FILES:
        hh = header(emu, b)
        _, _, _, sc = jp.parse(jp.load_emu(), b)
        data = np.concatenate([np.frombuffer(b, np.uint8)[int(s["off"]):int(s["off"] + s["len"])] for s in sc])
        P = parts(hh)
        for k in range(1, P):
            t = k * int(hh["scan_len"]) // P
            on00 += t > 0 and data[t] == 0 and data[t - 1] == 0xFF
    assert on00 > 0


def state(lib, b, scan, unit):
    src = np.frombuffer(b, np.uint8).copy()
    at = np.zeros(1, SYNC)
    assert lib.faa_emu_jpi_state(src.ctypes.data, src.size, scan, unit, at.ctypes.data) == 1
    return at


def test_hand_chosen_points_inside_long_eob_runs_decode(emu):
    """points chosen by hand inside the EOB runs of the eobrun stream (one of 32767 blocks across rows, in the first
    pass and the refinement), and in the interleaved DC scan: used as they stand, and exact"""
    b = STREAMS[0][1]
    st0, px0, coef0, _ = decode(emu, b, indexed=0)
    _, _, h, scans = jp.parse(jp.load_emu(), b)
    rows, cols = block_grid(*EOB_HW, [(1, 1)], 0)
    chosen = []
    for k in (1, 2):                                              # AC first pass, AC refinement
        for u in (20 * cols + 1, (rows - 8) * cols - 2):          # (inside one run the byte stays put)
            chosen.append(state(emu, b, k, u))
    chosen.append(state(emu, b, 0, 1234))
    pts = np.sort(np.concatenate(chosen), order="byte")
    assert (pts["pred"][:, 0] > 32700).any()                        # (the run starts a few blocks earlier)
    assert len(np.unique(pts["byte"])) == len(pts)
    st, px, coef, again = decode(emu, b, pts=pts, record=True)
    assert st == st0 and np.array_equal(coef, coef0) and np.array_equal(px, px0)
    assert len(again) == 0                                       # used: nothing recorded
    dc3 = STREAMS[1][1]
    st0, px0, coef0, _ = decode(emu, dc3, indexed=0)
    pts = np.concatenate([state(emu, dc3, 0, u) for u in (7, 300, 555)])
    assert (np.count_nonzero(pts["pred"], axis=1) == 3).all()
    st, px, coef, again = decode(emu, dc3, pts=pts, record=True)
    assert st == st0 and np.array_equal(coef, coef0) and len(again) == 0


def _fuzzed(pts, other, rng, scans_len):
    """(what, points) of every kind of wrong index"""
    out = []
    for f in ("mcu", "byte", "bit"):
        for d in (-1, 1):
            q = pts.copy()
            k = int(rng.integers(len(q)))
            q[f][k] += d
            out.append(("%s%+d@%d" % (f, d, k), q))
    for c in range(3):
        q = pts.copy()
        k = int(rng.integers(len(q)))
        q["pred"][k, c] += 1
        out.append(("pred%d+1@%d" % (c, k), q))
    q = pts.copy()
    ks = np.flatnonzero(q["pred"][:, 0] > 0)
    if len(ks):
        q["pred"][ks[0], 0] -= 1
        out.append(("eobrun-1", q))
    q = pts.copy()
    k = len(q) // 2
    q["byte"][k] = (q["byte"][k] + scans_len[0]) % int(np.sum(scans_len))       # into another scan
    out.append(("other scan", q))
    out.append(("other file", other))
    out.append(("shuffled", rng.permutation(pts)))
    out.append(("duplicated", np.concatenate([pts[:3], pts[2:]])))
    out.append(("truncated", pts[:-1]))
    out.append(("first only", pts[:1]))
    out.append(("128 points", np.concatenate([pts] * (128 // len(pts) + 1))[:128]))
    return out


@pytest.mark.parametrize("k", range(len(STREAMS) + 3))
def test_fuzzed_indexes_give_the_unindexed_pixels_and_status(emu, k):
    files = [f[1] for f in STREAMS] + [f[1] for f in FILES if f[0] in ("p375x500_2_q90", "p500x375_0_q75", "big2048")]
    b = files[k]
    other = rule(emu, files[(k + 1) % len(files)])
    st0, px0, coef0, _ = decode(emu, b, indexed=0)
    pts = rule(emu, b)
    assert len(pts) > 3
    _, _, _, scans = jp.parse(jp.load_emu(), b)
    rng = np.random.default_rng(k)
    for what, q in _fuzzed(pts, other, rng, scans["len"]):
        st, px, coef, _ = decode(emu, b, pts=q)
        assert st == st0 and np.array_equal(px, px0) and np.array_equal(coef, coef0), what


@pytest.mark.parametrize("k", range(len(STREAMS) + 1))
def test_corrupt_files_with_the_intact_files_index(emu, k):
    files = [f[1] for f in STREAMS] + [f[1] for f in FILES if f[0] == "p375x500_2_q90"]
    b = files[k]
    pts = rule(emu, b)
    _, _, _, scans = jp.parse(jp.load_emu(), b)
    rng = np.random.default_rng(100 + k)
    for trial in range(12):
        bad = bytearray(b)
        s = scans[int(rng.integers(len(scans)))]
        if s["len"] < 4:
            continue
        for _ in range(1 + trial % 3):
            at = int(s["off"] + rng.integers(s["len"]))
            bad[at] = int(rng.integers(256)) if trial % 4 else bad[at] ^ (1 << int(rng.integers(8)))
        if trial % 5 == 4:
            bad = bad[:int(s["off"] + s["len"] // 2)]                      # cut inside a scan
        bad = bytes(bad)
        e, _, h, sc2 = jp.parse(jp.load_emu(), bad)
        if e != 0 or len(sc2) != len(scans) or int(np.sum(sc2["len"])) != int(np.sum(scans["len"])):
            continue                                                        # the parse sees another file
        st0, px0, coef0, _ = decode(emu, bad, indexed=0)
        st, px, coef, rec = decode(emu, bad, pts=pts, record=True)
        assert st == st0 and np.array_equal(px, px0) and np.array_equal(coef, coef0), trial
        assert st == 0 or len(rec) == 0


def test_capacity_of_scan_indexed_headers(emu):
    for _, b in FILES[:4]:
        h1 = np.array([header(emu, b, 0)], _lib.JPEG_HEADER_DTYPE)
        h3 = np.array([header(emu, b, 1)], _lib.JPEG_HEADER_DTYPE)
        assert int(h3["reserved"][0]) == INDEXED and int(h1["reserved"][0]) == _lib.JPEG_PROGRESSIVE
        assert _lib.lib.faa_jpeg_index_capacity(h1.ctypes.data) == 0
        assert _lib.lib.faa_jpeg_index_capacity(h3.ctypes.data) == max(parts(h3[0]) - 1, 0)
        assert np.array_equal(engine.jpeg_index_capacities(h3), [0, max(parts(h3[0]) - 1, 0)])


def test_python_parse_marks_scan_indexed_files():
    b = jp.grid_files(PILLOW[0])
    base = jp.encode(jp.content("photo", 64, 64, 1), progressive=False, quality=90)
    with pytest.raises(ValueError):
        engine.parse_jpeg_headers([b], progressive_index=True)
    with pytest.raises(ValueError):
        engine.EncodedImages.from_bytes([b], "cpu", progressive_index=True)
    h1 = engine.parse_jpeg_headers([b, base], progressive=True)
    h3 = engine.parse_jpeg_headers([b, base], progressive=True, progressive_index=True)
    scans, first = h3[3], h3[4]
    assert int(h1[0]["reserved"][0]) == 1 and int(h1[0]["scan_len"][0]) == 0
    assert int(h3[0]["reserved"][0]) == INDEXED
    assert int(h3[0]["scan_len"][0]) == int(scans["len"][first[0]:first[1]].sum())
    assert h3[0][1].tobytes() == h1[0][1].tobytes()                        # the baseline file is untouched
    for k in ("pool", "h", "w", "mcu_x", "mcu_y", "table_at"):
        assert np.array_equal(h3[0][k], h1[0][k])
    enc = engine.EncodedImages.from_bytes([b, base], "cpu", progressive=True, progressive_index=True)
    assert enc.progressive().tolist() == [True, False]
    assert enc.progressive_indexed().tolist() == [True, False]


DEV = 0x1000


@pytest.mark.skipif(__import__("torch").cuda.is_available(),
                    reason="a call that passes its checks would launch on the dummy pointers")
def test_abi_refusals_for_scan_indexed_headers():
    b = jp.grid_files(PILLOW[0])
    headers, pool, _, scans, scan_first = engine.parse_jpeg_headers([b], progressive=True, progressive_index=True)
    out = np.zeros(1, dtype=_lib.IMAGE_DTYPE)
    out["data"], out["h"], out["w"] = DEV, headers["h"][0], headers["w"][0]
    dec = engine._JpegDecoder()
    cap = engine.jpeg_index_capacities(headers)

    def call(h, rec=(None,) * 4, find=0):
        return _lib.lib.faa_jpeg_decode(dec.handle, h.ctypes.data, DEV, DEV, len(pool), DEV, 1, out.ctypes.data, DEV,
                                        DEV, *(None,) * 3, *rec, scans.ctypes.data, DEV, scan_first.ctypes.data, DEV,
                                        find, None)
    assert call(headers) == _lib.ERR_NO_DEVICE
    assert call(headers, (cap.ctypes.data, DEV, DEV, DEV)) == _lib.ERR_NO_DEVICE
    assert call(headers, (cap.ctypes.data, DEV, DEV, DEV), 1) == _lib.ERR_NO_DEVICE
    for d in (-1, 1, -int(headers["scan_len"][0])):
        bad = headers.copy()
        bad["scan_len"] += d
        assert call(bad) == _lib.ERR_VALUE, d
    for f, v in (("scan_off", 1), ("restart", 1)):
        bad = headers.copy()
        bad[f] = v
        assert call(bad) == _lib.ERR_VALUE, f
    bad = headers.copy()
    bad["reserved"] = _lib.JPEG_PROGRESSIVE
    assert call(bad) == _lib.ERR_VALUE                   # reserved 1 keeps its scan_len 0
    first = np.array([0, 4], np.int64)
    args = (headers.ctypes.data, DEV, DEV, len(pool), DEV, 1, first.ctypes.data, DEV, DEV, DEV)
    assert _lib.lib.faa_jpeg_index_build(*args, DEV, None) == _lib.ERR_VALUE
    assert _lib.lib.faa_jpeg_index_find(*args, None) == _lib.ERR_VALUE
