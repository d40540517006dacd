"""The host build of the JPEG scan index (tests/emu/faa_emu_jpeg_index.cpp), the placement rule restated from its
definition, and the fuzzed indexes the decoder must survive, shared by the CPU and GPU tests of the index."""
import ctypes as C
import os
import subprocess

import numpy as np

import jpeg_streams as js
from helpers import ROOT
from jpeg_cases import content, encode

from fast_autoaugment_b200 import _lib

SYNC = _lib.JPEG_SYNC_DTYPE
MAX_PARTS, BYTES_PER_PART = 128, 1024


def load_emu_index():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_index.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_index.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64 = C.c_void_p, C.c_int64
    lib.faa_emu_jpeg_index.argtypes = [vp, i64, vp, C.c_int32, vp, vp]
    lib.faa_emu_jpeg_states.argtypes = [vp, i64, vp, i64]
    lib.faa_emu_jpeg_states.restype = i64
    lib.faa_emu_jpeg_decode_indexed.argtypes = [vp, i64, vp, i64, vp, i64, vp, vp]
    lib.faa_emu_jpeg_index_linked.argtypes = [vp, i64, vp, i64]
    return lib


def parts(scan_len, restart):
    """P of the placement rule: min(128, scan_len / 1024) segments, none below 2 or with a restart interval"""
    p = min(MAX_PARTS, scan_len // BYTES_PER_PART)
    return 0 if restart or p < 2 else p


def host_index(lib, b, cap=MAX_PARTS - 1):
    """(points, status, (scan_off, scan_len)) of the recording decode of the host build"""
    src = np.frombuffer(b, np.uint8).copy()
    out = np.zeros(max(cap, 1), SYNC)
    st = np.zeros(1, np.int32)
    scan = np.zeros(2, np.int64)
    n = lib.faa_emu_jpeg_index(src.ctypes.data, src.size, out.ctypes.data, cap, st.ctypes.data, scan.ctypes.data)
    assert n >= 0
    return out[:n].copy(), int(st[0]), (int(scan[0]), int(scan[1]))


def host_states(lib, b, mcus):
    """the serial decoder's state at MCU boundaries 0 .. mcus - 1 (chained one-MCU segments)"""
    src = np.frombuffer(b, np.uint8).copy()
    out = np.zeros(max(mcus, 1), SYNC)
    n = lib.faa_emu_jpeg_states(src.ctypes.data, src.size, out.ctypes.data, mcus)
    return out[:n]


def rule_points(states, scan_len, restart):
    """the points the placement rule puts on a scan whose boundary states are ``states``"""
    p = parts(scan_len, restart)
    out, last = [], -1
    for k in range(1, p):
        hit = np.nonzero((states["byte"][1:] >= k * scan_len // p))[0]
        if len(hit) and hit[0] + 1 != last:
            last = int(hit[0]) + 1
            out.append(states[last])
    return np.array(out, SYNC)


def decode_indexed(lib, b, pts, guard=64):
    """(status, pixels) of the host build's indexed decode, with guard bytes around the file, the points and the
    output that must keep their value"""
    pts = np.asarray(pts, SYNC).reshape(-1)
    src = np.full(len(b) + 2 * guard, 0x5A, np.uint8)
    src[guard:guard + len(b)] = np.frombuffer(b, np.uint8)
    praw = np.full(pts.nbytes + 2 * guard, 0x3C, np.uint8)
    praw[guard:guard + pts.nbytes] = pts.view(np.uint8)
    hw = np.zeros(2, np.int32)
    st = np.zeros(1, np.int32)
    assert lib.faa_emu_jpeg_decode_indexed(src.ctypes.data + guard, len(b), None, 0, None, 0, st.ctypes.data,
                                           hw.ctypes.data) == 0
    n = int(hw[0]) * int(hw[1]) * 3
    out = np.full(n + 2 * guard, 0xA5, np.uint8)
    assert lib.faa_emu_jpeg_decode_indexed(src.ctypes.data + guard, len(b), praw.ctypes.data + guard, len(pts),
                                           out.ctypes.data + guard, n, st.ctypes.data, hw.ctypes.data) == 0
    assert (src[:guard] == 0x5A).all() and (src[guard + len(b):] == 0x5A).all()
    assert src[guard:guard + len(b)].tobytes() == b
    assert (praw[:guard] == 0x3C).all() and (praw[guard + pts.nbytes:] == 0x3C).all()
    assert praw[guard:guard + pts.nbytes].tobytes() == pts.tobytes()
    assert (out[:guard] == 0xA5).all() and (out[guard + n:] == 0xA5).all()
    return int(st[0]), out[guard:guard + n].reshape(int(hw[0]), int(hw[1]), 3)


def linked(lib, b, pts):
    pts = np.ascontiguousarray(pts, SYNC).reshape(-1)
    src = np.frombuffer(b, np.uint8).copy()
    return lib.faa_emu_jpeg_index_linked(src.ctypes.data, src.size, pts.ctypes.data if len(pts) else None, len(pts))


# restart-free files with indexes of many segments, for the fuzzing
def indexed_files():
    out = []
    for name, (h, w, kind, opts) in {"photo-375x500-420-q90": (375, 500, "photo", {"subsampling": 2, "quality": 90}),
                                     "noise-96x128-444-q95": (96, 128, "noise", {"subsampling": 0, "quality": 95}),
                                     "photo-500x375-422-q75": (500, 375, "photo", {"subsampling": 1, "quality": 75}),
                                     "gray-480x640-q90": (480, 640, "photo", {"gray": True, "quality": 90})}.items():
        opts = dict(opts)
        gray = opts.pop("gray", False)
        out.append((name, encode(content(kind, h, w, 3), gray=gray, **opts)))
    return out


def big_file():
    """a restart-free file of more than 128 KiB of scan: an index of 127 points, 128 segments"""
    return encode(content("noise", 640, 640, 5), quality=95, subsampling=0)


def stuffed_offsets(b, scan_off, scan_len):
    """scan offsets of the 0x00 of every stuffed 0xFF 0x00 pair"""
    s = np.frombuffer(b, np.uint8)[scan_off:scan_off + scan_len]
    return (np.nonzero((s[:-1] == 0xFF) & (s[1:] == 0x00))[0] + 1).tolist()


def fuzzed(pts, other, scan, mcus, b, states=None):
    """[(name, points)]: an index broken in every way the decoder must survive (each field off by one at the first,
    a middle and the last point; another file's points; shuffled, duplicated, truncated lists; out-of-range values; a
    point on the 0x00 of a stuffed pair)"""
    out = []
    n = len(pts)
    for k in sorted({0, n // 2, n - 1}):
        for field in ("mcu", "byte", "bit", "pred0", "pred1", "pred2"):
            for d in (-1, 1):
                q = pts.copy()
                if field.startswith("pred"):
                    q["pred"][k, int(field[-1])] += d
                else:
                    q[field][k] += d
                out.append(("%s%+d@%d" % (field, d, k), q))
    out.append(("other-file", other))
    rng = np.random.default_rng(n)
    out.append(("shuffled", pts[rng.permutation(n)]))
    out.append(("duplicated", np.sort(np.concatenate([pts, pts[n // 2:n // 2 + 1]]), order="mcu", kind="stable")))
    out.append(("truncated-head", pts[:n // 2]))
    out.append(("truncated-tail", pts[n // 2:]))
    out.append(("one-point", pts[n // 2:n // 2 + 1]))
    for name, field, v in (("mcu0", "mcu", 0), ("mcu-end", "mcu", mcus), ("mcu-neg", "mcu", -5), ("byte-neg", "byte", -1),
                           ("byte-end", "byte", scan[1]), ("byte-huge", "byte", 2 ** 31 - 1), ("bit8", "bit", 8),
                           ("bit-neg", "bit", -1)):
        q = pts.copy()
        q[field][n // 2] = v
        out.append((name, q))
    out.append(("too-many", np.sort(np.concatenate([pts] * (MAX_PARTS // max(n, 1) + 1)), order="mcu")))
    garbage = np.frombuffer(np.random.default_rng(9).integers(0, 256, n * 16, dtype=np.uint8).tobytes(), SYNC)
    out.append(("random", garbage.copy()))
    stuffed = stuffed_offsets(b, *scan)
    if stuffed and states is not None:
        # a point whose byte is the 0x00 of the stuffed pair its real state sits on (or the nearest such pair)
        q = pts.copy()
        k = n // 2
        at = min(stuffed, key=lambda o: abs(o - 1 - int(q["byte"][k])))
        q["byte"][k] = at
        out.append(("on-stuffed-zero", q))
    return out


def stream_cases():
    """the restart-free hand-built streams of tests/jpeg_streams.py's geometry groups"""
    from fast_autoaugment_b200.engine import parse_jpeg
    out = []
    for n, b in js.RANDOM + js.EDGE + js.LAYOUTS + js.NARROW + js.TILE_EDGES + js.SEGMENT_COUNTS:
        hdr = parse_jpeg(b)[0]
        if hdr is not None and int(hdr["restart"][0]) == 0:
            out.append((n, b))
    return out
