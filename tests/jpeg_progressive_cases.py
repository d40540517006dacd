"""Progressive JPEG files of the progressive decoder tests, written by Pillow from seeded content, and the host build
of the progressive decoder (tests/emu/faa_emu_jpeg_progressive.cpp).

``GRID`` lists (name, h, w, content, save options) over sizes (every width and height residue mod 16 at small sizes,
photo sizes, 2048 x 1536), 4:4:4 / 4:2:2 / 4:2:0 / grayscale, qualities 1 to 100, optimised Huffman tables and restart
intervals; the baseline file of the same options holds the same quantised coefficients."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import PIL.Image
import PIL.ImageFile

from helpers import ROOT
from jpeg_cases import content

from fast_autoaugment_b200 import _lib

SCAN = _lib.JPEG_SCAN_DTYPE
HEADER = _lib.JPEG_HEADER_DTYPE


def encode(a, gray=False, **opts):
    """Pillow's JPEG of ``a`` (``progressive=True`` for a progressive file); MAXBLOCK raised so that large
    progressive saves need no suspension"""
    im = PIL.Image.fromarray(a)
    if gray:
        im = im.convert("L")
    bio = io.BytesIO()
    old = PIL.ImageFile.MAXBLOCK
    PIL.ImageFile.MAXBLOCK = max(old, a.shape[0] * a.shape[1] * 4 + 65536)
    try:
        im.save(bio, "JPEG", **opts)
    finally:
        PIL.ImageFile.MAXBLOCK = old
    return bio.getvalue()


def pillow(b):
    return np.asarray(PIL.Image.open(io.BytesIO(b)).convert("RGB"))


def _grid():
    g = []
    sizes = [(1, 1), (2, 3), (8, 8)] + [(h, 16 + r) for r, h in zip(range(16), [9, 17, 23, 31] * 4)] + \
        [(16 + r, w) for r, w in zip(range(16), [9, 17, 23, 31] * 4)]
    for k, (h, w) in enumerate(sizes):
        for sub in (0, 1, 2):
            g.append(("s%dx%d_%d" % (h, w, sub), h, w, ("noise", "photo", "gradient")[k % 3],
                      dict(quality=(1, 50, 75, 90, 100)[(k + sub) % 5], subsampling=sub)))
        g.append(("s%dx%d_g" % (h, w), h, w, "photo", dict(quality=75, gray=True)))
    for h, w in [(375, 500), (500, 375), (333, 500)]:
        for sub in (0, 1, 2):
            for q in (1, 75, 90, 100):
                g.append(("p%dx%d_%d_q%d" % (h, w, sub, q), h, w, "photo", dict(quality=q, subsampling=sub)))
        g.append(("p%dx%d_opt" % (h, w), h, w, "photo", dict(quality=90, subsampling=2, optimize=True)))
        g.append(("p%dx%d_g" % (h, w), h, w, "photo", dict(quality=90, gray=True)))
        g.append(("p%dx%d_rb1" % (h, w), h, w, "photo", dict(quality=90, subsampling=2, restart_marker_blocks=1)))
        g.append(("p%dx%d_rb3" % (h, w), h, w, "noise", dict(quality=75, subsampling=0, restart_marker_blocks=3)))
        g.append(("p%dx%d_rr1" % (h, w), h, w, "photo", dict(quality=75, subsampling=1, restart_marker_rows=1)))
    g.append(("big2048", 1536, 2048, "photo", dict(quality=90, subsampling=2)))
    return g


GRID = _grid()


def grid_files(entry, progressive=True):
    name, h, w, kind, opts = entry
    opts = dict(opts)
    gray = opts.pop("gray", False)
    a = content(kind, h, w, hash(name) % 1000)
    return encode(a, gray=gray, progressive=progressive, **opts)


def load_emu():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_progressive.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_progressive.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64 = C.c_void_p, C.c_int64
    lib.faa_emu_jpeg_progressive_parse.argtypes = [vp, i64, vp, vp, C.c_int, vp, C.POINTER(C.c_char_p)]
    lib.faa_emu_jpeg_scan_waves.argtypes = [vp, C.c_int]
    lib.faa_emu_jpeg_scan_waves.restype = None
    lib.faa_emu_jpeg_progressive_decode.argtypes = [vp, i64, vp, i64, vp, vp, vp, i64]
    return lib


def parse(lib, b):
    """(JPARSE code, reason, header, scans) of the host build"""
    src = np.frombuffer(b, np.uint8).copy()
    hdr = np.zeros(1, HEADER)
    scans = np.zeros(64, SCAN)
    n = np.zeros(1, np.int32)
    why = C.c_char_p()
    e = lib.faa_emu_jpeg_progressive_parse(src.ctypes.data, src.size, hdr.ctypes.data, scans.ctypes.data, 64,
                                           n.ctypes.data, C.byref(why))
    return e, (why.value or b"").decode(), hdr[0], scans[:int(n[0])].copy()


GUARD = 64


def decode(lib, b):
    """(status, pixels [h, w, 3], coefficients int16 [blocks, 64]) of the host build, guard bytes checked"""
    e, why, h, _ = parse(lib, b)
    assert e == 0, why
    src = np.frombuffer(b, np.uint8).copy()
    H, W = int(h["h"]), int(h["w"])
    blocks = int(h["mcu_x"]) * int(h["mcu_y"]) * (1 if int(h["ncomp"]) == 1 else int(h["hs"]) * int(h["vs"]) + 2)
    out = np.full(H * W * 3 + 2 * GUARD, 0xA5, np.uint8)
    coef = np.full(blocks * 64 + 2 * GUARD, 0x5A5A, np.int16)
    st = np.zeros(1, np.int32)
    hw = np.zeros(2, np.int32)
    assert lib.faa_emu_jpeg_progressive_decode(src.ctypes.data, src.size, out[GUARD:].ctypes.data, H * W * 3,
                                               st.ctypes.data, hw.ctypes.data, coef[GUARD:].ctypes.data,
                                               blocks * 64) == 0
    assert (out[:GUARD] == 0xA5).all() and (out[GUARD + H * W * 3:] == 0xA5).all()
    assert (coef[:GUARD] == 0x5A5A).all() and (coef[GUARD + blocks * 64:] == 0x5A5A).all()
    return int(st[0]), out[GUARD:GUARD + H * W * 3].reshape(H, W, 3), coef[GUARD:GUARD + blocks * 64].reshape(-1, 64)


def brute_waves(scans):
    """waves by the definition: 1 + the largest wave of an earlier scan sharing a component and a coefficient"""
    w = []
    for i, s in enumerate(scans):
        own = {(int(c), q) for c in s["comp"][:s["ns"]] for q in range(s["ss"], s["se"] + 1)}
        deps = [w[j] for j in range(i)
                if own & {(int(c), q) for c in scans[j]["comp"][:scans[j]["ns"]] for q in range(scans[j]["ss"], scans[j]["se"] + 1)}]
        w.append(max(deps) + 1 if deps else 0)
    return w
