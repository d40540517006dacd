"""JPEG files of the decoder tests, generated at test time with Pillow from seeded content, and the host build of the
decoder (tests/emu/faa_emu_jpeg.cpp).

``GRID`` lists (name, h, w, content, save options) over the sizes and encoder settings the decoder must match Pillow
on: small and odd sizes with every content, subsampling and quality; photo sizes with the settings a dataset holds;
Huffman tables of ``optimize=True``, restart intervals and grayscale everywhere."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import PIL.Image

from helpers import ROOT

SMALL = [(1, 1), (7, 9), (8, 8)] + [(a, b) for a in (15, 16, 17) for b in (31, 32, 33)] + \
    [(b, a) for a in (15, 16, 17) for b in (31, 32, 33)]
PHOTO = [(375, 500), (500, 375), (333, 500), (480, 640)]
CONTENTS = ("noise", "gradient", "flat0", "flat255", "photo")
QUALITIES = (1, 50, 75, 95, 100)
SUBSAMPLING = (0, 1, 2)                       # 4:4:4, 4:2:2, 4:2:0
EXTRAS = ({"optimize": True}, {"restart_marker_blocks": 1}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1})


def content(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        g = np.linspace(0, 255, w)[None, :, None] * np.array([1.0, 0.6, 0.2]) + np.linspace(0, 90, h)[:, None, None]
        return np.clip(g, 0, 255).astype(np.uint8)
    if kind in ("flat0", "flat255"):
        return np.full((h, w, 3), 0 if kind == "flat0" else 255, np.uint8)
    # photo-like: smooth shading, a few saturated shapes, fine texture and sensor noise
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 120 + 70 * np.sin(xx / max(w, 1) * 5 + seed)[..., None] * np.array([1.0, 0.7, 0.4]) + \
        40 * np.cos(yy / max(h, 1) * 3)[..., None]
    for _ in range(4):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(1, max(2, min(h, w) // 3 + 2))
        base[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.integers(0, 256, 3)
    base += 25 * np.sin(xx * 0.9 + yy * 0.4)[..., None] * (xx > w / 2)[..., None]
    base += rng.normal(0, 6, (h, w, 3))
    return np.clip(base, 0, 255).astype(np.uint8)


def encode(a, gray=False, **opts):
    im = PIL.Image.fromarray(a)
    if gray:
        im = im.convert("L")
    bio = io.BytesIO()
    im.save(bio, "JPEG", **opts)
    return bio.getvalue()


def pillow(b):
    return np.asarray(PIL.Image.open(io.BytesIO(b)).convert("RGB"))


def _grid():
    cases = []
    for h, w in SMALL:
        for kind in CONTENTS:
            for sub in SUBSAMPLING:
                for q in QUALITIES:
                    cases.append(("%s-%dx%d-s%d-q%d" % (kind, h, w, sub, q), h, w, kind, {"subsampling": sub, "quality": q}))
        for sub in SUBSAMPLING:
            for extra in EXTRAS:
                cases.append(("photo-%dx%d-s%d-%s" % (h, w, sub, "-".join("%s%s" % kv for kv in extra.items())), h, w, "photo",
                              dict(subsampling=sub, quality=90, **extra)))
        cases.append(("gray-%dx%d" % (h, w), h, w, "photo", {"gray": True, "quality": 75}))
    for h, w in PHOTO:
        for kind in ("photo", "noise"):
            for sub in SUBSAMPLING:
                for q in QUALITIES:
                    cases.append(("%s-%dx%d-s%d-q%d" % (kind, h, w, sub, q), h, w, kind, {"subsampling": sub, "quality": q}))
        for sub in SUBSAMPLING:
            for extra in EXTRAS:
                cases.append(("photo-%dx%d-s%d-%s" % (h, w, sub, "-".join("%s%s" % kv for kv in extra.items())), h, w, "photo",
                              dict(subsampling=sub, quality=85, **extra)))
        cases.append(("gray-%dx%d" % (h, w), h, w, "photo", {"gray": True, "quality": 90}))
        cases.append(("gray-%dx%d-rst" % (h, w), h, w, "gradient", {"gray": True, "quality": 50, "restart_marker_blocks": 3}))
    for extra in ({"subsampling": 2, "quality": 75}, {"subsampling": 0, "quality": 95, "restart_marker_rows": 1},
                  {"gray": True, "quality": 90}):
        cases.append(("photo-2048x1536-%s" % "-".join("%s%s" % kv for kv in extra.items()), 2048, 1536, "photo", extra))
    return cases


GRID = _grid()


def make(case, seed=0):
    """(file bytes, Pillow's decode) of one GRID case"""
    _, h, w, kind, opts = case
    opts = dict(opts)
    gray = opts.pop("gray", False)
    b = encode(content(kind, h, w, seed + h * 7 + w), gray=gray, **opts)
    return b, pillow(b)


def load_emu_jpeg():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    lib.faa_emu_jpeg_decode.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.faa_emu_jpeg_decode_mode.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    return lib


SERIAL, TILED, TILED_TRIMMED = 0, 1, 2      # decodes of the host build (faa_emu_jpeg_decode_mode)


def emu_decode(lib, b, mode=SERIAL):
    """(parse result, status bits, uint8 [h, w, 3]) of the host build on file bytes b: serially, or with the kernels'
    split of the work (TILED; TILED_TRIMMED with chroma windows one block too narrow)"""
    src = np.frombuffer(b, np.uint8).copy()
    hw = np.zeros(2, np.int32)
    st = np.zeros(1, np.int32)
    e = lib.faa_emu_jpeg_decode_mode(src.ctypes.data, src.size, None, 0, st.ctypes.data, hw.ctypes.data, mode)
    if e:
        return e, 0, None
    out = np.zeros((int(hw[0]), int(hw[1]), 3), np.uint8)
    e = lib.faa_emu_jpeg_decode_mode(src.ctypes.data, src.size, out.ctypes.data, out.size, st.ctypes.data,
                                     hw.ctypes.data, mode)
    return e, int(st[0]), out
