"""Oracle layer 2: NumPy restatement of the arithmetic *inside* Pillow and
torchvision for the calls the reference makes on the hot path.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Third-party algorithm notice.  The per-pixel arithmetic of the reference lives
in **Pillow** (C ``libImaging``), which is neither vendored under
the reference nor pinned by its ``requirements.txt``; the build image has
Pillow 12.2.0 (binary wheel, C sources absent).  The functions below restate
Pillow's published algorithms (``Geometry.c`` affine_fixed / ImagingScaleAffine,
``Blend.c``, ``Convert.c`` rgb2l, ``Filter.c`` 3x3, ``Point.c``, ``Histo.c``,
``Draw.c`` rectangle, and the Python-level ``ImageOps`` / ``ImageEnhance`` /
``Image.rotate``) and are pinned bit-exactly against Pillow 12.2.0 itself by
``tests/test_oracle_np_vs_pil.py`` and against outputs of the live reference by
``tests/golden``.  Each function names the reference call site it serves.

All images are ``uint8`` arrays of shape (H, W, 3), RGB, HWC.
"""
from __future__ import annotations

import math
import random

import numpy as np

from .pil_path import CUTOUT_RGB, RANGES, magnitude  # noqa: F401  (shared constants)

U8 = np.uint8
F32 = np.float32


# ---------------------------------------------------------------- geometry --
def fix16(z: float) -> int:
    """Pillow ``FIX(v) = FLOOR(v*65536.0 + 0.5)`` (Geometry.c, affine_fixed)."""
    return int(math.floor(z * 65536.0 + 0.5))


def fixed_coeffs(m):
    """6 float64 affine coefficients -> the six 16.16 integers of affine_fixed.
    The half-pixel centre offset is folded into a2 / a5."""
    m0, m1, m2, m3, m4, m5 = (float(t) for t in m)
    return (fix16(m0), fix16(m1), fix16(m2 + m0 * 0.5 + m1 * 0.5),
            fix16(m3), fix16(m4), fix16(m5 + m3 * 0.5 + m4 * 0.5))


def gather_fixed(img, a):
    """out[y,x] = in[yin,xin] with xin=(a2+a0*x+a1*y)>>16, yin=(a5+a3*x+a4*y)>>16
    (arithmetic shift), zero where outside.  Serves ShearX/ShearY/Rotate:
    augmentations.py:17,24,61."""
    h, w = img.shape[:2]
    a0, a1, a2, a3, a4, a5 = a
    x = np.arange(w, dtype=np.int64)[None, :]
    y = np.arange(h, dtype=np.int64)[:, None]
    xin = (a2 + a0 * x + a1 * y) >> 16
    yin = (a5 + a3 * x + a4 * y) >> 16
    ok = (xin >= 0) & (xin < w) & (yin >= 0) & (yin < h)
    out = np.zeros_like(img)
    out[ok] = img[yin[ok], xin[ok]]
    return out


def scale_axis_table(n_out, n_in, scale, offset):
    """ImagingScaleAffine's per-axis source table: ``o = offset + scale*0.5``,
    accumulated ``o += scale``; COORD(o) = -1 if o < 0 else int(o)."""
    tab = np.full(n_out, -1, dtype=np.int64)
    o = offset + scale * 0.5
    for i in range(n_out):
        c = -1 if o < 0.0 else int(o)
        if 0 <= c < n_in:
            tab[i] = c
        o += scale
    return tab


def gather_scale(img, m):
    """Pillow takes this path when m1 == m3 == 0 (pure scale + translate).
    Serves TranslateX/Y(/Abs): augmentations.py:32,40,47,54."""
    h, w = img.shape[:2]
    xs = scale_axis_table(w, w, float(m[0]), float(m[2]))
    ys = scale_axis_table(h, h, float(m[4]), float(m[5]))
    out = np.zeros_like(img)
    yok = np.nonzero(ys >= 0)[0]
    xok = np.nonzero(xs >= 0)[0]
    if len(yok) and len(xok):
        out[np.ix_(yok, xok)] = img[np.ix_(ys[yok], xs[xok])]
    return out


def affine_nearest(img, m):
    """``img.transform(size, AFFINE, m)`` with the default NEAREST filter."""
    if float(m[1]) == 0.0 and float(m[3]) == 0.0:
        return gather_scale(img, m)
    return gather_fixed(img, fixed_coeffs(m))


def rotate_matrix(angle_deg: float, w: int, h: int):
    """``Image.rotate`` (PIL/Image.py) up to the matrix; returns None for the
    angle==0 copy fast path, 'r180'/'r90'/'r270' for the transpose fast paths."""
    angle = angle_deg % 360.0
    if angle == 0:
        return None
    if angle == 180:
        return "r180"
    if angle in (90, 270) and w == h:
        return "r90" if angle == 90 else "r270"
    cx, cy = w / 2, h / 2
    t = -math.radians(angle)
    m = [round(math.cos(t), 15), round(math.sin(t), 15), 0.0,
         round(-math.sin(t), 15), round(math.cos(t), 15), 0.0]
    m[2] = m[0] * (-cx) + m[1] * (-cy) + m[2]
    m[5] = m[3] * (-cx) + m[4] * (-cy) + m[5]
    m[2] += cx
    m[5] += cy
    return m


def rotate(img, angle_deg):
    """augmentations.py:61 ``img.rotate(v)``."""
    h, w = img.shape[:2]
    m = rotate_matrix(angle_deg, w, h)
    if m is None:
        return img.copy()
    if m == "r180":
        return img[::-1, ::-1].copy()
    if m == "r90":
        return np.rot90(img, 1).copy()
    if m == "r270":
        return np.rot90(img, 3).copy()
    return affine_nearest(img, m)


# ------------------------------------------------------------- photometric --
def luma(img):
    """Pillow RGB->L: (19595 R + 38470 G + 7471 B + 0x8000) >> 16 (Convert.c)."""
    r = img[..., 0].astype(np.int64)
    g = img[..., 1].astype(np.int64)
    b = img[..., 2].astype(np.int64)
    return ((19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16).astype(U8)


def blend(deg, img, alpha: float):
    """``Image.blend(deg, img, alpha)`` (Blend.c): fp32, truncation, clip only
    when alpha is outside [0, 1]."""
    if alpha == 0.0:
        return deg.copy()
    if alpha == 1.0:
        return img.copy()
    a = F32(alpha)
    d = deg.astype(F32)
    t = d + a * (img.astype(F32) - d)          # every step rounds to fp32
    if 0.0 <= alpha <= 1.0:
        return t.astype(np.int32).astype(U8)
    out = np.where(t <= 0.0, 0, np.where(t >= 255.0, 255, t.astype(np.int32)))
    return out.astype(U8)


def brightness(img, v):     # augmentations.py:107-109
    return blend(np.zeros_like(img), img, v)


def color(img, v):          # augmentations.py:102-104
    g = luma(img)
    return blend(np.repeat(g[..., None], 3, axis=2), img, v)


def contrast_mean(img) -> int:
    """int(mean(L) + 0.5) of ImageEnhance.Contrast == (2*sum + N) // (2*N)."""
    g = luma(img).astype(np.int64)
    n = g.size
    return int((2 * int(g.sum()) + n) // (2 * n))


def contrast(img, v):       # augmentations.py:97-99
    return blend(np.full_like(img, contrast_mean(img)), img, v)


def smooth3x3(img):
    """ImageFilter.SMOOTH: [1 1 1; 1 5 1; 1 1 1] / 13, round half up, 1-pixel
    border copied; images thinner than 3 px are returned unchanged (Filter.c)."""
    h, w = img.shape[:2]
    out = img.copy()
    if h < 3 or w < 3:
        return out
    p = img.astype(np.int64)
    s = np.zeros((h - 2, w - 2, 3), dtype=np.int64)
    for dy in range(3):
        for dx in range(3):
            s += p[dy:dy + h - 2, dx:dx + w - 2]
    s += 4 * p[1:h - 1, 1:w - 1]
    out[1:h - 1, 1:w - 1] = ((2 * s + 13) // 26).astype(U8)
    return out


def sharpness(img, v):      # augmentations.py:112-114
    return blend(smooth3x3(img), img, v)


def point(img, lut3x256):
    """``Image.point`` with a 768-entry table; entries are clipped to 255."""
    lut = np.clip(np.asarray(lut3x256, dtype=np.int64).reshape(3, 256), 0, 255).astype(U8)
    out = np.empty_like(img)
    for c in range(3):
        out[..., c] = lut[c][img[..., c]]
    return out


def histogram3(img):
    return np.stack([np.bincount(img[..., c].ravel(), minlength=256) for c in range(3)])


def autocontrast_lut(hist256):
    """ImageOps.autocontrast(cutoff=0), one channel; float64, separate multiply
    and add, truncation toward zero (Python ``int``), then clamp."""
    nz = np.nonzero(hist256)[0]
    if len(nz) == 0:
        return list(range(256))
    lo, hi = int(nz[0]), int(nz[-1])
    if hi <= lo:
        return list(range(256))
    scale = 255.0 / (hi - lo)
    offset = -lo * scale
    lut = []
    for ix in range(256):
        t = int(ix * scale + offset)
        lut.append(0 if t < 0 else 255 if t > 255 else t)
    return lut


def autocontrast(img):      # augmentations.py:64-65
    hh = histogram3(img)
    lut = []
    for c in range(3):
        lut += autocontrast_lut(hh[c])
    return point(img, lut)


def equalize_lut(hist256):
    """ImageOps.equalize, one channel."""
    h = [int(t) for t in hist256]
    nonzero = [t for t in h if t]
    if len(nonzero) <= 1:
        return list(range(256))
    step = (sum(nonzero) - nonzero[-1]) // 255
    if not step:
        return list(range(256))
    n = step // 2
    lut = []
    for i in range(256):
        lut.append(n // step)
        n += h[i]
    return lut


def equalize(img):          # augmentations.py:72-73
    hh = histogram3(img)
    lut = []
    for c in range(3):
        lut += equalize_lut(hh[c])
    return point(img, lut)


def invert(img):            # augmentations.py:68-69
    return (255 - img).astype(U8)


def solarize(img, v: float):    # augmentations.py:80-82; ``i < v`` with float v
    thr = math.ceil(v)
    return np.where(img < thr, img, 255 - img).astype(U8)


def posterize(img, v: float):   # augmentations.py:85-94 (Posterize and Posterize2)
    bits = int(v)
    mask = ~(2 ** (8 - bits) - 1) & 0xFF
    return (img & U8(mask)).astype(U8)


def cutout_box(w, h, v_px: float, ux: float, uy: float):
    """CutoutAbs' box from the two uniforms u in [0,1) that numpy's legacy
    ``uniform(low=w, high=1.0)`` turns into ``w + (1.0 - w)*u``
    (augmentations.py:130-137).  Returns the *inclusive* integer box that
    ImageDraw.rectangle paints, before clipping to the image."""
    cx = w + (1.0 - w) * ux
    cy = h + (1.0 - h) * uy
    left = int(max(0, cx - v_px / 2.0))
    top = int(max(0, cy - v_px / 2.0))
    right = min(w, left + v_px)
    bottom = min(h, top + v_px)
    return left, top, int(right), int(bottom)


def cutout_abs(img, v_px, ux, uy):      # augmentations.py:126-144
    if v_px < 0:
        return img.copy()
    h, w = img.shape[:2]
    x0, y0, x1, y1 = cutout_box(w, h, v_px, ux, uy)
    out = img.copy()
    out[max(y0, 0):min(y1, h - 1) + 1, max(x0, 0):min(x1, w - 1) + 1] = CUTOUT_RGB
    return out


# ------------------------------------------------ one op with explicit draws --
MIRRORED = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate",
            "TranslateXAbs", "TranslateYAbs")
NEEDS_BOX = ("Cutout", "CutoutAbs")


def run_op_resolved(img, name, v, mirror=False, ux=0.0, uy=0.0):
    """One op at magnitude ``v`` with its random draws already resolved."""
    h, w = img.shape[:2]
    if name in MIRRORED and mirror:
        v = -v
    if name == "ShearX":
        return affine_nearest(img, (1, v, 0, 0, 1, 0))
    if name == "ShearY":
        return affine_nearest(img, (1, 0, 0, v, 1, 0))
    if name == "TranslateX":
        return affine_nearest(img, (1, 0, v * w, 0, 1, 0))
    if name == "TranslateY":
        return affine_nearest(img, (1, 0, 0, 0, 1, v * h))
    if name == "TranslateXAbs":
        return affine_nearest(img, (1, 0, v, 0, 1, 0))
    if name == "TranslateYAbs":
        return affine_nearest(img, (1, 0, 0, 0, 1, v))
    if name == "Rotate":
        return rotate(img, v)
    if name == "AutoContrast":
        return autocontrast(img)
    if name == "Invert":
        return invert(img)
    if name == "Equalize":
        return equalize(img)
    if name == "Solarize":
        return solarize(img, v)
    if name in ("Posterize", "Posterize2"):
        return posterize(img, v)
    if name == "Contrast":
        return contrast(img, v)
    if name == "Color":
        return color(img, v)
    if name == "Brightness":
        return brightness(img, v)
    if name == "Sharpness":
        return sharpness(img, v)
    if name == "Cutout":
        if v <= 0.0:
            return img.copy()
        return cutout_abs(img, v * w, ux, uy)
    if name == "CutoutAbs":
        return cutout_abs(img, v, ux, uy)
    raise KeyError(name)


def policy_call(img, policies):
    """``Augmentation.__call__`` (data.py:257-264) on the NumPy model, consuming
    the *global* Python/NumPy RNGs in the reference's order."""
    chosen = random.choice(policies)
    for name, pr, level in chosen:
        if random.random() > pr:
            continue
        v = magnitude(name, level)
        mirror, ux, uy = False, 0.0, 0.0
        if name in MIRRORED:
            mirror = random.random() > 0.5
        elif name in NEEDS_BOX and not (name == "Cutout" and v <= 0.0) and not (name == "CutoutAbs" and v < 0):
            ux = np.random.random_sample()      # == the u inside legacy uniform()
            uy = np.random.random_sample()
        img = run_op_resolved(img, name, v, mirror, ux, uy)
    return img


# --------------------------------------------------------------------- tail --
def pad_crop(img, pad, top, left, out_h, out_w):
    """torchvision RandomCrop(size, padding=pad) with resolved (top, left)
    (data.py:40)."""
    padded = np.zeros((img.shape[0] + 2 * pad, img.shape[1] + 2 * pad, 3), U8)
    padded[pad:pad + img.shape[0], pad:pad + img.shape[1]] = img
    return padded[top:top + out_h, left:left + out_w].copy()


def hflip(img):
    return img[:, ::-1].copy()


def to_tensor_normalize(img, mean, std):
    """ToTensor + Normalize (data.py:42-43): fp32 ``u8/255`` then
    ``(x-mean)/std`` with fp32 mean/std; HWC -> CHW."""
    x = img.astype(F32) / F32(255)
    x = (x - np.asarray(mean, F32)) / np.asarray(std, F32)
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def zero_box(chw, length, cy, cx):
    """CutoutDefault with resolved centre (data.py:235-250)."""
    h, w = chw.shape[1:]
    half = length // 2
    ya, yb = np.clip(cy - half, 0, h), np.clip(cy + half, 0, h)
    xa, xb = np.clip(cx - half, 0, w), np.clip(cx + half, 0, w)
    out = chw.copy()
    out[:, ya:yb, xa:xb] = 0.0
    return out


def mixup_resolved(data_f32, order, lam: float):
    """aug_mixup.py:21: ``data*lam + data[order]*(1-lam)`` with the Python-float
    scalars cast to fp32 and every product / sum rounded to fp32."""
    l0, l1 = F32(lam), F32(1 - lam)
    return (data_f32 * l0 + data_f32[order] * l1).astype(F32)
