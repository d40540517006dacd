"""NumPy model of the ImageNet chains' geometry, written from the arithmetic, for the tests.

* ``coeffs`` / ``resize``: Pillow ``Image.resize(size, BICUBIC)`` on 8-bit RGB (``ImagingResample``):
  fp64 bicubic weights (a = -0.5) per output index, normalised, converted to 22-bit fixed point;
  a horizontal pass into a uint8 intermediate, then a vertical pass; an axis that keeps its size
  is not resampled.
* ``center_box`` / ``RandomCropModel``: ``EfficientNetCenterCrop`` / ``EfficientNetRandomCrop``
  (reference data.py:267-345) as boxes (x0, y0, w, h), with ``Image.crop``'s ``int(round())`` of the box.
"""
from __future__ import annotations

import math
import random

import numpy as np

PRECISION_BITS = 22


def _bicubic(x):
    x = np.abs(x)
    a = -0.5
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def coeffs(n_in, n_out):
    """(xmin [n_out], n [n_out], k int32 [n_out][ksize]) of precompute_coeffs + normalize_coeffs_8bpc."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(n_out) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)          # (int) truncates toward zero
    cnt = np.minimum((center + support + 0.5).astype(np.int64), n_in) - xmin
    x = np.arange(ksize)
    w = _bicubic(((x[None, :] + xmin[:, None]) - center[:, None] + 0.5) * (1.0 / fs))
    w = np.where(x[None, :] < cnt[:, None], w, 0.0)
    ww = np.zeros(n_out)
    for t in range(ksize):                            # summed left to right, like the C loop
        ww = ww + w[:, t]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    f = w * (1 << PRECISION_BITS)
    k = np.where(w < 0, f - 0.5, f + 0.5).astype(np.int64).astype(np.int32)
    return xmin, cnt, k


def _pass(img, n_out, axis):
    """one 8-bit pass along `axis` (1 = horizontal, 0 = vertical) of a uint8 [H][W][3] image"""
    n_in = img.shape[axis]
    if n_in == n_out:
        return img
    xmin, cnt, k = coeffs(n_in, n_out)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((n_out,) + src.shape[1:], np.uint8)
    for xx in range(n_out):
        taps = src[xmin[xx]:xmin[xx] + cnt[xx]]
        s = (1 << (PRECISION_BITS - 1)) + np.tensordot(k[xx, :cnt[xx]].astype(np.int64), taps, axes=(0, 0))
        out[xx] = np.clip(s >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def resize(img, out_h, out_w):
    """uint8 [H][W][3] -> uint8 [out_h][out_w][3] like PIL ``resize((out_w, out_h), BICUBIC)``."""
    return np.ascontiguousarray(_pass(_pass(np.asarray(img), out_w, 1), out_h, 0))


def crop_resize(img, box, out_h, out_w):
    x0, y0, w, h = (int(v) for v in box)
    return resize(np.asarray(img)[y0:y0 + h, x0:x0 + w], out_h, out_w)


def center_box(h, w, imgsize):
    """EfficientNetCenterCrop box (x0, y0, w, h) of an h x w image"""
    c = float(imgsize) / (imgsize + 32) * min(w, h)
    top, left = int(round((h - c) / 2.)), int(round((w - c) / 2.))
    return left, top, int(round(left + c)) - left, int(round(top + c)) - top


class RandomCropModel:
    """EfficientNetRandomCrop's box draw from Python's ``random`` (same calls, same order)."""

    def __init__(self, imgsize, min_covered=0.1, aspect_ratio_range=(3. / 4, 4. / 3), area_range=(0.08, 1.0),
                 max_attempts=10):
        self.imgsize, self.min_covered = imgsize, min_covered
        self.aspect_ratio_range, self.area_range, self.max_attempts = aspect_ratio_range, area_range, max_attempts

    def box(self, h, w):
        W, H = w, h
        min_area, max_area = self.area_range[0] * (W * H), self.area_range[1] * (W * H)
        for _ in range(self.max_attempts):
            ar = random.uniform(*self.aspect_ratio_range)
            height = int(round(math.sqrt(min_area / ar)))
            max_height = int(round(math.sqrt(max_area / ar)))
            if max_height * ar > W:
                max_height = int((W + 0.5 - 1e-7) / ar)
                if max_height * ar > W:
                    max_height -= 1
            max_height = min(max_height, H)
            height = min(height, max_height)
            height = int(round(random.uniform(height, max_height)))
            width = int(round(height * ar))
            area = width * height
            if area < min_area or area > max_area or width > W or height > H or area < self.min_covered * (W * H):
                continue
            if width == W and height == H:
                break
            x = random.randint(0, W - width)
            y = random.randint(0, H - height)
            return x, y, width, height
        return center_box(h, w, self.imgsize)
