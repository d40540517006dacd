"""EfficientNet crops + Pillow bicubic resize on a CPU-only box: the NumPy model against Pillow, the kernel's
arithmetic (faa_core.cuh through the host build tests/emu/faa_emu_resize.cpp) against the model, and the crop samplers
against boxes recorded from the reference."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import PIL.Image
import pytest
from scipy import stats

import resize_model as M
from helpers import ROOT

from fast_autoaugment_b200 import _lib, data, engine

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_resize.npz")
OUT_SIZES = (32, 224, 240, 260, 300, 380, 456, 528, 600)


def load_emu_resize():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_resize.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_resize.cpp")
    core = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(core)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    lib.faa_emu_resize_ksize.argtypes = [i, i]
    lib.faa_emu_resize_coeffs.argtypes = [i, i, vp, vp, i]
    lib.faa_emu_crop_resize.argtypes = [vp, i, i, vp, i, i, vp]
    lib.faa_emu_center_crop_box.argtypes = [i, i, i, vp]
    lib.faa_emu_crop_attempt.argtypes = [vp, i, i, d, d, vp]
    lib.faa_emu_philox_crop_boxes.argtypes = [vp, i, i, i, vp]
    return lib


@pytest.fixture(scope="module")
def emu_rs():
    return load_emu_resize()


def emu_crop_resize(lib, img, box, oh, ow):
    img = np.ascontiguousarray(img)
    b = np.array(box, np.int32)
    out = np.zeros((oh, ow, 3), np.uint8)
    lib.faa_emu_crop_resize(img.ctypes.data, img.shape[0], img.shape[1], b.ctypes.data, oh, ow, out.ctypes.data)
    return out


def emu_philox_boxes(lib, cfg, n, h, w):
    out = np.zeros(n, dtype=_lib.CROP_BOX_DTYPE)
    lib.faa_emu_philox_crop_boxes(C.addressof(cfg), n, h, w, out.ctypes.data)
    return out


def image(kind, h, w, rng):
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "ramp":
        return np.clip(np.linspace(0, 255, w)[None, :, None] + np.linspace(-40, 40, h)[:, None, None]
                       + rng.normal(0, 10, (h, w, 3)), 0, 255).astype(np.uint8)
    return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()


GRID = [((256, 256), (224, 224)), ((375, 500), (224, 224)), ((80, 100), (224, 224)), ((517, 333), (380, 380)),
        ((900, 1200), (224, 224)), ((37, 41), (32, 32)), ((224, 300), (224, 224)), ((300, 224), (224, 224)),
        ((224, 224), (224, 224)), ((60, 50), (1, 1)), ((7, 9), (1, 3)), ((2100, 48), (224, 224)),
        ((40, 2300), (224, 40)), ((2048, 2048), (224, 224)), ((1, 1), (5, 7)), ((3, 600), (600, 3))]


@pytest.mark.parametrize("kind", ["noise", "ramp", "constant"])
def test_model_equals_pillow_bicubic(kind):
    rng = np.random.default_rng(hash(kind) & 0xFFFF)
    bad = total = 0
    for (h, w), (oh, ow) in GRID:
        img = image(kind, h, w, rng)
        want = np.asarray(PIL.Image.fromarray(img).resize((ow, oh), PIL.Image.BICUBIC))
        got = M.resize(img, oh, ow)
        assert got.shape == want.shape
        bad += int((got != want).sum())
        total += got.size
    assert bad == 0 and total > 0


def test_core_coefficients_equal_model(emu_rs):
    for n_out in OUT_SIZES:
        for n_in in range(1, 601):
            xmin, cnt, k = M.coeffs(n_in, n_out)
            ks = emu_rs.faa_emu_resize_ksize(n_in, n_out)
            if n_in == n_out:
                continue                      # identity axis: one tap of weight 1 << 22 (checked below)
            assert ks == k.shape[1], (n_in, n_out)
            b = np.zeros((n_out, 2), np.int32)
            kk = np.zeros((n_out, ks), np.int32)
            emu_rs.faa_emu_resize_coeffs(n_in, n_out, b.ctypes.data, kk.ctypes.data, ks)
            assert np.array_equal(b[:, 0], xmin) and np.array_equal(b[:, 1], cnt), (n_in, n_out)
            assert np.array_equal(kk, k), (n_in, n_out)
    b = np.zeros((224, 2), np.int32)
    kk = np.zeros((224, 5), np.int32)
    emu_rs.faa_emu_resize_coeffs(224, 224, b.ctypes.data, kk.ctypes.data, 5)
    assert np.array_equal(b[:, 0], np.arange(224)) and (b[:, 1] == 1).all() and (kk[:, 0] == 1 << 22).all()


def test_emulated_crop_resize_equals_model(emu_rs):
    rng = np.random.default_rng(7)
    cases = [((375, 500), (10, 20, 330, 300), (224, 224)), ((256, 256), (16, 16, 224, 224), (224, 224)),
             ((48, 64), (3, 5, 40, 30), (224, 224)), ((333, 500), (0, 0, 500, 333), (380, 380)),
             ((300, 301), (1, 2, 299, 224), (224, 224)), ((1536, 2048), (100, 50, 1900, 1400), (224, 224)),
             ((600, 600), (0, 0, 600, 600), (1, 1))]
    for (h, w), box, (oh, ow) in cases:
        img = image("noise", h, w, rng)
        want = M.crop_resize(img, box, oh, ow)
        x0, y0, bw, bh = box
        pil = np.asarray(PIL.Image.fromarray(img).crop((x0, y0, x0 + bw, y0 + bh)).resize((ow, oh), PIL.Image.BICUBIC))
        assert np.array_equal(want, pil)
        assert np.array_equal(emu_crop_resize(emu_rs, img, box, oh, ow), want), (h, w, box)


def test_center_boxes_match_reference_formula(emu_rs):
    ties = 0
    for s in (224, 240, 380, 600):
        for h in range(1, 700, 7):
            for w in range(1, 700, 11):
                want = M.center_box(h, w, s)
                c = float(s) / (s + 32) * min(w, h)
                ties += ((h - c) / 2.) % 1 == 0.5 or ((w - c) / 2.) % 1 == 0.5 or (round(c + 0.0) != c and (c % 1) == 0.5)
                assert engine.center_crop_box(h, w, s) == want, (h, w, s)
                b = np.zeros(1, _lib.CROP_BOX_DTYPE)
                emu_rs.faa_emu_center_crop_box(h, w, s, b.ctypes.data)
                assert tuple(int(v) for v in b[0]) == want
    # half-way cases of the rounding: W - c odd with c integral (256 -> 224 at s = 224: c = 224 exactly)
    assert engine.center_crop_box(256, 257, 224) == M.center_box(256, 257, 224)
    assert ties > 0


def test_center_crop_dropin_equals_pil_crop():
    img = PIL.Image.fromarray(np.random.default_rng(1).integers(0, 256, (375, 500, 3), dtype=np.uint8))
    c = data.EfficientNetCenterCrop(224)
    x0, y0, w, h = M.center_box(375, 500, 224)
    assert np.array_equal(np.asarray(c(img)), np.asarray(img.crop((x0, y0, x0 + w, y0 + h))))


def test_parity_crop_sampler_reproduces_reference_boxes():
    g = np.load(GOLDEN)
    n_fallback = 0
    for key in (k for k in g.files if k.startswith("boxes_")):
        s, hw = key.split("_")[1:]
        h, w = (int(v) for v in hw.split("x"))
        crop = data.EfficientNetRandomCrop(int(s))
        model = M.RandomCropModel(int(s))
        center = M.center_box(h, w, int(s))
        for i, want in enumerate(g[key]):
            random.seed(i)
            got = crop.sample_parity(1, h, w)[0]
            after = random.random()
            assert tuple(int(v) for v in got) == tuple(int(v) for v in want), (key, i)
            random.seed(i)
            assert model.box(h, w) == tuple(int(v) for v in want)
            assert random.random() == after                 # the same number of draws
            n_fallback += tuple(int(v) for v in want) == center
    assert n_fallback > 0                                   # (the tiny sources fall back often)


def test_python_dropin_consumes_random_like_reference():
    img = PIL.Image.fromarray(np.random.default_rng(2).integers(0, 256, (375, 500, 3), dtype=np.uint8))
    crop = data.EfficientNetRandomCrop(224)
    random.seed(5)
    a = [np.asarray(crop(img)) for _ in range(20)]
    random.seed(5)
    boxes = crop.sample_parity(20, 375, 500)
    for arr, b in zip(a, boxes):
        x0, y0, w, h = (int(v) for v in b)
        assert np.array_equal(arr, np.asarray(img)[y0:y0 + h, x0:x0 + w])


@pytest.mark.parametrize("s,h,w", [(224, 375, 500), (224, 256, 256), (380, 500, 375), (224, 1536, 2048)])
def test_philox_boxes_valid_and_distributed_like_reference(emu_rs, s, h, w):
    n = 6000
    cfg = engine.crop_cfg(s, seed=11, first_index=1000)
    ph = emu_philox_boxes(emu_rs, cfg, n, h, w)
    center = M.center_box(h, w, s)
    ok = np.array([tuple(int(v) for v in b) != center for b in ph])
    b = ph[ok]
    area, ar = b["w"].astype(float) * b["h"], b["w"].astype(float) / b["h"]
    assert (b["x0"] >= 0).all() and (b["y0"] >= 0).all() and (b["x0"] + b["w"] <= w).all() and (b["y0"] + b["h"] <= h).all()
    assert (area >= 0.08 * w * h).all() and (area <= w * h).all()
    assert (ar > 0.74).all() and (ar < 1.35).all()            # 3/4 .. 4/3 before the rounding of width and height
    # same key -> same boxes; another first_index -> other boxes
    assert np.array_equal(emu_philox_boxes(emu_rs, cfg, 64, h, w), ph[:64])
    assert not np.array_equal(emu_philox_boxes(emu_rs, engine.crop_cfg(s, seed=11, first_index=1001), 64, h, w), ph[:64])
    random.seed(0)
    par = data.EfficientNetRandomCrop(s).sample_parity(n, h, w)

    def hist(bx):
        fa = bx["w"].astype(float) * bx["h"] / (w * h)
        fx = (bx["x0"] + bx["w"] / 2) / w
        return (np.histogram(fa, bins=8, range=(0, 1.0001))[0], np.histogram(fx, bins=8, range=(0, 1))[0])
    for hp, hr in zip(hist(ph), hist(par)):
        keep = (hp + hr) > 0
        p = stats.chi2_contingency(np.stack([hp[keep], hr[keep]]))[1]
        assert p > 1e-4, (hp, hr, p)


def test_philox_attempt_matches_python_arithmetic(emu_rs):
    """crop_attempt from given uniforms == the reference's arithmetic on the same uniforms"""
    cfg = engine.crop_cfg(224)
    rng = np.random.default_rng(3)
    wh = np.zeros(2, np.int32)
    for h, w in ((375, 500), (48, 64), (2048, 1536), (1, 1), (3, 800)):
        for _ in range(300):
            ua, uh = rng.random(), rng.random()
            seq = iter([ua, uh])
            random._inst.random = lambda: next(seq)          # (random.uniform draws through the instance)
            try:
                res = M.RandomCropModel(224, max_attempts=1).box(h, w)
            finally:
                del random._inst.random
            r = emu_rs.faa_emu_crop_attempt(C.addressof(cfg), h, w, ua, uh, wh.ctypes.data)
            if r == 1:
                assert (res[2], res[3]) == (int(wh[0]), int(wh[1]))
            else:
                assert res == M.center_box(h, w, 224)


def test_crop_resize_abi_refuses_bad_arguments():
    cfg = engine.crop_cfg(224)
    t = engine.TailSpec.raw_u8().c_struct(10, 10)
    assert _lib.lib.faa_crop_resize(None, None, 1, 10, 10, C.byref(t), None, C.byref(cfg), None) == _lib.ERR_VALUE
    assert _lib.lib.faa_crop_resize(None, None, 0, 0, 10, C.byref(t), None, C.byref(cfg), None) == _lib.ERR_VALUE
    assert _lib.lib.faa_crop_resize(None, None, 0, 10, 8193, C.byref(t), None, C.byref(cfg), None) == _lib.ERR_VALUE
    bad = engine.crop_cfg(224, aspect_ratio_range=(2.0, 1.0))
    assert _lib.lib.faa_crop_resize(None, None, 0, 10, 10, C.byref(t), None, C.byref(bad), None) == _lib.ERR_MAGNITUDE
    with pytest.raises(ValueError):
        engine.center_crop_box(0, 10, 224)
