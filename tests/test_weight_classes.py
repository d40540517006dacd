"""The three-way split never launches the cluster kernel for the headline geometry (faa_cabi.cu: `no_heavy`), so the
program builder must sort EVERY program into the light or the mid kernel there - a heavy program would simply not be
written.  Checked on the host through the emulation build of faa_core.cuh (the same source the resolve kernel compiles):
every single op and every ordered op pair, every gate / sign combination, with and without Cutout boxes and flips - at
every image size of tests/geometry_cases.py where the planner sets `no_heavy` (compiled records depend on the size)."""
import ctypes as C
import itertools
import random

import numpy as np
import pytest

import geometry_cases as G
from helpers import ALL_OPS

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.engine import CompiledPolicy


def _classes(emu, pol, samples, boxes, H, W, allow):
    emu.faa_emu_weight_classes.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    emu.faa_emu_weight_classes.restype = C.c_int
    table = np.ascontiguousarray(pol.compiled_table(H, W))
    n = len(samples)
    wc, cls = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    s, b = np.ascontiguousarray(samples), np.ascontiguousarray(boxes)
    assert emu.faa_emu_weight_classes(table.ctypes.data, pol.n_op, s.ctypes.data, b.ctypes.data, n, H, W, W, 1, allow,
                                      wc.ctypes.data, cls.ctypes.data) == 0
    return wc, cls


# the image sizes of tests/geometry_cases.py where the planner sets `no_heavy`, besides the headline 224 x 224
_LEAN_SHAPES = sorted({c.shape for c in G.CASES
                       if G.plan(*c.shape, 64, in_off=c.in_off, out_off=c.out_off, split_min=0).no_heavy})


def _check_lean(emu, H, W):
    rng = random.Random(5)
    policies = [[(a, 1.0, rng.random()), (b, 1.0, rng.random())] for a in ALL_OPS for b in ALL_OPS]
    pol = CompiledPolicy(policies)
    rows = []
    for sub, (gate, sign, flip) in itertools.product(range(len(policies)), itertools.product((0, 1, 2, 3), (0, 1, 2, 3), (0, 1))):
        rows.append((sub, gate, sign, flip))
    n = len(rows)
    samples = np.zeros(n, dtype=_lib.SAMPLE_DTYPE)
    boxes = np.zeros((n, 2), dtype=_lib.BOX_DTYPE)
    for i, (sub, gate, sign, flip) in enumerate(rows):
        samples[i]["sub"], samples[i]["gate"], samples[i]["sign"], samples[i]["flip"] = sub, gate, sign, flip
        boxes[i]["x0"], boxes[i]["y0"], boxes[i]["x1"], boxes[i]["y1"] = 10 + i % 50, 20 + i % 70, 60 + i % 90, 100 + i % 60
    wc, cls = _classes(emu, pol, samples, boxes, H, W, allow=7)          # chunk + scratch + lean gathers: the headline launch
    heavy = [(policies[rows[i][0]], rows[i][1:], int(cls[i])) for i in range(n) if wc[i] == 0]
    assert not heavy, ((H, W), len(heavy), heavy[:5])
    assert (wc == 2).any() and (wc == 1).any()
    # sanity of the probe itself: without the lean gathers (bit 2) or without the scratch image (bit 1) some programs stay heavy
    wc3, _ = _classes(emu, pol, samples, boxes, H, W, allow=3)
    wc5, _ = _classes(emu, pol, samples, boxes, H, W, allow=5)
    assert (wc3 == 0).any() and (wc5 == 0).any()


def test_every_program_is_light_or_mid_in_a_lean_launch(emu):
    _check_lean(emu, 224, 224)


def test_the_lean_shapes_are_the_no_heavy_cases():
    assert len(_LEAN_SHAPES) >= 8 and (8192, 8) in _LEAN_SHAPES and (600, 600) in _LEAN_SHAPES
    for shape in [(224, 224)] + _LEAN_SHAPES:
        p = G.plan(*shape, 512 if shape == (224, 224) else 64, split_min=0)
        assert p.no_heavy and p.allow == 7, (shape, p)


@pytest.mark.parametrize("shape", _LEAN_SHAPES, ids=lambda s: "%dx%d" % s)
def test_every_program_is_light_or_mid_at_every_lean_size(emu, shape):
    """compiled records depend on the image size (Rotate, translations, Cutout): the same proof at every size where the
    planner does not launch the cluster kernel"""
    _check_lean(emu, *shape)


def test_archive_policies_have_no_heavy_program(emu):
    from fast_autoaugment_b200 import archive
    for name in ("fa_resnet50_rimagenet", "fa_reduced_cifar10", "fa_reduced_svhn"):
        policies = getattr(archive, name)()
        pol = CompiledPolicy(policies)
        rows = list(itertools.product(range(len(policies)), (0, 1, 2, 3), (0, 1, 2, 3)))
        samples = np.zeros(len(rows), dtype=_lib.SAMPLE_DTYPE)
        boxes = np.zeros((len(rows), pol.n_op), dtype=_lib.BOX_DTYPE)
        boxes["x1"], boxes["y1"] = 40, 50
        for i, (sub, gate, sign) in enumerate(rows):
            samples[i]["sub"], samples[i]["gate"], samples[i]["sign"], samples[i]["flip"] = sub, gate, sign, i & 1
        wc, cls = _classes(emu, pol, samples, boxes, 224, 224, allow=7)
        assert (wc != 0).all(), (name, [policies[rows[i][0]] for i in np.nonzero(wc == 0)[0][:5]])
