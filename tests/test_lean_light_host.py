"""The lean light launch (LaunchPlan::lean_light, allow bit 3), checked on the host through the emulation build of
faa_core.cuh - the same predicates the resolve kernel compiles.

The lean variant of the light kernel has the octet paths only (no generic evaluators: 64 registers, four CTAs per SM).
So in a lean launch every program must either be light AND one of the programs those paths take, or run in the mid
kernel; the cluster kernel is not launched at 224 x 224.  The programs the octet paths cannot finish (a LUT, Color,
Cutout or a gather followed by Color / Cutout) move to the mid kernel's two-stage path; Color in front of a gather
is rebuilt as the gather, then Color.  Launches without the bit classify every program exactly as before."""
import ctypes as C
import hashlib
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import geometry_cases as G
from helpers import ALL_OPS

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.engine import CompiledPolicy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_NONE, K_AFFINE, K_SHIFT, K_LUT, K_AUTOCONTRAST, K_EQUALIZE, K_BRIGHTNESS, K_COLOR, K_CONTRAST, K_SHARPNESS, K_CUTOUT = range(11)
C_PLAIN, C_LUT, C_POINT, C_GENERIC, C_SHARP, C_MAT, C_GEOM, C_SG, C_GEOM2 = range(9)
GATHER = (K_AFFINE, K_SHIFT)
STATIC_LUT = (K_LUT, K_BRIGHTNESS)

# sha256 of the (weight class, program class) bytes of _pairs() at 224 x 224 for allow = 0..7, computed with the
# program builder before the lean light launch existed
_BEFORE = "7aace35d1c329719c0d71b35c1a12d5355b69b1d3de92ef189e34ad8ee32878b"


@pytest.fixture(scope="module")
def lean_emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_lean.cpp")
    so = str(tmp_path_factory.mktemp("emu_lean") / "libfaa_emu_lean.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.faa_emu_lean_classes.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    lib.faa_emu_lean_plan.argtypes = [C.c_int] * 7 + [vp]
    return lib


def _pairs():
    """every ordered pair of the policy ops, every gate / sign combination, with and without a flip, Cutout boxes"""
    rng = random.Random(5)
    policies = [[(a, 1.0, rng.random()), (b, 1.0, rng.random())] for a in ALL_OPS for b in ALL_OPS]
    rows = list(itertools.product(range(len(policies)), (0, 1, 2, 3), (0, 1, 2, 3), (0, 1)))
    samples = np.zeros(len(rows), dtype=_lib.SAMPLE_DTYPE)
    boxes = np.zeros((len(rows), 2), dtype=_lib.BOX_DTYPE)
    for i, (sub, gate, sign, flip) in enumerate(rows):
        samples[i]["sub"], samples[i]["gate"], samples[i]["sign"], samples[i]["flip"] = sub, gate, sign, flip
        boxes[i]["x0"], boxes[i]["y0"], boxes[i]["x1"], boxes[i]["y1"] = 10 + i % 50, 20 + i % 70, 60 + i % 90, 100 + i % 60
    return policies, rows, samples, boxes


def _classes(lib, policies, samples, boxes, H, W, allow):
    """[n, 5]: weight class, program class, op kinds of slots 0 and 1, prog_two_stage"""
    pol = CompiledPolicy(policies)
    table = np.ascontiguousarray(pol.compiled_table(H, W))
    out = np.zeros((len(samples), 5), dtype=np.uint8)
    assert lib.faa_emu_lean_classes(table.ctypes.data, pol.n_op, samples.ctypes.data, boxes.ctypes.data, len(samples), H, W,
                                    allow, out.ctypes.data) == 0
    return out


def _plan(lib, H, W, batch=512, out_u8=False, out_mod16=0, crop_pad=0, philox=True):
    out = (C.c_int32 * 6)()
    assert lib.faa_emu_lean_plan(H, W, batch, int(out_u8), out_mod16, crop_pad, int(philox), out) == 6
    return dict(zip(("allow", "lean_light", "light_bands", "light_staged", "use_mid", "no_heavy"), out))


def _octet_path(cls, k0, k1):
    """does the lean light kernel have an octet path for this program (faa_augment_light_kernel<OUT, TAB, true>)?"""
    if cls in (C_PLAIN, C_LUT, C_GEOM2):
        return True
    if cls == C_POINT:          # Color / Cutout alone, or followed by a static LUT (the float table)
        return k0 in (K_COLOR, K_CUTOUT) and (k1 == K_NONE or k1 in STATIC_LUT)
    if cls == C_GEOM:           # a gather with a static LUT on either side or none; Cutout, then the gather
        g0 = k0 in GATHER
        pk = k1 if g0 else k0
        return pk == K_NONE or pk in STATIC_LUT or (not g0 and pk == K_CUTOUT)
    return False


def test_every_program_of_a_lean_launch_is_octet_light_or_mid(lean_emu):
    policies, rows, samples, boxes = _pairs()
    p = _plan(lean_emu, 224, 224)
    assert p["lean_light"] and p["allow"] == 15 and p["no_heavy"]
    c = _classes(lean_emu, policies, samples, boxes, 224, 224, p["allow"])
    bad = [(policies[rows[i][0]], rows[i][1:], c[i].tolist()) for i in range(len(rows))
           if c[i, 0] == 0 or (c[i, 0] == 2 and not _octet_path(*c[i, 1:4]))]
    assert not bad, (len(bad), bad[:5])
    # what moved: light without the bit, mid with it - every one a two-stage program of the mid kernel
    old = _classes(lean_emu, policies, samples, boxes, 224, 224, 7)
    moved = (old[:, 0] == 2) & (c[:, 0] != 2)
    assert moved.any() and (c[moved, 0] == 1).all() and (c[moved, 4] == 1).all()
    assert set(map(tuple, c[moved, 1:4].tolist())) <= {(cls, k0, k1) for cls in (C_POINT, C_GEOM)
                                                        for k0 in (K_AFFINE, K_SHIFT, K_LUT, K_BRIGHTNESS, K_COLOR, K_CUTOUT)
                                                        for k1 in (K_COLOR, K_CUTOUT)}
    # ... and the light programs the lean paths gained: Color / Cutout, then a static LUT; Cutout, then a gather
    for a, b in (("Color", "Posterize"), ("Cutout", "Invert"), ("CutoutAbs", "Rotate"), ("Cutout", "TranslateX")):
        i = rows.index((policies.index(next(q for q in policies if q[0][0] == a and q[1][0] == b)), 3, 0, 0))
        assert c[i, 0] == 2 and c[i, 1] in (C_POINT, C_GEOM), (a, b, c[i].tolist())


def test_color_in_front_of_a_gather_becomes_the_gather_then_color(lean_emu):
    policies, rows, samples, boxes = _pairs()
    lean, old = _classes(lean_emu, policies, samples, boxes, 224, 224, 15), _classes(lean_emu, policies, samples, boxes, 224, 224, 7)
    sel = (old[:, 1] == C_GEOM) & (old[:, 2] == K_COLOR) & np.isin(old[:, 3], GATHER)
    assert sel.sum() > 0
    assert (lean[sel, 2] == old[sel, 3]).all() and (lean[sel, 3] == K_COLOR).all() and (lean[sel, 0] == 1).all()
    assert (lean[~sel, 2:4] == old[~sel, 2:4]).all()


def test_launches_without_the_bit_classify_as_before(lean_emu):
    policies, rows, samples, boxes = _pairs()
    h = hashlib.sha256()
    for allow in range(8):
        c = _classes(lean_emu, policies, samples, boxes, 224, 224, allow)
        h.update(np.ascontiguousarray(c[:, :2]).tobytes())
    assert h.hexdigest() == _BEFORE


@pytest.mark.parametrize("shape", [(224, 224)] + sorted({c.shape for c in G.CASES}), ids=lambda s: "%dx%d" % s)
def test_the_planner_picks_the_lean_kernel_exactly_in_the_octet_regime(lean_emu, shape):
    H, W = shape
    for out_u8, out_mod16, crop_pad, philox in itertools.product((False, True), (0, 8), (0, 4), (False, True)):
        p = _plan(lean_emu, H, W, out_u8=out_u8, out_mod16=out_mod16, crop_pad=crop_pad, philox=philox)
        octets = bool(p["allow"] & 4) and p["light_staged"]
        assert bool(p["lean_light"]) == (octets and philox), (shape, out_u8, out_mod16, crop_pad, philox, p)
        assert bool(p["allow"] & 8) == bool(p["lean_light"])
        if p["lean_light"]:
            assert p["use_mid"] and W % 8 == 0 and crop_pad == 0 and out_mod16 == 0


def test_rows_and_ctas_of_the_flagship_step(lean_emu):
    """the chained step launches one resident wave of light rows: sm_count * CTAs per SM / bands (faa_cabi.cu
    launch_chained); the lean kernel's launch bounds give 4 CTAs per SM instead of 3"""
    p = _plan(lean_emu, 224, 224)
    assert p["lean_light"] and p["light_bands"] == 7
    rows = 132 * 4 // p["light_bands"]
    assert (rows, rows * p["light_bands"]) == (75, 525)
    assert not _plan(lean_emu, 224, 224, philox=False)["lean_light"]            # resolved records: 56 rows of the 3-CTA kernel
