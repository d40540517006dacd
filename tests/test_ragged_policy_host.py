"""The ragged policy launch (``faa_augment_ragged``) on a CPU-only box: the planner itself through its host build
(tests/emu/faa_emu_ragged_plan.cpp) - every image covered once, each size's geometry that of a uniform uint8 launch of
that size, one pixel launch per cluster size, largest first - and the C ABI's refusals before any device work."""
import ctypes as C

import numpy as np
import pytest
import torch

import geometry_cases as G
from geometry_cases import LIMIT_SHAPES, PHOTO_SHAPES, load_emu_ragged_plan, plan, plan_ragged

from fast_autoaugment_b200 import _lib, archive, engine
from fast_autoaugment_b200.engine import RaggedImages, TailSpec


@pytest.fixture(scope="module")
def emu_rp():
    return load_emu_ragged_plan()


def rcp(d):
    return 0 if d <= 1 else ((1 << 32) + d - 1) // d


def mixture(seed, n, extra=()):
    rng = np.random.default_rng(seed)
    sizes = [PHOTO_SHAPES[int(k)] for k in rng.integers(0, len(PHOTO_SHAPES), n)]
    sizes += [(int(rng.integers(1, 1025)), int(rng.integers(1, 1025))) for _ in range(n // 2)]
    sizes += list(extra)
    rng.shuffle(sizes)
    return [tuple(s) for s in sizes]


MIXES = {
    "header limits": [(8192, 2), (2, 8192), (1, 1), (3, 4), (1, 1), (8192, 2)],
    "photo shapes": list(PHOTO_SHAPES) + [(3, 4), (1, 1)],
    "limit shapes": list(LIMIT_SHAPES) + [(375, 500), (1, 1)],
    "random 40+ sizes": mixture(0, 48, [(8192, 2), (2, 8192), (1, 1), (3, 4)]),
    "one size": [(375, 500)] * 7,
}


@pytest.mark.parametrize("name", list(MIXES))
@pytest.mark.parametrize("aligned", [True, False])
def test_planner_covers_and_matches_plan_launch(emu_rp, emu, name, aligned):
    sizes = MIXES[name]
    n = len(sizes)
    rng = np.random.default_rng(len(name))
    in_mod = np.zeros(n, np.int32) if aligned else rng.integers(0, 16, n).astype(np.int32)
    out_mod = np.zeros(n, np.int32) if aligned else rng.integers(0, 4, n).astype(np.int32) * 4
    geom_of, order, launches, geoms = plan_ragged(emu_rp, sizes, in_mod, out_mod)
    # every image exactly once, launch by launch
    assert sorted(order.tolist()) == list(range(n))
    assert sum(c for _, _, c, _ in launches) == n
    assert [f for _, f, _, _ in launches] == list(np.cumsum([0] + [c for _, _, c, _ in launches])[:-1])
    # one launch per cluster size present, no more
    bands_present = {geoms[geom_of[i]]["bands"] for i in range(n)}
    assert len(launches) == len(bands_present) <= 4 and {b for b, _, _, _ in launches} == bands_present
    px = [sizes[i][0] * sizes[i][1] for i in range(n)]
    for b, f, c, smem in launches:
        imgs = order[f:f + c].tolist()
        assert all(geoms[geom_of[i]]["bands"] == b for i in imgs)
        # largest first inside the launch (ties in batch order)
        assert all((px[a], -a) >= (px[z], -z) for a, z in zip(imgs, imgs[1:]))
        assert smem == max(geoms[geom_of[i]]["band_cap"] + geoms[geom_of[i]]["mat_cap"] for i in imgs)
    # launches largest first (by their first image)
    firsts = [px[order[f]] for _, f, _, _ in launches]
    assert firsts == sorted(firsts, reverse=True)
    # each image's geometry is plan_launch's cluster-kernel geometry of a uniform uint8 launch of its size and bases
    for i, (h, w) in enumerate(sizes):
        g = geoms[geom_of[i]]
        assert (g["H"], g["W"]) == (h, w)
        p = plan(emu, h, w, 1, u8=True, in_off=int(in_mod[i]), out_off=int(out_mod[i]), split_min=1 << 62)
        assert (g["bands"], g["band_cap"], bool(g["stage"]), bool(g["octets"]), g["mat_cap"] > 0, g["allow"]) == \
            (p.bands, p.band_cap, p.stage, p.octets, p.mat, p.allow), (name, h, w)
        assert g["allow"] & 4 == 0 and bool(g["scratch"]) == (w % 4 == 0)
        assert (g["rcp_out_qpr"] & 0xFFFFFFFF, g["rcp_w"] & 0xFFFFFFFF, g["rcp_wq"] & 0xFFFFFFFF,
                g["rcp_opr"] & 0xFFFFFFFF) == (rcp((w + 3) // 4), rcp(w), rcp(w // 4), 0 if w % 8 else rcp(w // 8))
        # no TMA staging unless the base and the byte count are 16-byte aligned; a cluster is never taller than the image
        if in_mod[i] % 16 or (h * w * 3) % 16:
            assert not g["stage"] and g["band_cap"] == 0
        assert g["bands"] <= h


def test_planner_groups_alignment_variants_of_one_size(emu_rp):
    sizes = [(224, 224)] * 4
    geom_of, _, launches, geoms = plan_ragged(emu_rp, sizes, [0, 4, 0, 8], [0, 0, 4, 0])
    assert [bool(geoms[k]["stage"]) for k in geom_of] == [True, False, True, False]
    assert [bool(geoms[k]["octets"]) for k in geom_of] == [True, False, False, False]
    assert len(launches) == 1 and len(geoms) == 3
    _, _, _, g2 = plan_ragged(emu_rp, sizes, has_sg=False)
    assert len(g2) == 1 and not g2[0]["scratch"] and g2[0]["allow"] & 2 == 0


def test_planner_empty_batch(emu_rp):
    geom_of, order, launches, geoms = plan_ragged(emu_rp, [])
    assert launches == [] and geoms == []


# ------------------------------------------------------------------------- the ragged geometry table --
@pytest.mark.parametrize("case", G.RAGGED_CASES + [G.RAGGED_HUGE], ids=lambda c: c.id)
def test_every_ragged_case_is_in_the_regime_it_claims(emu_rp, case):
    _, _, launches, geoms = plan_ragged(emu_rp, [case.shape], [case.in_off], [case.out_off])
    assert G.ragged_regime(geoms[0], case.in_off, case.out_off) == case.regime, (case.id, geoms[0])
    assert launches == [(case.regime[0], 0, 1, geoms[0]["band_cap"] + geoms[0]["mat_cap"])]
    # only offsets the library accepts, each a different reason: aligned, 4 past 16 (no TMA base / no octets), odd
    assert case.in_off in (0, 4) or case.in_off % 2 == 1
    assert case.out_off in (0, 4)
    # the same image without a Sharpness -> gather program: no scratch image, no allow bit 1
    _, _, _, g = plan_ragged(emu_rp, [case.shape], [case.in_off], [case.out_off], has_sg=False)
    assert not g[0]["scratch"] and g[0]["allow"] & 2 == 0
    assert g[0]["allow"] == geoms[0]["allow"] & ~2
    assert G.ragged_regime(g[0], case.in_off, case.out_off)[:4] == case.regime[:4]


def test_every_value_of_every_ragged_dimension_has_a_case():
    ids = [c.id for c in G.RAGGED_CASES]
    assert len(ids) == len(set(ids))
    for dim, values in enumerate(G.RAGGED_DIMENSIONS):
        seen = {c.regime[dim] for c in G.RAGGED_CASES}
        assert seen == set(values), (dim, {"without a case": set(values) - seen, "unlisted": seen - set(values)})
    # the header limits are in the table (8192 x 8192 is its own GPU test)
    assert {c.shape for c in G.RAGGED_CASES if not c.in_off and not c.out_off} >= set(LIMIT_SHAPES) - {(8192, 8192)}
    assert G.RAGGED_HUGE.shape == (8192, 8192)


def test_a_band_at_the_stage_limit_is_staged_and_one_row_more_is_not(emu_rp):
    _, _, launches, g = plan_ragged(emu_rp, [(624, 640), (632, 640)])
    assert [x["band_cap"] for x in g] == [G.STAGE_LIMIT, 0] and g[0]["stage"] and not g[1]["stage"]
    assert launches == [(8, 0, 2, G.STAGE_LIMIT + g[0]["mat_cap"])] and g[0]["mat_cap"] == g[1]["mat_cap"] > 0


@pytest.mark.parametrize("name", list(G.RAGGED_MIXES))
def test_every_ragged_mixture_plans_the_launches_it_claims(emu_rp, name):
    ids, want = G.RAGGED_MIXES[name]
    cases = [G.ragged_case(i) for i in ids]
    geom_of, order, launches, geoms = plan_ragged(emu_rp, [c.shape for c in cases], [c.in_off for c in cases],
                                                  [c.out_off for c in cases])
    assert launches == want, name
    # each image keeps the geometry it has alone
    for i, c in enumerate(cases):
        assert G.ragged_regime(geoms[geom_of[i]], c.in_off, c.out_off) == c.regime, (name, c.id)
    # a call mixes staged, unstaged, chunk-less and copied images
    regimes = [c.regime for c in cases]
    assert {"staged", "base + copy"} <= {r[1] for r in regimes} and len({r[1] for r in regimes}) >= 2
    assert {"chunk", "no chunk"} == {r[3] for r in regimes}


def test_the_ragged_mixtures_reach_every_case_and_launch_shape(emu_rp):
    """every case runs in some mixture; some call has all four cluster sizes (four pixel launches, the most there can
    be); some 8-CTA launch takes its shared memory from an image that is not its first"""
    in_mixes = {i for ids, _ in G.RAGGED_MIXES.values() for i in ids}
    assert in_mixes == {c.id for c in G.RAGGED_CASES}
    assert any(len(want) == 4 for _, want in G.RAGGED_MIXES.values())
    not_first = []
    for name, (ids, want) in G.RAGGED_MIXES.items():
        cases = [G.ragged_case(i) for i in ids]
        geom_of, order, launches, geoms = plan_ragged(emu_rp, [c.shape for c in cases], [c.in_off for c in cases],
                                                      [c.out_off for c in cases])
        for bands, first, count, smem in launches:
            g = geoms[geom_of[order[first]]]
            if g["band_cap"] + g["mat_cap"] < smem:
                not_first.append((name, bands))
    assert ("four_cluster_sizes", 8) in not_first and ("smem_from_the_second_image", 8) in not_first, not_first


# ------------------------------------------------------------------------------------------------------ C ABI --
def _call(pol, images, outs=None, batch=None, samples=None, boxes=None, rng=None, op_base=0, null=()):
    n = len(images)
    h = np.zeros(max(1, n), _lib.IMAGE_DTYPE)
    for i, (ptr, hh, ww) in enumerate(images):
        h[i] = (ptr, hh, ww)
    o = np.zeros(max(1, n), _lib.IMAGE_DTYPE)
    for i, (ptr, hh, ww) in enumerate(outs if outs is not None else [(4096 * (k + 1), a, b) for k, (_, a, b) in
                                                                     enumerate(images)]):
        o[i] = (ptr, hh, ww)
    args = [pol.handle, h.ctypes.data, h.ctypes.data, n if batch is None else batch, o.ctypes.data, o.ctypes.data,
            samples, boxes, C.byref(rng) if rng is not None else None, op_base, None]
    for k in null:
        args[k] = None
    return _lib.lib.faa_augment_ragged(*args)


def test_abi_refusals_before_device_work():
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    pol3 = engine.CompiledPolicy([[("Invert", 0.5, 0.5), ("Sharpness", 0.5, 0.5), ("ShearX", 0.5, 0.5)]])
    rng = engine.make_rng(1, 0, TailSpec.raw_u8())
    ok = [(4096, 375, 500), (8192 + 1, 500, 375)]
    assert _call(pol, ok, null=(0,)) == _lib.ERR_VALUE                              # null policy
    for k in (1, 2, 4, 5):                                                          # a null descriptor array
        assert _call(pol, ok, rng=rng, null=(k,)) == _lib.ERR_VALUE
    assert _call(pol, ok) == _lib.ERR_VALUE                                         # neither samples nor rng
    assert _call(pol, ok, rng=rng, batch=-1) == _lib.ERR_VALUE
    assert _call(pol, ok, rng=rng, batch=65536) == _lib.ERR_UNSUPPORTED
    for bad in ((8192, 0, 8), (8192, 8193, 8), (8192, 8, 8193), (8192, -1, 1)):   # a size outside check_shape
        assert _call(pol, ok + [bad], rng=rng) == _lib.ERR_VALUE
        assert b"image 2" in _lib.lib.faa_last_error()
    assert _call(pol, ok + [(0, 20, 20)], rng=rng) == _lib.ERR_VALUE               # no data
    assert b"image 2" in _lib.lib.faa_last_error()
    # an output whose size differs from its input's
    assert _call(pol, ok, outs=[(4096, 375, 500), (8192, 375, 500)], rng=rng) == _lib.ERR_VALUE
    assert b"image 1" in _lib.lib.faa_last_error()
    # an output that breaks the uint8 alignment rule (W % 4 == 0: 4-byte aligned); W % 4 != 0 may start anywhere
    assert _call(pol, ok, outs=[(4098, 375, 500), (8192, 500, 375)], rng=rng) == _lib.ERR_UNSUPPORTED
    assert b"image 0" in _lib.lib.faa_last_error()
    # op_base out of range
    assert _call(pol, ok, rng=rng, op_base=2) == _lib.ERR_VALUE
    assert _call(pol, ok, rng=rng, op_base=-1) == _lib.ERR_VALUE
    assert _call(pol3, ok, rng=rng, op_base=3) == _lib.ERR_VALUE
    # a tail the ragged output cannot have
    for field in ("crop_pad", "hflip", "zero_box_len"):
        r = engine.make_rng(1, 0, TailSpec.raw_u8())
        setattr(r, field, 4)
        assert _call(pol, ok, rng=r) == _lib.ERR_VALUE
    # nothing was compiled or uploaded for any of these
    n, b = C.c_int(-1), C.c_uint64(1)
    _lib.check(_lib.lib.faa_policy_cached_tables(pol.handle, C.byref(n), C.byref(b)))
    assert (n.value, b.value) == (0, 0)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the refusal of a machine without a device")
def test_valid_ragged_call_needs_a_device():
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    rng = engine.make_rng(1, 0, TailSpec.raw_u8())
    # misaligned inputs and outputs of odd widths are valid
    assert _call(pol, [(4097, 375, 500), (8193, 500, 375), (9001, 1, 1)],
                 outs=[(4096, 375, 500), (8193, 500, 375), (9003, 1, 1)], rng=rng) == _lib.ERR_NO_DEVICE
    assert _call(pol, [(4096, 3, 4)], samples=C.c_void_p(64), boxes=C.c_void_p(64), op_base=1) == _lib.ERR_NO_DEVICE


def test_python_refusals():
    pol = engine.CompiledPolicy(archive.fa_resnet50_rimagenet())
    r = RaggedImages(torch.zeros(48, dtype=torch.uint8), [0, 12], [(2, 2), (1, 4)])
    raw = TailSpec.raw_u8()
    for tail in (TailSpec.imagenet(), TailSpec(None, 0, True, out_dtype=torch.uint8), TailSpec((1, 1), 0, False, out_dtype=torch.uint8)):
        with pytest.raises(ValueError):
            engine.augment_batch(pol, r, tail, rng=engine.make_rng(1))
    for kw in ({"partner": [0, 1]}, {"pool": r}, {"lighting_rgb": torch.zeros(2, 3)}):
        with pytest.raises(ValueError):
            engine.augment_batch(pol, r, raw, rng=engine.make_rng(1), **kw)
    with pytest.raises(ValueError):
        engine.augment_batch(pol, r, raw)                                  # neither records nor rng


def test_empty_layout_starts_every_image_on_16_bytes():
    e = RaggedImages.empty([(3, 5), (1, 1), (7, 4), (2, 2)], device="cpu")
    assert e.offsets.tolist() == [0, 48, 64, 160] and e.storage.numel() == 176
    assert e.sizes.tolist() == [[3, 5], [1, 1], [7, 4], [2, 2]]
    assert len(RaggedImages.empty(np.zeros((0, 2)), device="cpu")) == 0
