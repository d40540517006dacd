"""The lean light launch's case table (tests/geometry_cases.py LEAN_CASES) and the record oracle (tests/record_oracle.py),
without a GPU.

Every case must be a lean launch in the regime it claims, in float and in uint8 HWC output, at the batch sizes
tests/test_gpu_lean_geometries.py runs and at the library's default split threshold; every lean regime must have a case;
every lean shape of the other tables must be in LEAN_CASES or covered by a named case of the same regime; the negative
cases must not be lean.

The record oracle renders a decision record through `oracle.pil_path`'s Pillow calls.  It is pinned here against
`PolicyTransform` itself: under `seed_all(k)` both must give the same bytes for the records `sample_parity` replays from
the same generators, over every op at every level of the oracle sweeps, every ordered pair, Cutout boxes at the image
borders and at level 0, at sizes with an odd number of octets per row and with H != W."""
import itertools

import numpy as np
import PIL.Image
import pytest

import geometry_cases as G
from helpers import ALL_OPS, seed_all, synth_batch
from record_oracle import render_record
from test_gpu_fastpaths import _policies
from test_gpu_lean_geometries import _light_programs
from test_lean_light_host import _classes, lean_emu  # noqa: F401  (lean_emu: the fixture)

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.data import EFFICIENTNET_SIZES
from fast_autoaugment_b200.engine import CompiledPolicy
from oracle import pil_path

SMS = (132, 114)              # H100 SXM / PCIe: the persistent-rows test derives its batches from the SM count


@pytest.mark.parametrize("case", G.LEAN_CASES, ids=lambda c: c.id)
def test_every_lean_case_is_in_the_regime_it_claims(emu, case):
    H, W = case.shape
    batches = {case.batch, 2 * case.batch}                           # plain calls and a TTA launch of 2 replicas
    for u8 in (False, True):
        for b in batches:
            p = case.plan(emu, u8=u8, batch=b)
            assert G.lean_regime(p) == case.regime, (case.id, u8, b, p)
            assert p.use_chain and p.use_mid and p.light_staged and p.light_cap <= G.LIGHT_STAGE_LIMIT, (case.id, p)
        # the same launch on resolved records keeps the 80-register kernel
        assert not G.plan(emu, H, W, case.batch, u8=u8).lean
    assert case.big == (max(H, W) > 640)
    assert case.batch >= 48                                          # room for every sub-policy of the GPU test's policy


def test_every_lean_regime_has_a_case():
    seen = [c.regime for c in G.LEAN_CASES]
    assert set(seen) == set(G.LEAN_REGIMES) and len(G.LEAN_REGIMES) == len(set(G.LEAN_REGIMES)), \
        {"regimes without a case": set(G.LEAN_REGIMES) - set(seen), "unlisted regimes": set(seen) - set(G.LEAN_REGIMES)}
    # the dimensions a regime is made of: band counts 2 and 4 - 8, uneven bands with either W/8 parity, the limit, one-row
    # bands, the cluster kernel beside the lean kernel
    assert {int(r.split()[0]) for r in seen} == {2, 4, 5, 6, 7, 8}
    assert {r.split(", ")[2] for r in seen if "uneven" in r} == {"W/8 odd", "W/8 even"}
    for extra in ("near the limit", "one-row bands", "one octet per row", "cluster kernel"):
        assert any(extra in r for r in seen), extra


def test_the_lean_shapes_of_the_other_tables_are_covered(emu):
    ids = {c.id for c in G.LEAN_CASES}
    shapes = ({c.shape for c in G.CASES if not c.in_off and not c.out_off} | {(s, s) for s in EFFICIENTNET_SIZES.values()}
              | set(G.PHOTO_SHAPES))
    lean = {s for s in shapes if G.plan(emu, *s, 512, philox=True, allow_ahead=True).lean}
    assert lean >= {(224, 224), (240, 240), (456, 456)}
    for s in sorted(lean):
        if "%dx%d" % s in ids:
            continue
        assert s in G.LEAN_COVERED_BY, ("a lean shape without a case", s)
        by = next(c for c in G.LEAN_CASES if c.id == G.LEAN_COVERED_BY[s])
        assert G.lean_regime(G.plan(emu, *s, 512, philox=True, allow_ahead=True)) == by.regime, (s, by.id)
    assert set(G.LEAN_COVERED_BY) <= lean


@pytest.mark.parametrize("shape,in_off,out_off,why", G.LEAN_NEGATIVE, ids=lambda v: str(v))
def test_the_negative_cases_are_not_lean(emu, shape, in_off, out_off, why):
    for u8 in ((False, True) if not out_off else (False,)):
        for b in (64, 512):
            p = G.plan(emu, *shape, b, u8=u8, in_off=in_off, out_off=out_off, philox=True, allow_ahead=True)
            assert not p.lean and G.lean_regime(p) is None, (shape, in_off, out_off, u8, b, why, p)


def test_the_persistent_rows_batches_are_lean(emu, lean_emu):
    """tests/test_gpu_lean_geometries.py runs 240 x 240 at one batch below, at and above the light row count, with
    programs that are all the lean kernel's - whatever the draws - so that one row gets no entry, or a second one"""
    case = next(c for c in G.LEAN_CASES if c.id == "240x240")
    for sms in SMS:
        rows = sms * 4 // case.plan(emu).light_bands
        for b in (rows - 1, rows, rows + 1):
            for u8 in (False, True):
                assert G.lean_regime(case.plan(emu, u8=u8, batch=b)) == case.regime, (sms, b, u8)
    policies = _light_programs()
    rows = list(itertools.product(range(len(policies)), range(4), range(4), (0, 1)))
    samples = np.zeros(len(rows), dtype=_lib.SAMPLE_DTYPE)
    boxes = np.zeros((len(rows), 2), dtype=_lib.BOX_DTYPE)
    for i, (sub, gate, sign, flip) in enumerate(rows):
        samples[i]["sub"], samples[i]["gate"], samples[i]["sign"], samples[i]["flip"] = sub, gate, sign, flip
        boxes[i]["x0"], boxes[i]["y0"], boxes[i]["x1"], boxes[i]["y1"] = i % 50, i % 70, 150 + i % 90, 100 + i % 140
    c = _classes(lean_emu, policies, samples, boxes, *case.shape, case.plan(emu).allow)
    assert (c[:, 0] == 2).all(), [(policies[rows[i][0]], rows[i][1:]) for i in np.flatnonzero(c[:, 0] != 2)][:6]


# ------------------------------------------------------------------------------------------------- record oracle --
def _pin(policies, shape, seed, flip_odd=True):
    """every image of a batch, each with its own policy: PolicyTransform against render_record of sample_parity's
    records from the same generator state; returns the records"""
    H, W = shape
    batch = synth_batch(len(policies), shape, seed=seed)
    seed_all(seed)
    want = [np.asarray(pil_path.PolicyTransform([p])(PIL.Image.fromarray(a))) for p, a in zip(policies, batch)]
    seed_all(seed)
    bad, recs = [], []
    for i, p in enumerate(policies):
        s, b = CompiledPolicy([p]).sample_parity(1, H, W)
        s["flip"] = i & 1 if flip_odd else 0
        got = render_record([p], batch[i], s[0], b[0])
        w = want[i][:, ::-1] if s["flip"][0] else want[i]
        if not np.array_equal(got, w):
            bad.append((i, p))
        recs.append((s[0], b[0]))
    assert not bad, (shape, len(bad), bad[:6])
    return recs


@pytest.mark.parametrize("shape", [(40, 56), (64, 40)], ids=lambda s: "%dx%d" % s)
def test_the_record_oracle_equals_the_policy_transform(shape):
    """every op at every level of the oracle sweeps in either slot, every ordered pair, gather + LUT partners, Sharpness
    pairs (test_gpu_fastpaths._policies); W / 8 odd, H != W; odd images mirrored"""
    recs = _pin(_policies(), shape, seed=5)
    signs = [s["sign"] for s, _ in recs]
    assert any(signs) and not all(signs)                               # both mirror signs occurred


def test_the_record_oracle_draws_cutout_boxes_at_the_borders_and_at_level_0():
    H, W = 24, 40
    policies = [[(op, 1.0, lv), ("Invert", 0.0, 0.0)] for op in ("Cutout", "CutoutAbs") for lv in (0.0, 0.5, 1.0)
                for _ in range(24)]
    recs = _pin(policies, (H, W), seed=9)
    boxes = [(p[0][0], p[0][2], tuple(int(b[0][k]) for k in ("x0", "y0", "x1", "y1"))) for p, (_, b) in zip(policies, recs)]
    assert all(box[2] == -1 for op, lv, box in boxes if op == "Cutout" and lv == 0.0)          # no box
    assert all(box[0] == box[2] for op, lv, box in boxes if op == "CutoutAbs" and lv == 0.0)   # one pixel
    drawn = [box for _, _, box in boxes if box[2] != -1]
    for side in ((0, 0), (1, 0), (2, W), (3, H)):
        assert any(b[side[0]] == side[1] for b in drawn), side                                # every border is touched


def test_the_record_oracle_selects_sub_policies_and_gates():
    """one policy of many sub-policies with gate probabilities between 0 and 1, as the sampler draws it for a batch"""
    import random
    rng = random.Random(3)
    policies = [[(rng.choice(ALL_OPS), rng.choice((0.0, 0.3, 0.7, 1.0)), rng.random()) for _ in range(2)] for _ in range(25)]
    policies += [[(rng.choice(ALL_OPS), rng.random(), rng.random()) for _ in range(3)] for _ in range(5)]      # three ops
    H, W = 48, 24
    n = 240
    batch = synth_batch(n, (H, W), seed=2)
    seed_all(7)
    t = pil_path.PolicyTransform(policies)
    want = [np.asarray(t(PIL.Image.fromarray(a))) for a in batch]
    pol = CompiledPolicy(policies)
    seed_all(7)
    samples, boxes = pol.sample_parity(n, H, W)
    bad = [i for i in range(n) if not np.array_equal(render_record(policies, batch[i], samples[i], boxes[i]), want[i])]
    assert not bad, bad[:8]
    gates = {int(s["gate"]) for s in samples}
    assert len({int(s["sub"]) for s in samples}) == len(policies) and {0, 1, 2, 3} <= gates
