"""The launch-geometry case table (tests/geometry_cases.py) against the planner's decisions, without a GPU.

Every case must sit in the regime it claims under the Python restatement of `augment_common`, with the launch count it
claims; every regime must have a case; and the table must cover the sizes the ImageNet loaders produce and the header's
size limits.  On the GPU, tests/test_gpu_geometries.py asserts the same launch counts against the real planner."""
import pytest

import geometry_cases as G

from fast_autoaugment_b200.data import EFFICIENTNET_SIZES


@pytest.mark.parametrize("case", G.CASES, ids=lambda c: c.id)
def test_every_case_is_in_the_regime_it_claims(case):
    H, W = case.shape
    p = G.plan(H, W, 64, in_off=case.in_off, out_off=case.out_off, split_min=0)
    assert G.regime(p) == case.regime, (case.id, p)
    assert p.launches() == case.launches, (case.id, p)
    assert G.plan(H, W, 64, in_off=case.in_off, out_off=case.out_off, split_min=1 << 62).launches() == 2
    assert case.in_off % 4 == 0 and case.out_off % 8 == 0          # only offsets the kernels accept
    assert case.big == (max(H, W) > 640)


def test_every_regime_has_a_case():
    seen = {c.regime for c in G.CASES}
    assert seen == set(G.REGIMES), {"regimes without a case": set(G.REGIMES) - seen, "unlisted regimes": seen - set(G.REGIMES)}


def test_the_table_covers_the_loader_sizes_and_the_header_limits():
    plain = {c.shape for c in G.CASES if not c.in_off and not c.out_off}
    want = {(s, s) for s in EFFICIENTNET_SIZES.values() if s != 224} | set(G.PHOTO_SHAPES) | set(G.LIMIT_SHAPES)
    assert plain == want | {(256, 256)}, {"missing": want - plain, "extra": plain - want}
    offsets = {(c.shape, c.in_off, c.out_off) for c in G.CASES if c.in_off or c.out_off}
    assert offsets == {((224, 224), 4, 0), ((600, 600), 4, 0), ((224, 224), 0, 8)}


def test_the_restatement_matches_the_known_launch_counts():
    """the counts the schedule tests assert at production sizes (tests/test_gpu_schedules.py: 224 b512 splits with the
    mid kernel and no cluster kernel, 380 b256 keeps the cluster kernel, 224 b64 runs one pixel kernel)"""
    assert G.plan(224, 224, 512).launches() == 3 and G.plan(224, 224, 512).no_heavy
    assert G.plan(380, 380, 256).launches() == 4
    assert G.plan(224, 224, 64).launches() == 2
    assert G.plan(224, 224, 512, u8=True).launches() == 3            # uint8 output splits through the octet paths
    assert G.plan(375, 500, 512, u8=True).launches() == 2
