"""The launch-geometry case table (tests/geometry_cases.py) against the launch planner, without a GPU.

Every case must sit in the regime it claims under the library's planner (`plan_launch` in csrc/faa_core.cuh, through
the host build), with the launch count it claims; every regime must have a case; and the table must cover the sizes the
ImageNet loaders produce and the header's size limits.  The same holds for the RandomCrop and fused Mixup tables
(CROP_CASES, MIX_CASES).  On the GPU, tests/test_gpu_geometries.py and tests/test_gpu_crop_mix_geometries.py assert the
same launch counts against the launches the library counts."""
import pytest

import geometry_cases as G

from fast_autoaugment_b200.data import EFFICIENTNET_SIZES


@pytest.mark.parametrize("case", G.CASES, ids=lambda c: c.id)
def test_every_case_is_in_the_regime_it_claims(emu, case):
    H, W = case.shape
    p = G.plan(emu, H, W, 64, in_off=case.in_off, out_off=case.out_off, split_min=0)
    assert G.regime(p) == case.regime, (case.id, p)
    assert p.launches() == case.launches, (case.id, p)
    assert G.plan(emu, H, W, 64, in_off=case.in_off, out_off=case.out_off, split_min=1 << 62).launches() == 2
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


def test_the_restatement_matches_the_known_launch_counts(emu):
    """the counts the schedule tests assert at production sizes (tests/test_gpu_schedules.py: 224 b512 splits with the
    mid kernel and no cluster kernel, 380 b256 keeps the cluster kernel, 224 b64 runs one pixel kernel)"""
    assert G.plan(emu, 224, 224, 512).launches() == 3 and G.plan(emu, 224, 224, 512).no_heavy
    assert G.plan(emu, 380, 380, 256).launches() == 4
    assert G.plan(emu, 224, 224, 64).launches() == 2
    assert G.plan(emu, 224, 224, 512, u8=True).launches() == 3       # uint8 output splits through the octet paths
    assert G.plan(emu, 375, 500, 512, u8=True).launches() == 2


@pytest.mark.parametrize("case", G.CROP_CASES + G.MIX_CASES, ids=lambda c: c.id)
def test_every_crop_and_mixup_case_is_in_the_regime_it_claims(emu, case):
    p = case.plan(emu)
    assert G.regime(p) == case.regime, (case.id, p)
    assert p.launches() == case.launches, (case.id, p)
    assert case.plan(emu, split_min=1 << 62).launches() == 2
    assert case.two_src == p.two_src and p.crop == (case.pad > 0 or case.out != case.shape)
    assert case.in_off % 4 == 0 and case.pad <= 127                 # int8 records
    assert case.big == (max(case.shape) > 640)


def test_every_crop_and_mixup_regime_has_a_case():
    for cases, regimes in ((G.CROP_CASES, G.CROP_REGIMES), (G.MIX_CASES, G.MIX_REGIMES)):
        seen = {c.regime for c in cases}
        assert seen == set(regimes), {"regimes without a case": set(regimes) - seen, "unlisted regimes": seen - set(regimes)}


def test_the_crop_and_mixup_tables_reproduce_the_planner_rows(emu):
    """what the planner decides for the launches the tables were built from (batch 64, FAA_SPLIT_MIN 0, float output)"""
    def at(shape, pad=0, out=None, **kw):
        return G.plan(emu, *shape, 64, split_min=0, out_h=(out or shape)[0], out_w=(out or shape)[1], crop_pad=pad, **kw)
    # the light kernel's band stops being staged with the crop slack
    p = at((224, 224), 127)
    assert p.stage and p.band_cap == 224 * 224 * 3 <= G.STAGE_LIMIT and not p.light_staged and p.octets and p.split
    p = at((380, 380), 32)
    assert p.stage and p.band_cap == 130048 and not p.light_staged and not p.octets
    assert at((224, 224), 4).light_staged and at((224, 224), 4).light_bands == 7
    # outputs smaller than the image: no octets; a crop never runs the mid kernel
    assert not any(at(s, pad, out).octets or at(s, pad, out).use_mid for s, pad, out in
                   (((224, 224), 0, (200, 200)), ((256, 256), 8, (224, 224)), ((240, 240), 8, (224, 224))))
    assert not at((1536, 2048), 8).mat and not at((8, 8192), 4).mat and at((8192, 8), 4).octets
    assert at((375, 500), 4, (368, 496)).light_bands == 5
    # Mixup: unstaged at 456 - 600 because two bands do not fit, although one source's band does
    for s in ((456, 456), (528, 528), (600, 600)):
        assert not at(s, two_src=True).stage and at(s).stage, s
        assert at(s, two_src=True).stage_off == "doubled band"
    for s in ((224, 224), (240, 240), (256, 256), (260, 260), (300, 300), (380, 380), (8, 8192)):
        p = at(s, two_src=True)
        assert p.stage and 2 * p.band_cap <= G.STAGE_LIMIT and not p.mat and not p.split, s
    assert at((8, 8192), two_src=True).band_cap == 72 * 1024
    assert at((224, 224), 16, two_src=True).stage and at((380, 380), 32, two_src=True).stage_off == "doubled band"
    assert at((224, 224), two_src=True, in_off=4).stage_off == "base"


def test_cifar_philox_launches_split_from_4096_images(emu):
    """CIFAR with the Philox sampler and resolve-ahead: B = 2048 is one self-resolving kernel; from B = 4096 (4 M pixels)
    the launch splits into resolve + light + cluster kernels on the chained schedule, with crops - as does a TTA launch
    of 1024 images x 5 replicas"""
    def cifar(B):
        return G.plan(emu, 32, 32, B, crop_pad=4, philox=True, allow_ahead=True)
    p = cifar(2048)
    assert p.self_resolving and not p.split and p.launches() == 1
    for B in (4096, 8192, 1024 * 5):
        p = cifar(B)
        assert not p.self_resolving and p.split and p.use_chain and not p.use_mid and p.launches() == 3, B
