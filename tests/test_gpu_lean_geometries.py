"""The lean light kernel at every launch geometry the planner gives it, against the host build and the record oracle.

`plan_launch` runs the lean variant of the light kernel (octet paths only, no per-CTA geometry check) in every Philox
launch with octets, a staged light band and no crop: the production step at 224, `FusedAugmenter`, `run_many` and TTA
at the EfficientNet sizes.  tests/geometry_cases.py LEAN_CASES holds one case per lean regime (light band count, even or
uneven bands, W / 8 parity, a band near its staging limit, one-row bands, the cluster kernel beside the lean kernel).

Each case runs a policy whose sub-policies reach every octet path of the lean kernel and every program class of the mid
(and cluster) kernel in the same launch, with a seed whose Philox draws give every sub-policy and both flips to the
batch.  Every `out=` buffer is filled with a sentinel first (NaN, 0xAB), so a band or octet no CTA wrote fails.

References: every image must equal the host build (helpers.philox_reference); up to 640 px every image of the host
build must also equal tests/record_oracle.py (Pillow, from the same records), above that a sample of 8.  fp32 is the
exact normalisation table applied to those bytes, fp16 / bf16 that value rounded once.  Every call asserts the planner's
lean bit and its launch count (`faa_launch_count`).

At the production sizes 224, 240 and 456 every output (uint8 HWC, fp32, fp16, bf16, CutoutDefault in fp32, Lighting in
fp16 and fp32) goes through every Philox entry point (`augment_batch(rng=...)`, `FusedAugmenter(overlap_calls=True)`
three calls back to back, `run_many` over 3 steps, `augment_tta` with 2 replicas) and a three-op policy; elsewhere fp16
and uint8 through `augment_batch`.  At 240 the batch runs one below, at and one above the light kernel's persistent row
count, so rows run zero, one and two rounds.
"""
import random

import numpy as np
import pytest
import torch

import geometry_cases as G
from helpers import emu_philox_records, exact_norm_table, philox_reference, reference_output, synth_batch
from record_oracle import render_batch

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.engine import (IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, FusedAugmenter, TailSpec,
                                          augment_batch, augment_tta, make_rng)

pytestmark = pytest.mark.gpu

MEAN, STD = IMAGENET_MEAN, IMAGENET_STD
U8 = TailSpec(None, 0, True, MEAN, STD, 0, torch.uint8)
FIRST = 7000


def _launches():
    return int(_lib.lib.faa_launch_count())


def _light_programs():
    """programs the lean light kernel finishes itself (prog_is_light under allow bit 8), one per octet path"""
    return [
        [("Invert", 0.0, 0.5), ("Solarize", 0.0, 0.5)],                 # C_PLAIN: both gates off
        [("Solarize", 1.0, 0.4), ("Posterize", 1.0, 0.6)],              # C_LUT
        [("Brightness", 1.0, 0.3), ("Invert", 0.0, 0.0)],               # C_LUT: Brightness
        [("Color", 1.0, 0.8), ("Invert", 0.0, 0.5)],                    # Color alone
        [("Cutout", 1.0, 0.6), ("Invert", 0.0, 0.0)],                   # Cutout alone
        [("Color", 1.0, 0.3), ("Posterize", 1.0, 0.5)],                 # Color -> static LUT: the float table
        [("CutoutAbs", 1.0, 0.9), ("Invert", 1.0, 0.0)],                # Cutout -> static LUT
        [("TranslateX", 1.0, 0.7), ("Invert", 0.5, 0.0)],               # row shift (alone or -> LUT: pad lut(0))
        [("Solarize", 1.0, 0.3), ("TranslateY", 1.0, 0.8)],             # LUT -> row shift
        [("TranslateXAbs", 1.0, 0.9), ("Invert", 1.0, 0.0)],            # row shift -> LUT: pad lut(0) = 255
        [("Posterize2", 1.0, 0.5), ("Rotate", 1.0, 0.7)],               # LUT -> warp-tiled gather
        [("ShearY", 1.0, 0.6), ("Invert", 1.0, 0.0)],                   # warp-tiled gather -> LUT
        [("Rotate", 1.0, 0.4), ("Invert", 0.0, 0.0)],                   # warp-tiled gather alone
        [("ShearX", 1.0, 0.6), ("TranslateY", 1.0, 0.7)],               # two gathers (C_GEOM2)
        [("TranslateYAbs", 1.0, 0.9), ("ShearY", 1.0, 0.2)],            # two gathers (C_GEOM2)
        [("Cutout", 1.0, 0.9), ("Rotate", 1.0, 0.1)],                   # Cutout -> gather
    ]


def _programs():
    """the light programs and what the mid kernel takes beside them in the same launch (at most 24 sub-policies)"""
    return _light_programs() + [
        [("Color", 1.0, 0.2), ("TranslateX", 1.0, 0.8)],                # Color -> gather: rebuilt as gather -> Color
        [("Solarize", 1.0, 0.5), ("Color", 1.0, 0.7)],                  # two-stage: LUT -> Color
        [("Rotate", 1.0, 0.4), ("CutoutAbs", 1.0, 0.8)],                # two-stage: gather -> Cutout
        [("Equalize", 1.0, 0.5), ("ShearY", 1.0, 0.4)],                 # statistics LUT -> gather
        [("AutoContrast", 1.0, 0.5), ("Contrast", 1.0, 0.3)],           # statistics ops
        [("Sharpness", 1.0, 0.9), ("TranslateX", 1.0, 0.6)],            # Sharpness -> gather
        [("Sharpness", 1.0, 0.7), ("Posterize", 1.0, 0.2)],             # Sharpness -> LUT
        [("Rotate", 0.5, 0.3), ("Color", 0.5, 0.6)],                    # gates drawn: any of four programs
    ]


def _three_op():
    """a three-op policy: the first window writes uint8, the last one (op 2 alone) runs on the event schedule"""
    return [
        [("Rotate", 1.0, 0.3), ("Invert", 1.0, 0.0), ("Color", 1.0, 0.6)],
        [("Equalize", 1.0, 0.5), ("TranslateX", 1.0, 0.7), ("Posterize", 1.0, 0.4)],
        [("Cutout", 1.0, 0.6), ("ShearY", 0.5, 0.4), ("TranslateYAbs", 1.0, 0.8)],
        [("Sharpness", 1.0, 0.8), ("Brightness", 1.0, 0.6), ("CutoutAbs", 1.0, 0.9)],
        [("Color", 1.0, 0.2), ("Contrast", 0.5, 0.6), ("Solarize", 1.0, 0.3)],
        [("AutoContrast", 0.0, 0.5), ("Invert", 0.0, 0.3), ("ShearX", 1.0, 0.5)],
    ]


def _seed_covering(emu, pol, shape, B):
    """the first seed whose Philox draws give every sub-policy and both flips to the batch at FIRST"""
    for seed in range(1, 400):
        s, _ = emu_philox_records(emu, pol, B, *shape, U8, seed, FIRST)
        if len(set(s["sub"].tolist())) == pol.n_sub and 0 < int(s["flip"].sum()) < B:
            return seed
    raise AssertionError("no covering seed")


def _sentinel(shape, dtype):
    if dtype == torch.uint8:
        return torch.full(shape, 0xAB, dtype=dtype, device="cuda")
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _bad(got, want):
    """indices of the images that differ (NaN never equals)"""
    got, want = got.cpu(), want.cpu()
    return [i for i in range(got.shape[0]) if not torch.equal(got[i], want[i])]


class _Refs:
    """host references of one batch at the record indices FIRST + k * B: the uint8 bytes (host build, checked against the
    record oracle), exact fp32, and the CutoutDefault(16) zero boxes"""

    def __init__(self, emu, policies, case, xh, seed, steps):
        self.emu, self.policies, self.case, self.xh, self.seed = emu, policies, case, xh, seed
        self.pol = CompiledPolicy(policies)
        B = xh.shape[0]
        self.u8 = [self._u8(FIRST + k * B) for k in range(steps)]
        self.tab = torch.from_numpy(exact_norm_table(MEAN, STD))

    def _u8(self, first):
        B, H, W, _ = self.xh.shape
        samples, boxes = emu_philox_records(self.emu, self.pol, B, H, W, U8, self.seed, first)
        want = reference_output(self.emu, self.pol, self.xh, U8, samples, boxes)
        idx = sorted(random.Random(H * W + first).sample(range(B), 8)) if self.case.big else range(B)
        oracle = render_batch(self.policies, self.xh, samples, boxes, idx)
        bad = [(i, self.policies[samples["sub"][i]]) for i in idx if not np.array_equal(want[i].numpy(), oracle[i])]
        assert not bad, (self.case.id, "host build != record oracle", first, len(bad), bad[:4])
        return want

    def f32(self, k):
        x = self.u8[k].permute(0, 3, 1, 2).long()
        return torch.stack([self.tab[c][x[:, c]] for c in range(3)], 1)

    def want(self, k, tail):
        """the expected output of step k in `tail` (uint8, fp32 / fp16 / bf16, CutoutDefault)"""
        if tail.out_dtype == torch.uint8:
            return self.u8[k]
        w = self.f32(k)
        if tail.cutout:
            B, H, W, _ = self.xh.shape
            s, _ = emu_philox_records(self.emu, self.pol, B, H, W, tail, self.seed, FIRST + k * B)
            for i in range(B):
                y0, y1, x0, x1 = (int(v) for v in s["zero_box"][i])
                w[i, :, y0:y1, x0:x1] = 0
        return w.to(tail.out_dtype)


TAILS = {"uint8": U8, "fp32": TailSpec.imagenet(0, torch.float32), "fp16": TailSpec.imagenet(0, torch.float16),
         "bf16": TailSpec.imagenet(0, torch.bfloat16), "cutout fp32": TailSpec.imagenet(16, torch.float32)}


class _Case:
    """one LEAN_CASES entry on the device: collects every wrong value and launch count, asserts once"""

    def __init__(self, emu, case, policies, B=None, steps=1, seed=None):
        self.emu, self.case, self.policies = emu, case, policies
        self.B = B or case.batch
        self.shape = case.shape
        xh = synth_batch(self.B, self.shape, seed=self.shape[0] * 7 + self.shape[1] + self.B)
        self.x = torch.from_numpy(xh).cuda()
        self.seed = seed or _seed_covering(emu, CompiledPolicy(policies), self.shape, self.B)
        self.refs = _Refs(emu, policies, case, xh, self.seed, steps)
        self.errors = []

    def pixel(self, u8, batch=None):
        """pixel kernels of one chained call, after asserting the planner runs the lean kernel in it"""
        p = self.case.plan(self.emu, u8=u8, batch=batch or self.B)
        assert p.lean and G.lean_regime(p) == self.case.regime, (self.case.id, u8, p)
        return p.launches() - 1

    def expect(self, what, n0, want_launches, got, want):
        n = _launches() - n0
        if n != want_launches:
            self.errors.append((what, "launches", n, want_launches))
        bad = _bad(got, want)
        if bad:
            self.errors.append((what, len(bad), bad[:6]))

    def out(self, tail, lead=()):
        B, (H, W) = self.B, self.shape
        shape = lead + ((B, H, W, 3) if tail.out_dtype == torch.uint8 else (B, 3, H, W))
        return _sentinel(shape, tail.out_dtype)

    def augment_batch(self, name, tail):
        pol = CompiledPolicy(self.policies)                             # a fresh handle: a miss, resolve + resolve-ahead
        u8 = tail.out_dtype == torch.uint8
        n0 = _launches()
        got = augment_batch(pol, self.x, tail, rng=make_rng(self.seed, FIRST, tail), out=self.out(tail))
        self.expect(("augment_batch", name), n0, self.pixel(u8) + 2, got, self.refs.want(0, tail))

    def lighting(self, dt):
        from fast_autoaugment_b200.data import Lighting
        torch.manual_seed(self.B + self.shape[1])
        rgb = Lighting(0.1).sample_rgb(self.B).float()
        tail = TailSpec.imagenet(0, dt)
        pol = CompiledPolicy(self.policies)
        n0 = _launches()
        got = augment_batch(pol, self.x, tail, rng=make_rng(self.seed, FIRST, tail), out=self.out(tail),
                            lighting_rgb=rgb.cuda())
        s, b = emu_philox_records(self.emu, pol, self.B, *self.shape, tail, self.seed, FIRST)
        want = reference_output(self.emu, pol, self.refs.xh, tail, s, b, lighting_rgb=rgb)
        self.expect(("Lighting", str(dt)), n0, self.pixel(False) + 3, got, want)       # + the per-image tables

    def fused(self, name, tail):
        """three calls back to back on one stream: miss, hit, hit"""
        pol = CompiledPolicy(self.policies)
        aug = FusedAugmenter(pol, tail, *self.shape, seed=self.seed, overlap_calls=True)
        pixel = self.pixel(tail.out_dtype == torch.uint8)
        for k in range(3):
            out = self.out(tail)
            n0 = _launches()
            aug(self.x, out, FIRST + k * self.B)
            self.expect(("FusedAugmenter", name, k), n0, pixel + (2 if k == 0 else 1), out, self.refs.want(k, tail))

    def run_many(self, name, tail):
        pol = CompiledPolicy(self.policies)
        aug = FusedAugmenter(pol, tail, *self.shape, seed=self.seed)
        outs = [self.out(tail) for _ in range(3)]
        plan = aug.plan_many([self.x] * 3, outs)
        pixel = self.pixel(tail.out_dtype == torch.uint8)
        n0 = _launches()
        aug.run_many(plan, FIRST)
        n = _launches() - n0
        if n != 3 * pixel + 4:                                          # miss, hit, hit
            self.errors.append((("run_many", name), "launches", n, 3 * pixel + 4))
        for k in range(3):
            bad = _bad(outs[k], self.refs.want(k, tail))
            if bad:
                self.errors.append((("run_many", name, k), len(bad), bad[:6]))

    def tta(self, name, tail):
        pol = CompiledPolicy(self.policies)
        out = self.out(tail, lead=(2,))
        n0 = _launches()
        augment_tta(pol, self.x, tail, 2, self.seed, FIRST, out=out)
        want = torch.stack([self.refs.want(r, tail) for r in range(2)])
        n = _launches() - n0
        pixel = self.pixel(tail.out_dtype == torch.uint8, batch=2 * self.B)
        if n != pixel + 2:
            self.errors.append((("tta", name), "launches", n, pixel + 2))
        bad = [r for r in range(2) if _bad(out[r], want[r])]
        if bad:
            self.errors.append((("tta", name), "replicas", bad, [_bad(out[r], want[r])[:6] for r in bad]))
        # ... and the reference of a replicated launch itself
        if tail.out_dtype == torch.float16:
            ref = philox_reference(self.emu, pol, self.refs.xh, tail, self.seed, FIRST, replicas=2)
            if _bad(out.flatten(0, 1), ref.flatten(0, 1)):
                self.errors.append((("tta", name), "philox_reference(replicas=2)"))

    def three_op(self, name, tail):
        policies = _three_op()
        pol = CompiledPolicy(policies)
        B, (H, W) = self.B, self.shape
        u8 = tail.out_dtype == torch.uint8
        last = G.plan(self.emu, H, W, B, u8=u8, philox=True, allow_ahead=False)
        assert last.lean and not last.use_chain, (self.case.id, "the last window", last)
        first = G.plan(self.emu, H, W, B, u8=True, philox=True, allow_ahead=False, apply_tail=False)
        n0 = _launches()
        got = augment_batch(pol, self.x, tail, rng=make_rng(self.seed, FIRST, tail), out=self.out(tail))
        samples, boxes = emu_philox_records(self.emu, pol, B, H, W, tail, self.seed, FIRST)
        want = reference_output(self.emu, pol, self.refs.xh, U8, samples, boxes)
        idx = sorted(random.Random(H + W).sample(range(B), 8))
        oracle = render_batch(policies, self.refs.xh, samples, boxes, idx)
        assert all(np.array_equal(want[i].numpy(), oracle[i]) for i in idx), (self.case.id, "three ops: host build != oracle")
        if not u8:
            x = want.permute(0, 3, 1, 2).long()
            want = torch.stack([self.refs.tab[c][x[:, c]] for c in range(3)], 1).to(tail.out_dtype)
        self.expect(("three ops", name), n0, first.launches() + last.launches(), got, want)

    def check(self):
        assert not self.errors, (self.case.id, self.case.regime, self.B, self.errors)


FULL = [c for c in G.LEAN_CASES if c.full]
REDUCED = [c for c in G.LEAN_CASES if not c.full]


@pytest.mark.parametrize("case", FULL, ids=lambda c: c.id)
def test_every_output_and_entry_point_at_production_sizes(emu, case, monkeypatch):
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    run = _Case(emu, case, _programs(), steps=3)
    for name, tail in TAILS.items():
        run.augment_batch(name, tail)
        run.fused(name, tail)
        run.run_many(name, tail)
        run.tta(name, tail)
    for dt in (torch.float16, torch.float32):
        run.lighting(dt)
    for name in ("uint8", "fp16"):
        run.three_op(name, TAILS[name])
    run.check()


@pytest.mark.parametrize("case", REDUCED, ids=lambda c: c.id)
def test_fp16_and_uint8_at_every_lean_geometry(emu, case, monkeypatch):
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    run = _Case(emu, case, _programs())
    for name in ("uint8", "fp16"):
        run.augment_batch(name, TAILS[name])
    run.check()


def test_persistent_rows_run_zero_one_and_two_rounds(emu, monkeypatch):
    """light programs only, so every entry is the lean kernel's: one batch below the row count (a row without an entry),
    at it (one each) and one above (a row runs a second round, and reloads its per-image Lighting table)"""
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    case = next(c for c in G.LEAN_CASES if c.id == "240x240")
    p = case.plan(emu)
    rows = torch.cuda.get_device_properties(0).multi_processor_count * 4 // p.light_bands
    for B in (rows - 1, rows, rows + 1):
        run = _Case(emu, case, _light_programs(), B=B)
        assert run.pixel(False) == 2 and run.pixel(True) == 2          # light + mid
        for name in ("uint8", "fp16"):
            run.augment_batch(name, TAILS[name])
        run.lighting(torch.float32)
        run.check()
