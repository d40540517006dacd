"""RandomCrop and fused Mixup launches at every launch geometry the planner can choose, against the oracle.

tests/geometry_cases.py holds one case per regime of the two planner inputs that tests/test_gpu_geometries.py keeps
fixed: the crop (`crop_pad`, outputs smaller than the image: the staged bands and the chunk include the crop slack, the
octet paths only serve images at offset (0, 0), `crop_dx % 4 != 0` turns pointwise programs into C_GENERIC) and the
second source of fused Mixup (the cluster kernel alone, both bands staged within 150 KB, no chunk, no scratch image).
Each case runs through both launch paths (FAA_SPLIT_MIN 0 and huge) and asserts the planner's launch count for every
call.

References: the policy output of every image comes from oracle.pil_path.PolicyTransform (up to 640 px, the whole
`test_gpu_fastpaths._policies()` list) or from the host build of the kernels (above 640 px, the reduced list; a sample
of 8 must equal the oracle).  The rest of the chain is torchvision and torch: F.pad(fill=0) and F.crop at each record's
offset, the flip, the exact ToTensor + Normalize table, the CutoutDefault box, and for Mixup
`A * f32(lam) + A[perm] * f32(1 - lam)` (aug_mixup.py:21) on those fp32 tensors.  fp32 is exact; fp16 / bf16 is the
fp32 value rounded once.  No GPU result is its own reference.
"""
import dataclasses
import functools
import random

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from torchvision import transforms as T

import geometry_cases as G
from helpers import exact_norm_table, philox_reference, reference_output, seed_all, synth_batch
from test_gpu_fastpaths import _policies
from test_gpu_geometries import MEAN, SPLIT, STD, U8, _bad, _big_batch, _device_input, _launches, _records, _reduced

from fast_autoaugment_b200 import archive
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec, augment_batch, augment_tta
from oracle import pil_path

pytestmark = pytest.mark.gpu

FLOATS = (torch.float32, torch.float16, torch.bfloat16)


@functools.lru_cache(maxsize=1)
def _policy_output(shape, emu):
    """(policies, input batch, records, boxes, uint8 policy output [n, H, W, 3] before the tail) of one input shape.  The
    records are the oracle's draws, image i runs policies[i] and odd images are mirrored; the caller sets the crop
    offsets and the CutoutDefault boxes.  The cases run sorted by shape, so a shape's oracle work is done once."""
    H, W = shape
    if max(shape) <= 640:
        policies = _policies()
        batch = synth_batch(len(policies), shape, seed=H * 5 + W)
        samples, boxes, want = _records(policies, batch, range(len(policies)))
    else:
        policies, batch = _big_batch(_reduced(), shape, seed=H + 5 * W)
        sample = sorted(random.Random(H * W).sample(range(len(policies)), 8))
        samples, boxes, oracle = _records(policies, batch, set(sample))
        want = reference_output(emu, CompiledPolicy(policies), batch, U8, samples, boxes).numpy()
        for i in sample:
            assert np.array_equal(want[i], oracle[i]), (shape, i, policies[i])
    u8 = np.stack([want[i][:, ::-1] if i & 1 else want[i] for i in range(len(policies))])     # the flip is the tail's
    return policies, batch, samples, boxes, torch.from_numpy(u8)


def _crop_records(samples, shape, out, pad, reach=(), seed=0):
    """records with crop offsets over [-pad, H + pad - oh] x [-pad, W + pad - ow] and a CutoutDefault box per image:
    every fourth image at (0, 0) (octet and quad paths in one launch); two in four at the ends of the range, at the
    `reach` values, +-1 and every residue of crop_dx mod 4 in both signs; the rest uniform.  With reach, the range is
    [-max(reach), max(reach)] whatever the padding."""
    (H, W), (oh, ow) = shape, out
    n = len(samples)
    lo_y, hi_y, lo_x, hi_x = -pad, H + pad - oh, -pad, W + pad - ow
    if reach:
        lo_y = lo_x = -max(reach)
        hi_y = hi_x = max(reach)
    rng = np.random.default_rng(seed)

    def ends(lo, hi):
        v = [lo, hi] + [s * r for r in reach for s in (-1, 1)] + [0, -1, 1, -2, 2, -3, 3, -4, 4]
        return [x for x in dict.fromkeys(v) if lo <= x <= hi]
    sy, sx = ends(lo_y, hi_y), ends(lo_x, hi_x)
    s = samples.copy()
    for i in range(n):
        if i % 4 == 0:
            dy = dx = 0
        elif i % 4 < 3:                         # (crop_dx shifts by one each round: other pairs, the other flip)
            j = 2 * (i // 4) + i % 4 - 1
            dy, dx = sy[j % len(sy)], sx[(j + j // len(sx)) % len(sx)]
        else:
            dy, dx = int(rng.integers(lo_y, hi_y + 1)), int(rng.integers(lo_x, hi_x + 1))
        s[i]["crop_dy"], s[i]["crop_dx"] = dy, dx
        cy, cx = (37 * i) % oh, (53 * i) % ow
        s[i]["zero_box"] = (max(0, cy - 8), min(oh, cy + 8), max(0, cx - 8), min(ow, cx + 8))
    assert set(sy) <= set(s["crop_dy"].tolist()) and set(sx) <= set(s["crop_dx"].tolist())
    return s


def _tail_reference(u8, samples, out, tab=None):
    """the chain after the policy, on the device: RandomCrop as torchvision's F.pad(fill=0) by the records' largest reach
    and F.crop at each record's offset, then the flip.  u8: the policy output [n, H, W, 3].  Without `tab` the uint8
    HWC result [n, oh, ow, 3]; with the exact ToTensor + Normalize table the fp32 [n, 3, oh, ow] result with each
    record's CutoutDefault box zeroed."""
    n, H, W, _ = u8.shape
    oh, ow = out
    dy, dx = samples["crop_dy"].astype(np.int64), samples["crop_dx"].astype(np.int64)
    p = int(max(0, -dy.min(), -dx.min(), (dy + oh - H).max(), (dx + ow - W).max()))
    padded = F.pad(u8.permute(0, 3, 1, 2), [p], fill=0)
    x = torch.stack([F.crop(padded[i], int(dy[i]) + p, int(dx[i]) + p, oh, ow) for i in range(n)])
    del padded
    flip = torch.from_numpy(samples["flip"] != 0).to(x.device)[:, None, None, None]
    x = torch.where(flip, x.flip(-1), x)
    if tab is None:
        return x.permute(0, 2, 3, 1).contiguous()
    v = torch.stack([tab[c][x[:, c].long()] for c in range(3)], 1)
    for i, (y0, y1, x0, x1) in enumerate(samples["zero_box"].tolist()):
        v[i, :, y0:y1, x0:x1] = 0
    return v


class _Calls:
    """augment_batch calls of one case; the launch count of every call is checked against the planner's"""

    def __init__(self, case, policies, x, monkeypatch):
        self.case, self.pol, self.x, self.mp = case, CompiledPolicy(policies), x, monkeypatch
        self.errors = []

    def run(self, path, what, want_n, want, tail, samples, boxes, **kw):
        self.mp.setenv("FAA_SPLIT_MIN", SPLIT[path])
        n0 = _launches()
        got = augment_batch(self.pol, kw.pop("x", self.x), tail, samples, boxes, **kw)
        if _launches() - n0 != want_n:
            self.errors.append((path, what, "launches", _launches() - n0, want_n))
        bad = _bad(got, want)
        if bad:
            self.errors.append((path, what, len(bad), bad[:6]))

    def done(self):
        assert not self.errors, (self.case.id, self.case.regime, self.errors)


def _check_crop(case, emu, monkeypatch, reach=()):
    policies, batch, samples, boxes, pout = _policy_output(case.shape, emu)
    s = _crop_records(samples, case.shape, case.out, case.pad, reach, seed=case.shape[0] + case.pad)
    tab = torch.from_numpy(exact_norm_table(MEAN, STD)).cuda()
    pd = pout.cuda()
    no_box = s.copy()
    no_box["zero_box"] = 0
    want_u8 = _tail_reference(pd, s, case.out)
    want = _tail_reference(pd, s, case.out, tab)
    want_no_box = _tail_reference(pd, no_box, case.out, tab)
    del pd
    run = _Calls(case, policies, _device_input(batch, case.in_off), monkeypatch)
    u8_split = dataclasses.replace(case, u8=True).plan(emu).launches()
    for path in SPLIT:
        n_float = case.launches if path == "split" else 2
        for dt in FLOATS:
            run.run(path, str(dt), n_float, want.to(dt), TailSpec(case.out, case.pad, True, MEAN, STD, 16, dt), s, boxes)
        # and without CutoutDefault
        run.run(path, "fp32 without a box", n_float, want_no_box, TailSpec(case.out, case.pad, True, MEAN, STD, 0, torch.float32),
                no_box, boxes)
        run.run(path, "uint8", u8_split if path == "split" else 2, want_u8,
                TailSpec(case.out, case.pad, True, MEAN, STD, 0, torch.uint8), s, boxes)
    run.done()


def _mix_pairings(n):
    """(name, partner of each image, lam): a random permutation with a Beta(0.2) draw (aug_mixup.py:19-20), the identity,
    lam = 1 and lam = 0.5"""
    g = torch.Generator().manual_seed(n)
    perm = torch.randperm(n, generator=g)
    lam = float(np.random.default_rng(n).beta(0.2, 0.2))
    lam = max(lam, 1.0 - lam)
    assert 0.5 < lam < 1.0
    return [("permutation", perm, lam), ("identity", torch.arange(n), lam), ("lam 1", perm, 1.0), ("lam 0.5", perm, 0.5)]


def _mixed(a, b, lam):
    return a * np.float32(lam) + b * np.float32(1 - lam)


def _check_mix(case, emu, monkeypatch):
    policies, batch, samples, boxes, pout = _policy_output(case.shape, emu)
    n = len(policies)
    s = _crop_records(samples, case.shape, case.out, case.pad, seed=case.shape[0] + case.pad)
    if not case.pad:                                # without a crop every record's offset is (0, 0)
        s["crop_dy"] = s["crop_dx"] = 0
    tab = torch.from_numpy(exact_norm_table(MEAN, STD)).cuda()
    a = _tail_reference(pout.cuda(), s, case.out, tab)                  # each source's flip, crop and box
    x = _device_input(batch, case.in_off)
    run = _Calls(case, policies, x, monkeypatch)
    pairings = _mix_pairings(n)
    for name, partner, lam in pairings:
        want = _mixed(a, a[partner.cuda()], lam)
        for path in SPLIT:
            run.run(path, name, case.launches, want, TailSpec(case.out, case.pad, True, MEAN, STD, 16, torch.float32), s, boxes,
                    partner=partner, lam=lam)
        if name == "permutation":
            for dt in FLOATS[1:]:
                run.run("split", name + " " + str(dt), case.launches, want.to(dt),
                        TailSpec(case.out, case.pad, True, MEAN, STD, 16, dt), s, boxes, partner=partner, lam=lam)
        del want
    # pool-indexed (the single-GPU form of the multi-GPU route): this batch is pool[first:first + B], partners anywhere
    first, B = n // 4, n // 2
    partner = torch.randint(0, n, (B,), generator=torch.Generator().manual_seed(n + 1))
    assert ((partner < first) | (partner >= first + B)).any()
    lam = pairings[0][2]
    run.run("split", "pool", case.launches, _mixed(a[first:first + B], a[partner.cuda()], lam),
            TailSpec(case.out, case.pad, True, MEAN, STD, 16, torch.float32), None, None, x=x[first:first + B], pool=x,
            pool_samples=s, pool_boxes=boxes, partner=partner, lam=lam, first=first)
    run.done()


def _by_shape(cases):
    return sorted(cases, key=lambda c: (c.shape, c.id))


# (the uint8 crop case is the uint8 output every crop case runs)
_SMALL = _by_shape([c for c in G.CROP_CASES + G.MIX_CASES if not c.big and not c.u8])
_BIG = _by_shape([c for c in G.CROP_CASES + G.MIX_CASES if c.big])


@pytest.mark.parametrize("case", _SMALL, ids=lambda c: c.id)
def test_crop_and_mixup_launches_match_the_oracle(case, emu, monkeypatch):
    (_check_mix if case.two_src else _check_crop)(case, emu, monkeypatch)


@pytest.mark.parametrize("case", _BIG, ids=lambda c: c.id)
def test_crop_and_mixup_launches_match_the_host_build_at_large_sizes(case, emu, monkeypatch):
    (_check_mix if case.two_src else _check_crop)(case, emu, monkeypatch)


def test_crop_records_beyond_the_tails_padding(emu, monkeypatch):
    """the tail's crop_pad is a hint that sizes the staged bands: records of a launch with padding 4 that reach 20 and 127
    pixels read the rows outside the staged copy from global memory and must give the same result"""
    case = next(c for c in G.CROP_CASES if c.id == "crop_224x224_pad4")
    _check_crop(case, emu, monkeypatch, reach=(20, 127))


@pytest.mark.parametrize("shape,out,pad", [((224, 224), (224, 224), 16), ((256, 256), (224, 224), 8)])
def test_randomcrop_draws_match_torchvision_beyond_cifar(shape, out, pad, emu, monkeypatch):
    """policy -> T.RandomCrop(out, padding=pad) -> flip -> ToTensor -> Normalize -> CutoutDefault on seeded generators
    against CompiledPolicy.sample_parity with the same tail: the order of the crop draws among the others, on multi-band
    launches"""
    policies = archive.fa_resnet50_rimagenet()
    n = 96
    batch = synth_batch(n, shape, seed=shape[0] + pad)
    chain = T.Compose([pil_path.PolicyTransform(policies), T.RandomCrop(out, padding=pad), T.RandomHorizontalFlip(),
                       T.ToTensor(), T.Normalize(MEAN, STD), pil_path.ZeroBoxCutout(16)])
    seed_all(13)
    want = pil_path.run_chain_on_batch(chain, batch).cuda()
    tail = TailSpec(out, pad, True, MEAN, STD, 16, torch.float32)
    pol = CompiledPolicy(policies)
    seed_all(13)
    samples, boxes = pol.sample_parity(n, shape[0], shape[1], tail)
    assert len(set(samples["crop_dx"].tolist())) > 8 and (samples["crop_dx"] % 4 != 0).any()
    case = G.TailCase(shape, out, pad, "", 0, "")
    run = _Calls(case, policies, torch.from_numpy(batch).cuda(), monkeypatch)
    for path in SPLIT:
        run.run(path, "parity draws", case.plan(emu, n).launches() if path == "split" else 2, want, tail, samples, boxes)
    run.done()


@pytest.mark.parametrize("B", [4096, 8192])
def test_cifar_philox_calls_split_with_crops(B, emu, monkeypatch):
    """CIFAR at B >= 4096 (4 M pixels): FusedAugmenter with overlap_calls runs resolve + light + cluster kernels with
    crops on the chained schedule - three calls back to back (the first resolves its batch and the next one ahead, the
    others hit), then one run_many over the same batches - against helpers.philox_reference"""
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    pol = CompiledPolicy(archive.fa_reduced_cifar10())
    tail = TailSpec.cifar(16, torch.float16)
    p = G.plan(emu, 32, 32, B, crop_pad=4, philox=True, allow_ahead=True)
    assert p.split and p.use_chain
    pixel = p.launches() - 1                                            # pixel kernels per call
    aug = FusedAugmenter(pol, tail, 32, 32, seed=21, overlap_calls=True)
    xs = [synth_batch(B, (32, 32), seed=60 + k) for k in range(3)]
    xd = [torch.from_numpy(x).cuda() for x in xs]
    outs = [aug.empty_out(B) for _ in range(3)]
    counts = []
    for k in range(3):
        n0 = _launches()
        aug(xd[k], outs[k], 1000 + k * B)
        counts.append(_launches() - n0)
    torch.cuda.synchronize()
    assert counts == [pixel + 2, pixel + 1, pixel + 1], counts
    wants = [philox_reference(emu, pol, xs[k], tail, 21, 1000 + k * B) for k in range(3)]
    for k in range(3):
        bad = _bad(outs[k].cpu(), wants[k])
        assert not bad, ("call", B, k, bad[:8])
    many = [aug.empty_out(B) for _ in range(3)]
    n0 = _launches()
    aug.run_many(aug.plan_many(xd, many), 1000)
    torch.cuda.synchronize()
    assert _launches() - n0 == 3 * pixel + 4                           # a miss, then two hits
    for k in range(3):
        bad = _bad(many[k].cpu(), wants[k])
        assert not bad, ("run_many", B, k, bad[:8])


def test_cifar_tta_splits_with_crops(emu, monkeypatch):
    """augment_tta of 1024 CIFAR images x 5 replicas: 5120 entries split into resolve + light + cluster kernels with
    crops; replica r equals the plain launch of samples first_index + r * B + i"""
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    B, R = 1024, 5
    pol = CompiledPolicy(archive.fa_reduced_cifar10())
    tail = TailSpec.cifar(16, torch.float16)
    p = G.plan(emu, 32, 32, B * R, crop_pad=4, philox=True, allow_ahead=True)
    assert p.split and p.use_chain
    x = synth_batch(B, (32, 32), seed=70)
    n0 = _launches()
    got = augment_tta(pol, torch.from_numpy(x).cuda(), tail, R, seed=9, first_index=3000)
    torch.cuda.synchronize()
    assert _launches() - n0 == p.launches() + 1                         # + the next call's resolve
    want = philox_reference(emu, pol, x, tail, 9, 3000, replicas=R)
    bad = _bad(got.cpu().flatten(0, 1), want.flatten(0, 1))
    assert not bad, bad[:8]
