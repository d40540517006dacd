"""The policy kernels at every launch geometry the planner can choose, against the oracle.

tests/geometry_cases.py holds one case per planner regime (TMA staging on / off and why, the light kernel's band
staged or not, the materialisation chunk, the octet paths, the mid kernel's bands and threads, the cluster kernel
launched or not) plus the sizes the ImageNet loaders feed the policy: the EfficientNet sizes, source photos and the
header's size limits.  Each case runs through both launch paths (FAA_SPLIT_MIN 0: the split kernels; huge: the cluster
kernel alone), writes uint8 HWC, fp32, fp16 and bf16 and one CutoutDefault pass, and asserts the planner's launch
count for every call, so that no case can quietly run another schedule than the one it claims.

References: up to 640 px every image of the `test_gpu_fastpaths._policies()` list must equal
oracle.pil_path.PolicyTransform.  Above that a reduced list with every program class runs, every image must equal the
host build of the kernels (tests/emu) and a sample of at least 8 must equal the oracle.  fp32 is the exact
normalisation table applied to those bytes; fp16 / bf16 is that value rounded once.  No GPU result is its own reference.
"""
import random

import numpy as np
import PIL.Image
import pytest
import torch

import geometry_cases as G
from helpers import exact_norm_table, philox_reference, reference_output, seed_all, synth, synth_batch
from test_gpu_fastpaths import _policies

from fast_autoaugment_b200 import _lib, archive
from fast_autoaugment_b200.engine import (IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, FusedAugmenter, TailSpec,
                                          augment_batch, make_rng)
from oracle import pil_path

pytestmark = pytest.mark.gpu

SPLIT = {"split": "0", "cluster": "1000000000000"}
MEAN, STD = IMAGENET_MEAN, IMAGENET_STD
U8 = TailSpec(None, 0, True, MEAN, STD, 0, torch.uint8)


def _launches():
    return int(_lib.lib.faa_launch_count())


def _reduced():
    """at least one program of every class (faa_core.cuh build_prog), each op at least once; odd images are mirrored"""
    return [
        [("Invert", 0.0, 0.5), ("Solarize", 0.0, 0.5)],                 # C_PLAIN (nothing applied)
        [("Solarize", 1.0, 0.4), ("Posterize", 1.0, 0.6)],              # C_LUT
        [("Invert", 1.0, 0.0), ("Posterize2", 1.0, 0.3)],               # C_LUT
        [("Color", 1.0, 0.8), ("Brightness", 1.0, 0.3)],                # C_POINT
        [("Cutout", 1.0, 0.6), ("CutoutAbs", 1.0, 0.9)],                # C_POINT
        [("Rotate", 1.0, 0.7), ("Invert", 1.0, 0.0)],                   # C_GEOM
        [("Color", 1.0, 0.2), ("TranslateX", 1.0, 0.8)],                # C_GEOM
        [("ShearX", 1.0, 0.6), ("TranslateY", 1.0, 0.7)],               # C_GEOM2 (lean gathers) / C_GENERIC
        [("TranslateXAbs", 1.0, 0.9), ("ShearY", 1.0, 0.2)],            # C_GEOM2 / C_GENERIC
        [("Equalize", 1.0, 0.5), ("ShearY", 1.0, 0.4)],                 # statistics LUT -> gather
        [("AutoContrast", 1.0, 0.5), ("Rotate", 1.0, 0.3)],             # statistics LUT -> gather
        [("Contrast", 1.0, 0.9), ("TranslateYAbs", 1.0, 0.6)],          # statistics LUT -> gather
        [("Sharpness", 1.0, 0.9), ("Color", 1.0, 0.4)],                 # Sharpness-first two-stage
        [("Sharpness", 1.0, 0.1), ("Cutout", 1.0, 0.5)],                # Sharpness-first two-stage
        [("Sharpness", 1.0, 0.7), ("Posterize", 1.0, 0.2)],             # C_SHARP
        [("Rotate", 1.0, 0.3), ("Equalize", 1.0, 0.5)],                 # C_MAT (gather, then a histogram op)
        [("Color", 1.0, 0.6), ("Sharpness", 1.0, 0.8)],                 # C_MAT (then Sharpness)
        [("ShearX", 1.0, 0.2), ("Contrast", 1.0, 0.3)],                 # C_MAT
        [("Solarize", 1.0, 0.5), ("AutoContrast", 1.0, 0.5)],           # LUT -> histogram (pushed forward)
        [("Sharpness", 1.0, 0.95), ("TranslateX", 1.0, 0.6)],           # C_SG
        [("Sharpness", 1.0, 0.3), ("Rotate", 1.0, 0.9)],                # C_SG
        [("Sharpness", 1.0, 0.2), ("Sharpness", 1.0, 0.9)],             # C_MAT / C_GENERIC without a chunk
        [("Equalize", 1.0, 0.5), ("Equalize", 1.0, 0.5)],               # C_MAT / C_GENERIC
        [("Cutout", 1.0, 0.9), ("Rotate", 1.0, 0.1)],                   # C_GEOM with a box
        [("Equalize", 1.0, 0.5), ("Invert", 0.0, 0.5)],                 # single statistics op
        # C_LUT with a luma mean in slot 1: without a chunk its statistics are taken lazily through op 0's records
        # (the kernel once left those records unset for C_LUT programs: wrong means at W > 1820)
        [("Brightness", 1.0, 0.95), ("Contrast", 1.0, 0.05)],
        [("Equalize", 1.0, 0.5), ("Contrast", 1.0, 0.8)],
        [("Contrast", 1.0, 0.2), ("Contrast", 1.0, 0.9)],
    ]


def _records(policies, batch, oracle_idx):
    """per-image parity records (image i runs policies[i], odd images mirrored) and the oracle's uint8 result of the
    images in oracle_idx (the same draws: PolicyTransform consumes the generators like sample_parity)"""
    n, H, W = batch.shape[0], batch.shape[1], batch.shape[2]
    seed_all(4)
    want = {}
    for i in range(n):
        out = np.asarray(pil_path.PolicyTransform([policies[i]])(PIL.Image.fromarray(batch[i])))
        if i in oracle_idx:
            want[i] = out[:, ::-1] if i & 1 else out
    seed_all(4)
    ss, bb = [], []
    for i in range(n):
        s, b = CompiledPolicy([policies[i]]).sample_parity(1, H, W)
        s["sub"], s["flip"] = i, i & 1
        ss.append(s)
        bb.append(b)
    return np.concatenate(ss), np.concatenate(bb), want


def _at_offset(shape, dtype, offset_bytes):
    """a contiguous CUDA tensor that starts `offset_bytes` past a 256-byte aligned allocation"""
    esize = torch.empty((), dtype=dtype).element_size()
    assert offset_bytes % esize == 0
    n = int(np.prod(shape))
    k = offset_bytes // esize
    return torch.empty(n + k, dtype=dtype, device="cuda")[k:].view(shape)


def _bad(got, want):
    """indices of the images that differ"""
    return (got != want).flatten(1).any(1).nonzero().flatten().tolist()


class _Run:
    """all output types of one case through both launch paths, against one uint8 reference"""

    def __init__(self, emu, case, pol, x, samples, boxes, want_u8, monkeypatch):
        self.emu, self.case, self.pol, self.x, self.samples, self.boxes = emu, case, pol, x, samples, boxes
        self.want_u8 = want_u8                                          # [n, H, W, 3] uint8 on the device
        self.mp = monkeypatch
        tab = torch.from_numpy(exact_norm_table(MEAN, STD)).cuda()
        self.want = torch.stack([tab[c][want_u8[..., c].long()] for c in range(3)], 1)     # exact fp32
        self.errors = []

    def expected(self, path, u8):
        H, W = self.case.shape
        n = self.x.shape[0]
        if path == "cluster":
            return 2
        if u8:           # uint8 output splits only through the octet paths
            return G.plan(self.emu, H, W, n, u8=True, in_off=self.case.in_off, split_min=0).launches()
        return self.case.launches

    def call(self, path, tail, samples, out=None):
        n0 = _launches()
        got = augment_batch(self.pol, self.x, tail, samples, self.boxes, out=out)
        want_n = self.expected(path, tail.out_dtype == torch.uint8)
        if _launches() - n0 != want_n:
            self.errors.append((path, str(tail.out_dtype), "launches", _launches() - n0, want_n))
        return got

    def check(self, dtypes, cutout=True, u8=True):
        n, H, W = self.x.shape[0], self.x.shape[1], self.x.shape[2]
        for path, split_min in SPLIT.items():
            self.mp.setenv("FAA_SPLIT_MIN", split_min)
            for dt in dtypes:
                tail = TailSpec(None, 0, True, MEAN, STD, 0, dt)
                out = _at_offset((n, 3, H, W), dt, self.case.out_off) if self.case.out_off else None
                got = self.call(path, tail, self.samples, out)
                bad = _bad(got, self.want.to(dt))
                if bad:
                    self.errors.append((path, str(dt), len(bad), bad[:6]))
                del got
            if u8:
                got = self.call(path, U8, self.samples)
                bad = _bad(got, self.want_u8)
                if bad:
                    self.errors.append((path, "uint8", len(bad), bad[:6]))
                del got
            if cutout:                                                  # CutoutDefault(16) on top
                s = self.samples.copy()
                want = self.want.clone()
                for i in range(n):
                    cy, cx = (37 * i) % H, (53 * i) % W
                    zb = (max(0, cy - 8), min(H, cy + 8), max(0, cx - 8), min(W, cx + 8))
                    s[i]["zero_box"] = zb
                    want[i, :, zb[0]:zb[1], zb[2]:zb[3]] = 0
                got = self.call(path, TailSpec(None, 0, True, MEAN, STD, 16, torch.float32), s)
                bad = _bad(got, want)
                if bad:
                    self.errors.append((path, "cutout fp32", len(bad), bad[:6]))
                del got, want
        assert not self.errors, (self.case.id, self.case.regime, self.errors)


def _device_input(batch, in_off):
    if not in_off:
        return torch.from_numpy(batch).cuda()
    x = _at_offset(batch.shape, torch.uint8, in_off)
    x.copy_(torch.from_numpy(batch))
    return x


def _dtypes(case):
    # an output offset of 8 bytes is only acceptable for 2-byte outputs
    return (torch.float16, torch.bfloat16) if case.out_off else (torch.float32, torch.float16, torch.bfloat16)


@pytest.mark.parametrize("case", [c for c in G.CASES if not c.big], ids=lambda c: c.id)
def test_policy_kernels_match_the_oracle(case, emu, monkeypatch):
    H, W = case.shape
    policies = _policies()
    n = len(policies)
    batch = synth_batch(n, case.shape, seed=H * 7 + W)
    samples, boxes, want = _records(policies, batch, range(n))
    want_u8 = torch.from_numpy(np.stack([want[i] for i in range(n)])).cuda()
    x = _device_input(batch, case.in_off)
    del batch, want
    run = _Run(emu, case, CompiledPolicy(policies), x, samples, boxes, want_u8, monkeypatch)
    run.check(_dtypes(case), cutout=not case.out_off, u8=not case.out_off)


def _big_batch(policies, shape, seed):
    """one image per program of the reduced list, the input families (noise, ramp, constant) in turn"""
    rng = np.random.default_rng(seed)
    return policies, np.stack([synth(shape, i % 3, rng) for i in range(len(policies))])


@pytest.mark.parametrize("case", [c for c in G.CASES if c.big and c.shape != (8192, 8192)], ids=lambda c: c.id)
def test_policy_kernels_match_the_host_build_at_large_sizes(case, emu, monkeypatch):
    H, W = case.shape
    policies, batch = _big_batch(_reduced(), case.shape, seed=H + 3 * W)
    n = len(policies)
    sample = sorted(random.Random(H * W).sample(range(n), 8))
    samples, boxes, oracle = _records(policies, batch, set(sample))
    pol = CompiledPolicy(policies)
    ref = reference_output(emu, pol, batch, U8, samples, boxes)          # every image: the host build
    for i in sample:                                                     # ... which equals the oracle on the sample
        assert np.array_equal(ref[i].numpy(), oracle[i]), (case.id, i, policies[i])
    x = _device_input(batch, case.in_off)
    del batch
    run = _Run(emu, case, pol, x, samples, boxes, ref.cuda(), monkeypatch)
    limit = case.shape in G.LIMIT_SHAPES
    run.check((torch.float16,) if limit else _dtypes(case), cutout=not limit)


def test_statistics_ops_over_67_million_pixels(emu, monkeypatch):
    """four 8192 x 8192 images (the header's limit) per launch, single ops: the histogram and luma-sum ops on ramp and
    constant images put 67 M pixels into one histogram; uint8 and fp16 output against the oracle"""
    H = W = 8192
    case = next(c for c in G.CASES if c.shape == (H, W))
    rng = np.random.default_rng(8)
    batch = np.stack([synth((H, W), k, rng) for k in (1, 2, 1, 2)])      # ramp, constant, ramp, constant
    for ops in (["Equalize", "AutoContrast", "Contrast", "Equalize"], ["AutoContrast", "Contrast", "Rotate", "Sharpness"]):
        policies = [[(op, 1.0, 0.7), ("Invert", 0.0, 0.0)] for op in ops]
        samples, boxes, want = _records(policies, batch, range(4))
        want_u8 = torch.from_numpy(np.stack([want[i] for i in range(4)])).cuda()
        del want
        run = _Run(emu, case, CompiledPolicy(policies), torch.from_numpy(batch).cuda(), samples, boxes, want_u8, monkeypatch)
        run.check((torch.float16,), cutout=False)
        del run, want_u8
        torch.cuda.empty_cache()


@pytest.mark.parametrize("shape,B,dtype", [((240, 240), 96, torch.float16), ((456, 456), 32, torch.float16),
                                           ((600, 600), 16, torch.float16), ((375, 500), 64, torch.uint8)])
def test_production_philox_calls_back_to_back(shape, B, dtype, emu, monkeypatch):
    """FusedAugmenter with overlap_calls: three calls on one stream without a synchronize (the first resolves its batch
    and the next one ahead, the others hit), at the EfficientNet sizes in fp16 and at a source photo in uint8 - the
    policy stage of ImageNetChain - against helpers.philox_reference"""
    monkeypatch.delenv("FAA_SPLIT_MIN", raising=False)
    H, W = shape
    pol = CompiledPolicy(archive.fa_resnet50_rimagenet())
    tail = U8 if dtype == torch.uint8 else TailSpec.imagenet(0, dtype)
    aug = FusedAugmenter(pol, tail, H, W, seed=21, overlap_calls=True)
    xs = [synth_batch(B, shape, seed=40 + k) for k in range(3)]
    xd = [torch.from_numpy(x).cuda() for x in xs]
    outs = [aug.empty_out(B) for _ in range(3)]
    pixel = G.plan(emu, H, W, B, u8=dtype == torch.uint8).launches() - 1    # pixel kernels per call
    counts = []
    for k in range(3):
        n0 = _launches()
        aug(xd[k], outs[k], 1000 + k * B)
        counts.append(_launches() - n0)
    torch.cuda.synchronize()
    # miss: this batch's resolve + the next one's; hit: only the next one's
    assert counts == [pixel + 2, pixel + 1, pixel + 1], counts
    for k in range(3):
        want = philox_reference(emu, pol, xs[k], tail, 21, 1000 + k * B)
        bad = _bad(outs[k].cpu(), want)
        assert not bad, (shape, k, bad[:8])


def test_misaligned_views_are_refused_without_a_launch():
    """contiguous views at an offset the vector paths cannot take raise, and nothing is launched"""
    pol = CompiledPolicy(archive.fa_resnet50_rimagenet())
    B, H, W = 4, 224, 224
    x = torch.from_numpy(synth_batch(B, (H, W), seed=3)).cuda()
    fp32 = TailSpec.imagenet(0, torch.float32)
    r = make_rng(5, 0, fp32)
    cases = [(x, _at_offset((B, 3, H, W), torch.float32, 4), fp32),
             (x, _at_offset((B, 3, H, W), torch.float16, 2), TailSpec.imagenet(0, torch.float16)),
             (x, _at_offset((B, H, W, 3), torch.uint8, 2), U8),
             (_at_offset((B, H, W, 3), torch.uint8, 2).copy_(x), None, fp32)]
    for xin, out, tail in cases:
        n0 = _launches()
        with pytest.raises(_lib.FaaRuntimeError, match="aligned"):
            augment_batch(pol, xin, tail, rng=r, out=out)
        torch.cuda.synchronize()
        assert _launches() == n0
    aug = FusedAugmenter(pol, fp32, H, W, seed=5)
    n0 = _launches()
    with pytest.raises(_lib.FaaRuntimeError, match="16-byte"):
        aug(x, _at_offset((B, 3, H, W), torch.float32, 8), 0)
    assert _launches() == n0
    # the accepted offsets still compute what an aligned launch computes
    ok = augment_batch(pol, x, TailSpec.imagenet(0, torch.float16), rng=r)
    got = augment_batch(pol, x, TailSpec.imagenet(0, torch.float16), rng=r, out=_at_offset((B, 3, H, W), torch.float16, 8))
    assert torch.equal(got, ok)
