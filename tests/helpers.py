"""Shared helpers of the test-suite (inputs, emulator driver, comparisons)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")

ALL_OPS = ["ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "AutoContrast", "Invert",
           "Equalize", "Solarize", "Posterize", "Contrast", "Color", "Brightness", "Sharpness",
           "Cutout", "CutoutAbs", "Posterize2", "TranslateXAbs", "TranslateYAbs"]


def synth(shape, kind, rng):
    """The three input families of SURVEY.md 8(d) (same generator as tests/golden/make_golden.py)."""
    h, w = shape
    if kind == 0:
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == 1:
        lo = int(rng.integers(0, 200))
        hi = int(rng.integers(lo + 1, 256))
        ramp = np.linspace(lo, hi, w)[None, :, None] + rng.normal(0, 8, (h, w, 3))
        return np.clip(ramp, 0, 255).astype(np.uint8)
    return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()


def synth_batch(n, shape, seed):
    rng = np.random.default_rng(seed)
    return np.stack([synth(shape, i % 3, rng) for i in range(n)])


def live_input(rng, i, s):
    """input i of a make_golden.py LIVE_CASES run (same generator): noise (odd i) or a low-contrast ramp + noise"""
    if i % 2:
        return rng.integers(0, 256, (s, s, 3), dtype=np.uint8)
    return np.clip(np.linspace(60, 180, s)[None, :, None] + rng.normal(0, 6, (s, s, 3)), 0, 255).astype(np.uint8)


def policy_sha(policies) -> str:
    """digest of a policy table, as make_golden.py stores it for the reference's archive"""
    import hashlib
    import json
    return hashlib.sha256(json.dumps([[list(o) for o in sub] for sub in policies]).encode()).hexdigest()


def exact_norm_table(mean, std):
    """fp32 ToTensor+Normalize value of every byte, computed with torch itself."""
    import torch
    u = torch.arange(256, dtype=torch.uint8)
    x = u.to(torch.float32).div(255)
    m = torch.as_tensor(mean, dtype=torch.float32)[:, None]
    s = torch.as_tensor(std, dtype=torch.float32)[:, None]
    return ((x[None, :] - m) / s).numpy().astype(np.float32).copy()


def emu_augment(emu, pol, batch_u8, samples, boxes, tail=None, norm=None, partner=None, lam=1.0,
                force_generic=False, pool=None, pool_samples=None, pool_boxes=None, first=0):
    """Drive tests/emu like engine.augment_batch drives the kernels.  norm=None -> uint8 HWC."""
    from fast_autoaugment_b200.engine import TailSpec
    tail = tail or TailSpec.raw_u8()
    B, H, W, _ = batch_u8.shape
    oh, ow = tail.out_size if tail.out_size is not None else (H, W)
    table = np.ascontiguousarray(pol.compiled_table(H, W))
    src = np.ascontiguousarray(batch_u8 if pool is None else pool)
    smp = np.ascontiguousarray(samples if pool_samples is None else pool_samples)
    bxs = np.ascontiguousarray(boxes if pool_boxes is None else pool_boxes)
    cur = src
    n_op = pol.n_op
    base = 0
    while base + 2 < n_op:                      # chained windows, like the engine
        nxt = np.zeros_like(cur)
        rc = emu.faa_emu_augment(cur.ctypes.data, cur.shape[0], 0, cur.shape[0], H, W, table.ctypes.data,
                                 pol.n_sub, n_op, smp.ctypes.data, bxs.ctypes.data, base, 0, H, W, 0, None,
                                 nxt.ctypes.data, None, C.c_float(1.0), C.c_float(0.0), int(force_generic))
        assert rc == 0
        cur, base = nxt, base + 2
    if norm is None:
        out = np.zeros((B, oh, ow, 3), np.uint8)
        tab = None
    else:
        out = np.zeros((B, 3, oh, ow), np.float32)
        norm = np.ascontiguousarray(norm, dtype=np.float32)
        tab = norm.ctypes.data
    part = None
    if partner is not None:
        partner = np.ascontiguousarray(partner, dtype=np.int32)
        part = partner.ctypes.data
    rc = emu.faa_emu_augment(cur.ctypes.data, cur.shape[0], first, B, H, W, table.ctypes.data, pol.n_sub, n_op,
                             smp.ctypes.data, bxs.ctypes.data, base, 1, oh, ow, int(tail.cutout > 0), tab,
                             out.ctypes.data, part, C.c_float(np.float32(lam)), C.c_float(np.float32(1 - lam)),
                             int(force_generic))
    assert rc == 0
    return out


def emu_philox_records(emu, pol, n, h, w, tail, seed, first_index):
    """Decision records of samples [first_index, first_index + n) from the emulator's Philox sampler (the kernels'
    sampler compiled for the host): what a fused Philox launch draws for those indices, without a GPU."""
    from fast_autoaugment_b200 import _lib
    from fast_autoaugment_b200.engine import make_rng
    oh, ow = tail.out_size if tail.out_size is not None else (h, w)
    table = np.ascontiguousarray(pol.compiled_table(h, w))
    probs = np.ascontiguousarray(pol.probs, dtype=np.float64)
    rng = make_rng(seed, first_index, tail)
    samples = np.zeros(n, dtype=_lib.SAMPLE_DTYPE)
    boxes = np.zeros((n, pol.n_op), dtype=_lib.BOX_DTYPE)
    rc = emu.faa_emu_philox(table.ctypes.data, probs.ctypes.data, pol.n_sub, pol.n_op, C.addressof(rng), n, h, w, oh, ow,
                            samples.ctypes.data, boxes.ctypes.data)
    assert rc == 0
    return samples, boxes


def reference_output(emu, pol, batch_u8, tail, samples, boxes, lighting_rgb=None, partner=None, lam=1.0, threads=16):
    """Host reference of one launch on resolved records: emu_augment, then the exact ToTensor+Normalize table.  Returns a
    CPU tensor laid out like the launch's output: uint8 [B, oh, ow, 3] for uint8 tails, else [B, 3, oh, ow] in
    tail.out_dtype - fp16 / bf16 being the fp32 value rounded once.  Lighting (lighting_rgb [B, 3]): the uint8 result,
    then ((u / 255 + rgb) - mean) / std in torch fp32.  Images are split over threads (the emulator releases the GIL)."""
    import concurrent.futures
    import torch
    from fast_autoaugment_b200.engine import TailSpec
    B = batch_u8.shape[0]
    u8_out = tail.out_dtype == torch.uint8 or lighting_rgb is not None
    if lighting_rgb is not None:
        assert tail.cutout == 0, "CutoutDefault zeroes the normalised value: not modelled together with Lighting"
        run_tail = TailSpec(tail.out_size, tail.crop_pad, tail.hflip, tail.mean, tail.std, 0, torch.uint8)
    else:
        run_tail = tail
    norm = None if u8_out else exact_norm_table(tail.mean, tail.std)
    if partner is not None:                     # fused Mixup: the partners index the whole batch
        out = emu_augment(emu, pol, batch_u8, samples, boxes, run_tail, norm, partner=partner, lam=lam)
    else:
        step = max(1, -(-B // threads))
        parts = [(lo, min(B, lo + step)) for lo in range(0, B, step)]
        with concurrent.futures.ThreadPoolExecutor(len(parts)) as ex:
            outs = list(ex.map(lambda r: emu_augment(emu, pol, np.ascontiguousarray(batch_u8[r[0]:r[1]]),
                                                     samples[r[0]:r[1]], boxes[r[0]:r[1]], run_tail, norm), parts))
        out = np.concatenate(outs)
    out = torch.from_numpy(out)
    if lighting_rgb is not None:
        t = out.permute(0, 3, 1, 2).float().div(255)
        t = t.add(torch.as_tensor(lighting_rgb, dtype=torch.float32).cpu().view(B, 3, 1, 1).expand_as(t))
        m = torch.tensor(tail.mean, dtype=torch.float32).view(1, 3, 1, 1)
        s = torch.tensor(tail.std, dtype=torch.float32).view(1, 3, 1, 1)
        return ((t - m) / s).to(tail.out_dtype)
    return out if u8_out else out.to(tail.out_dtype)


def philox_reference(emu, pol, batch_u8, tail, seed, first_index, replicas=1, **kw):
    """Host reference of a fused Philox launch (FusedAugmenter, augment_batch(rng=...), run_many steps): records from
    emu_philox_records, pixels from reference_output.  replicas > 1: a TTA launch, replica r draws the samples
    first_index + r * B + i and the result is stacked [replicas, B, ...]."""
    B, H, W, _ = batch_u8.shape
    outs = [reference_output(emu, pol, batch_u8, tail,
                             *emu_philox_records(emu, pol, B, H, W, tail, seed, first_index + r * B), **kw)
            for r in range(replicas)]
    if replicas == 1:
        return outs[0]
    import torch
    return torch.stack(outs)


def set_emu_sigs(emu):
    vp = C.c_void_p
    emu.faa_emu_augment.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp,
                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_float, C.c_float,
                                    C.c_int]
    emu.faa_emu_augment.restype = C.c_int
    emu.faa_emu_philox.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    emu.faa_emu_philox.restype = C.c_int
    emu.faa_emu_philox_block.argtypes = [vp, vp, vp]
    emu.faa_emu_philox_block.restype = None
    emu.faa_emu_plan_fields.restype = C.c_char_p
    emu.faa_emu_plan.argtypes = [C.c_int] * 12 + [C.c_longlong, C.c_int, C.c_int, vp]     # returns the field count
    return emu


def seed_all(s):
    import random
    import torch
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
