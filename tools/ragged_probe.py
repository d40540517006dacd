#!/usr/bin/env python
"""CUDA-event timing of the ImageNet chains on batches of differently sized sources (``RaggedImages``).

    python tools/ragged_probe.py [--iters 30]

1. The ragged crop-resize launch (``faa_crop_resize_ragged``) against the uniform ``faa_crop_resize`` on the same
   same-size b512 batches (the three cases of DESIGN.md 4.7), alternated call by call.
2. A b256 train chain over a SYNTHETIC size mixture (not measured from ImageNet: mostly 375x500, 500x375 and 333x500,
   plus a tail of random sizes), stage by stage: the per-size policy groups (positional sampler + policy launches on the
   gathered images), the ragged crop-resize, ColorJitter, the jitter / Lighting records and HFlip + Lighting + Normalize;
   then the whole ``ImageNetChain.train`` call.  Also: policy groups per batch, and the per-size policy tables the
   handle has cached after the run.
4. The ragged policy launch (``augment_batch`` on ``RaggedImages``) against the per-size groups on the same mixture
   (packed back to back and 16-byte aligned), and against the uniform launch on b256 batches of one size (375x500, which
   the uniform launch runs in the cluster kernel, and 480x640, which it splits into the light / mid kernels).

Prints the card's name and power limit from the same run."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast_autoaugment_b200 import _lib, archive, data, engine  # noqa: E402
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, RaggedImages, TailSpec  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def time_us(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def alternated(fns, iters, rounds=5):
    """mean us per call of each fn, timed in `rounds` alternating windows of `iters` calls"""
    for f in fns:
        for _ in range(3):
            f()
    tot = [0.0] * len(fns)
    for _ in range(rounds):
        for k, f in enumerate(fns):
            tot[k] += time_us(f, iters)
    return [t / rounds for t in tot]


def mixture(rng, n):
    """SYNTHETIC source sizes: 40 % 375x500, 25 % 500x375, 20 % 333x500, 15 % random in [64, 1024]^2"""
    out = []
    for u in rng.random(n):
        if u < 0.40:
            out.append((375, 500))
        elif u < 0.65:
            out.append((500, 375))
        elif u < 0.85:
            out.append((333, 500))
        else:
            out.append((int(rng.integers(64, 1025)), int(rng.integers(64, 1025))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print("card: %s, power limit: %s W" % (torch.cuda.get_device_name(0), power_limit()))
    rng = np.random.default_rng(0)
    b = 512
    f16 = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, torch.float16)
    print("\n1. uniform faa_crop_resize vs faa_crop_resize_ragged on the same same-size batch, b512, alternated")
    for name, (h, w), cfg, tail in (("center crop + resize 375x500 -> 224, fp16", (375, 500), engine.crop_cfg(224, center=True), f16),
                                    ("random crop + resize 375x500 -> 224, uint8", (375, 500), engine.crop_cfg(224, seed=1), None),
                                    ("random crop + resize 256x256 -> 224, uint8", (256, 256), engine.crop_cfg(224, seed=1), None)):
        x = torch.from_numpy(rng.integers(0, 256, (b, h, w, 3), dtype=np.uint8)).cuda()
        r = RaggedImages(x.view(-1), np.arange(b, dtype=np.int64) * h * w * 3, [(h, w)] * b)
        dt = torch.uint8 if tail is None else tail.out_dtype
        shape = (b, 224, 224, 3) if dt == torch.uint8 else (b, 3, 224, 224)
        o1, o2 = torch.empty(shape, dtype=dt, device="cuda"), torch.empty(shape, dtype=dt, device="cuda")
        u, g = alternated([lambda: engine.crop_resize(x, 224, rng=cfg, tail=tail, out=o1),
                           lambda: engine.crop_resize(r, 224, rng=cfg, tail=tail, out=o2)], args.iters)
        assert torch.equal(o1, o2)
        print("  %-46s uniform %8.1f us   ragged %8.1f us   (%+.1f %%)" % (name, u, g, 100.0 * (g / u - 1)))
        del x, r, o1, o2

    bb = 256
    sizes = mixture(rng, bb)
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    x = RaggedImages.from_list(imgs)
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float16)
    groups = x.groups()
    print("\n2. train chain, b256, SYNTHETIC size mixture (%d distinct sizes = policy groups in this batch; "
          "%d images in the three common sizes)" % (len(groups), sum(s in ((375, 500), (500, 375), (333, 500)) for s in sizes)))
    for _ in range(2):
        chain.train(x, seed=1, first_index=0)
    raw = TailSpec.raw_u8()
    pol = chain.aug.compiled
    inter = chain._policy_ragged(x, None, 1, 0)
    y = engine.crop_resize(inter, 224, rng=chain.crop.cfg(1, 0))
    recs, rgb = chain._device_records(bb, y.device, 1, 0)
    fin = torch.empty(bb, 3, 224, 224, dtype=torch.float16, device="cuda")
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)  # noqa: E731
    gathered = [torch.stack([x.image(int(i)) for i in pos]) for _, pos in groups]
    steps = [
        ("gather each group's images (torch.stack)", lambda: [torch.stack([x.image(int(i)) for i in pos]) for _, pos in groups]),
        ("positional sampler, all groups", lambda: [engine.sample_philox_at(pol, pos, h, w, raw, engine.make_rng(1, 0, raw), y.device)
                                                    for (h, w), pos in groups]),
        ("policy launches on the gathered groups", lambda: [engine.augment_batch(pol, g_, raw, *engine.sample_philox_at(
            pol, pos, h, w, raw, engine.make_rng(1, 0, raw), y.device)) for g_, ((h, w), pos) in zip(gathered, groups)]),
        ("policy stage as the chain runs it (all of the above)", lambda: chain._policy_ragged(x, None, 1, 0)),
        ("ragged random crop + resize -> 224 uint8", lambda: engine.crop_resize(inter, 224, rng=chain.crop.cfg(1, 0), out=y)),
        ("ColorJitter in place", lambda: _lib.check(_lib.lib.faa_color_jitter(y.data_ptr(), y.data_ptr(), bb, 224, 224,
                                                                              recs.data_ptr(), stream()))),
        ("jitter + Lighting records (torch)", lambda: chain._device_records(bb, y.device, 1, 0)),
        ("HFlip + Lighting + Normalize fp16", lambda: engine.augment_batch(chain.flip_policy, y, chain.tail,
                                                                           rng=engine.make_rng(1, 0, chain.tail), out=fin,
                                                                           lighting_rgb=rgb)),
        ("ImageNetChain.train end to end", lambda: chain.train(x, seed=1, first_index=0)),
    ]
    for name, fn in steps:
        fn()
        print("  %-56s %9.1f us" % (name, time_us(fn, args.iters)))
    n_tab, nbytes = engine.cached_tables(pol)
    print("\n3. per-size policy tables cached by the handle after the run: %d tables, %.1f KB (%.1f KB each; never evicted)"
          % (n_tab, nbytes / 1024, nbytes / 1024 / max(1, n_tab)))

    print("\n4. the ragged policy launch (faa_augment_ragged, uint8 at source size, Philox), alternated call by call")
    rng_raw = engine.make_rng(1, 0, raw)
    xa = RaggedImages.empty(x.sizes)                      # the same images, every one on a 16-byte boundary
    for i in range(bb):
        xa.image(i).copy_(x.image(i))
    for name, src in (("packed back to back (from_list; W % 4 == 0 images re-aligned)", x), ("16-byte aligned images", xa)):
        out = RaggedImages.empty(x.sizes)
        want = chain._policy_ragged(src, None, 1, 0)
        n0 = _lib.lib.faa_launch_count()
        engine.augment_batch(pol, src, raw, rng=rng_raw, out=out)
        torch.cuda.synchronize()
        n_launch = _lib.lib.faa_launch_count() - n0
        assert all(torch.equal(out.image(i), want.image(i)) for i in range(bb))
        grp, rag = alternated([lambda: chain._policy_ragged(src, None, 1, 0),
                               lambda: engine.augment_batch(pol, src, raw, rng=rng_raw, out=out)], args.iters)
        print("  b256 mixture, %-62s per-size groups %8.1f us   ragged %8.1f us (%d launches)" % (name, grp, rag, n_launch))
    for h, w in ((375, 500), (480, 640)):
        xu = torch.from_numpy(rng.integers(0, 256, (bb, h, w, 3), dtype=np.uint8)).cuda()
        r = RaggedImages(xu.view(-1), np.arange(bb, dtype=np.int64) * h * w * 3, [(h, w)] * bb)
        ou, orag = torch.empty_like(xu), RaggedImages.empty(r.sizes)
        uni, rag = alternated([lambda: engine.augment_batch(pol, xu, raw, rng=rng_raw, out=ou),
                               lambda: engine.augment_batch(pol, r, raw, rng=rng_raw, out=orag)], args.iters)
        assert all(torch.equal(orag.image(i), ou[i]) for i in range(bb))
        print("  b256 of one size %dx%d: uniform augment_batch %8.1f us   ragged %8.1f us   (%+.1f %%)"
              % (h, w, uni, rag, 100.0 * (rag / uni - 1)))


if __name__ == "__main__":
    main()
