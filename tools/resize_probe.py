#!/usr/bin/env python
"""CUDA-event timing of faa_crop_resize (EfficientNet crop + bicubic Resize) and of the ImageNet train chain per launch.

    python tools/resize_probe.py [--iters 50]

Per case: mean time per launch, bytes moved (the crop regions' bytes read + the output bytes written) and their share
of the H100 SXM data-sheet bandwidth (3.35 TB/s), with the card's name and power limit from the same run."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast_autoaugment_b200 import _lib, archive, data, engine  # noqa: E402
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, TailSpec  # noqa: E402

PEAK = 3.35e12


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def time_us(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def report(name, us, nbytes):
    print("%-52s %9.1f us  %8.1f MB  %5.1f%% of 3.35 TB/s" % (name, us, nbytes / 1e6, 100.0 * nbytes / (us * 1e-6) / PEAK))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print("card: %s, power limit: %s W" % (torch.cuda.get_device_name(0), power_limit()))
    rng = np.random.default_rng(0)
    b = 512
    src = {(375, 500): torch.from_numpy(rng.integers(0, 256, (b, 375, 500, 3), dtype=np.uint8)).cuda(),
           (256, 256): torch.from_numpy(rng.integers(0, 256, (b, 256, 256, 3), dtype=np.uint8)).cuda()}
    f16 = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, torch.float16)

    x = src[(375, 500)]
    cfg = engine.crop_cfg(224, center=True)
    out = torch.empty(b, 3, 224, 224, dtype=torch.float16, device="cuda")
    cb = engine.center_crop_box(375, 500, 224)
    us = time_us(lambda: engine.crop_resize(x, 224, rng=cfg, tail=f16, out=out), args.iters)
    report("center crop + resize 375x500 -> 224, fp16, b512", us, b * (cb[2] * cb[3] * 3 + 224 * 224 * 3 * 2))

    for (h, w), xx in src.items():
        cfg = engine.crop_cfg(224, seed=1)
        emu_boxes = np.zeros(b, _lib.CROP_BOX_DTYPE)
        try:
            import ctypes as C
            lib = C.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "emu",
                                      "libfaa_emu_resize.so"))
            lib.faa_emu_philox_crop_boxes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
            lib.faa_emu_philox_crop_boxes(C.addressof(cfg), b, h, w, emu_boxes.ctypes.data)
            read = int((emu_boxes["w"].astype(np.int64) * emu_boxes["h"]).sum()) * 3
        except OSError:
            read = None                                     # (the host build of the sampler is not there)
        o8 = torch.empty(b, 224, 224, 3, dtype=torch.uint8, device="cuda")
        us = time_us(lambda: engine.crop_resize(xx, 224, rng=cfg, out=o8), args.iters)
        if read is None:
            print("random crop + resize %dx%d -> 224, uint8, b512: %.1f us (bytes not measured)" % (h, w, us))
        else:
            report("random crop + resize %dx%d -> 224, uint8, b512" % (h, w), us, read + b * 224 * 224 * 3)

    # the train chain at b256, launch by launch (Philox mode)
    bb = 256
    x = src[(375, 500)][:bb].contiguous()
    chain = data.ImageNetChain(archive.fa_resnet50_rimagenet(), 224, torch.float16)
    raw = TailSpec.raw_u8()
    pol = chain.aug.compiled
    pol_out = torch.empty_like(x)
    y = torch.empty(bb, 224, 224, 3, dtype=torch.uint8, device="cuda")
    recs, rgb = chain._device_records(bb, x.device, 1, 0)
    fin = torch.empty(bb, 3, 224, 224, dtype=torch.float16, device="cuda")
    import ctypes as C
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)  # noqa: E731
    steps = [
        ("policy (fa_resnet50_rimagenet) 375x500 uint8", lambda: engine.augment_batch(pol, x, raw, rng=engine.make_rng(1, 0, raw), out=pol_out),
         2 * bb * 375 * 500 * 3),
        ("random crop + resize -> 224 uint8", lambda: engine.crop_resize(pol_out, 224, rng=chain.crop.cfg(1, 0), out=y), None),
        ("ColorJitter in place", lambda: _lib.check(_lib.lib.faa_color_jitter(y.data_ptr(), y.data_ptr(), bb, 224, 224,
                                                                              recs.data_ptr(), stream())), 2 * bb * 224 * 224 * 3),
        ("jitter + Lighting records (torch)", lambda: chain._device_records(bb, x.device, 1, 0), None),
        ("HFlip + Lighting + Normalize fp16", lambda: engine.augment_batch(chain.flip_policy, y, chain.tail,
                                                                           rng=engine.make_rng(1, 0, chain.tail), out=fin,
                                                                           lighting_rgb=rgb), bb * 224 * 224 * 3 * 3),
    ]
    total = 0.0
    for name, fn, nbytes in steps:
        us = time_us(fn, args.iters)
        total += us
        if nbytes:
            report("train b256: " + name, us, nbytes)
        else:
            print("%-52s %9.1f us" % ("train b256: " + name, us))
    print("%-52s %9.1f us" % ("train b256: sum of the launches", total))
    us = time_us(lambda: chain.train(x, seed=1, first_index=0), args.iters)
    print("%-52s %9.1f us" % ("train b256: ImageNetChain.train end to end", us))


if __name__ == "__main__":
    main()
