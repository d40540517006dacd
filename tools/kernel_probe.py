#!/usr/bin/env python
"""Device-time decomposition of the fused kernel: which program classes cost what.
Usage (on an H100): python tools/kernel_probe.py [H W B]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import bench
from fast_autoaugment_b200 import archive
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec

H, W, B = (int(a) for a in sys.argv[1:4]) if len(sys.argv) >= 4 else (224, 224, 512)
PEAK = bench.hbm_peak()[0]
x = [torch.from_numpy(bench.synth_batch(B, H, W, 1 + i)).cuda() for i in range(4)]


def timeit(name, policies, tail, n=int(os.environ.get("PROBE_N", "200"))):
    pol = CompiledPolicy(policies)
    f = FusedAugmenter(pol, tail, H, W, 1, overlap_calls=True)
    outs = [f.empty_out(B) for _ in range(4)]
    for i in range(5):
        f(x[i % 4], outs[i % 4], i * B)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        f(x[i % 4], outs[i % 4], i * B)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / n
    out_b = outs[0].numel() * outs[0].element_size()
    gbs = (B * H * W * 3 + out_b) / us / 1e3
    print("%-34s %8.1f us  %7.0f GB/s  %5.1f%% of %.0f" % (name, us, gbs, 100 * gbs / PEAK, PEAK), flush=True)


t16 = TailSpec.imagenet(0, torch.float16) if H != 32 else TailSpec.cifar(16, torch.float16)
tnf = TailSpec(None, 0, False, t16.mean, t16.std, 0, torch.float16)
one = lambda name, lv=0.7, p=1.0: [[(name, p, lv), (name, 0.0, lv)]]
timeit("identity (prob 0), no flip", one("Invert", p=0.0), tnf)
timeit("identity (prob 0), flip", one("Invert", p=0.0), t16)
for nm in ("Invert", "Brightness", "Color", "Cutout", "AutoContrast", "Equalize", "Contrast", "TranslateX",
           "ShearX", "ShearY", "Rotate", "Sharpness"):
    timeit("100%% %s" % nm, one(nm), t16)
timeit("fa_resnet50_rimagenet", archive.fa_resnet50_rimagenet(), t16)
timeit("fa_reduced_cifar10", archive.fa_reduced_cifar10(), t16)
timeit("fa_resnet50_rimagenet fp32 out", archive.fa_resnet50_rimagenet(), TailSpec.imagenet(0, torch.float32))
timeit("fa_resnet50_rimagenet u8 out", archive.fa_resnet50_rimagenet(), TailSpec.raw_u8())
