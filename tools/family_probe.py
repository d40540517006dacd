#!/usr/bin/env python
"""Device time of single-op policies per input family (noise / ramp / constant): shows how much of a
statistics op's cost is histogram contention.  Usage (on an H100): python tools/family_probe.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from helpers import synth
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec

H = W = 224
B = 512


def batch(kind, seed):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(np.stack([synth((H, W), kind, rng) for _ in range(B)])).cuda()


tail = TailSpec.imagenet(0, torch.float16)
for kind, fam in enumerate(("noise", "ramp", "constant")):
    x = [batch(kind, 10 + i) for i in range(4)]
    for name in ("Invert", "AutoContrast", "Equalize", "Contrast", "Sharpness", "Rotate"):
        pol = CompiledPolicy([[(name, 1.0, 0.7), (name, 0.0, 0.7)]])
        f = FusedAugmenter(pol, tail, H, W, 1, overlap_calls=True)
        outs = [f.empty_out(B) for _ in range(4)]
        for i in range(5):
            f(x[i % 4], outs[i % 4], i * B)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(100):
            f(x[i % 4], outs[i % 4], i * B)
        e1.record()
        torch.cuda.synchronize()
        print("%-9s %-13s %7.1f us" % (fam, name, e0.elapsed_time(e1) * 10), flush=True)
