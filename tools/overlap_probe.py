#!/usr/bin/env python
"""How much of a step is the per-step barrier (both pixel kernels drain before the next step starts)?
Runs the bench workload (a) as bench.py does - one policy handle, one stream - and (b) alternating between
two handles on two streams, so that consecutive steps have no stream-order dependency and may overlap.
Usage (on an H100): python tools/overlap_probe.py"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from fast_autoaugment_b200 import archive
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec
H, W, B = 224, 224, 512
x = [torch.from_numpy(bench.synth_batch(B, H, W, 1 + i)).cuda() for i in range(4)]
tail = TailSpec.imagenet(0, torch.float16)
f = [FusedAugmenter(CompiledPolicy(archive.fa_resnet50_rimagenet()), tail, H, W, 1) for _ in range(2)]
outs = [f[0].empty_out(B) for _ in range(4)]
streams = [torch.cuda.Stream(), torch.cuda.Stream()]


def run(n, two):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        k = (i & 1) if two else 0
        f[k](x[i % 4], outs[i % 4], i * B, streams[k].cuda_stream)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e6


for two in (False, True):
    run(20, two)
    for n in (20, 200, 1000):
        print("%-28s steps %4d  %7.1f us/step (wall clock)" % ("two handles, two streams" if two else "one handle, one stream", n, run(n, two)), flush=True)
