#!/usr/bin/env python
"""Time the bench workload's policy mix (224x224 b512, fp16)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from fast_autoaugment_b200 import archive
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec
H, W, B = 224, 224, 512
x = [torch.from_numpy(bench.synth_batch(B, H, W, 1 + i)).cuda() for i in range(4)]
pol = CompiledPolicy(archive.fa_resnet50_rimagenet())
tail = TailSpec.imagenet(0, torch.float16)
f = FusedAugmenter(pol, tail, H, W, 1, overlap_calls=True)
outs = [f.empty_out(B) for _ in range(4)]
for i in range(5): f(x[i % 4], outs[i % 4], i * B)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
n = int(os.environ.get("MIX_N", "1000"))
e0.record()
for i in range(n): f(x[i % 4], outs[i % 4], i * B)
e1.record(); torch.cuda.synchronize()
us = e0.elapsed_time(e1) * 1e3 / n
peak = bench.hbm_peak()[0]
print("%7.1f us  %5.1f%% of %.0f GB/s" % (us, 100 * B * H * W * 9 / us / 1e3 / peak, peak), flush=True)
