#!/usr/bin/env python
"""CIFAR-sized steps (32x32, b512, full train chain): is the step host-bound?  Host enqueue time per call vs device time."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from fast_autoaugment_b200 import archive
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec
B = int(os.environ.get("CIFAR_B", "512"))
x = [torch.from_numpy(bench.synth_batch(B, 32, 32, 1 + i)).cuda() for i in range(4)]
pol = CompiledPolicy(archive.fa_reduced_cifar10())
tail = TailSpec.cifar(16, torch.float16)
f = FusedAugmenter(pol, tail, 32, 32, 1, overlap_calls=True)
outs = [f.empty_out(B) for _ in range(4)]
for i in range(20): f(x[i % 4], outs[i % 4], i * B)
torch.cuda.synchronize()
n = 300
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); t0 = time.perf_counter()
for i in range(n): f(x[i % 4], outs[i % 4], (20 + i) * B)
t1 = time.perf_counter(); e1.record(); torch.cuda.synchronize()
dev_loop = e0.elapsed_time(e1) * 1e3 / n
plan = f.plan_many([x[i % 4] for i in range(n)], [outs[i % 4] for i in range(n)])
f.run_many(plan, 1000 * B); torch.cuda.synchronize()
e0.record(); t2 = time.perf_counter()
f.run_many(plan, 2000 * B)
t3 = time.perf_counter(); e1.record(); torch.cuda.synchronize()
print("run_many: host %6.2f us/step   device %6.2f us/step" % ((t3 - t2) * 1e6 / n, e0.elapsed_time(e1) * 1e3 / n), flush=True)
print("per call: host enqueue %6.2f us/call   device %6.2f us/step" % ((t1 - t0) * 1e6 / n, dev_loop), flush=True)
