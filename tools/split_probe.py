import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, bench
from fast_autoaugment_b200.engine import CompiledPolicy, FusedAugmenter, TailSpec
H=W=224; B=512
x = [torch.from_numpy(bench.synth_batch(B, H, W, 1 + i)).cuda() for i in range(4)]
tail = TailSpec.imagenet(0, torch.float16)
for name, p in (("identity", 0.0), ("Invert", 1.0), ("Contrast", 1.0), ("AutoContrast", 1.0), ("Rotate", 1.0)):
    pol = CompiledPolicy([[(name if p else "Invert", p, 0.7), ("Invert", 0.0, 0.7)]])
    f = FusedAugmenter(pol, tail, H, W, 1)
    outs = [f.empty_out(B) for _ in range(4)]
    for i in range(5): f(x[i % 4], outs[i % 4], i * B)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(100): f(x[i % 4], outs[i % 4], i * B)
    e1.record(); torch.cuda.synchronize()
    print("%-13s %7.1f us" % (name, e0.elapsed_time(e1) * 10), flush=True)
