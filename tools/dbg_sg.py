import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ["FAA_SPLIT_MIN"] = "0"
import numpy as np, PIL.Image, torch
from helpers import exact_norm_table, seed_all, synth_batch
from fast_autoaugment_b200.engine import IMAGENET_MEAN, IMAGENET_STD, CompiledPolicy, TailSpec, augment_batch
from oracle import pil_path
tab = torch.from_numpy(exact_norm_table(IMAGENET_MEAN, IMAGENET_STD))
for second in (("TranslateY", 0.1), ("Rotate", 0.3), ("ShearX", 0.9), ("Cutout", 0.5), ("Sharpness", 0.2), ("AutoContrast", 0.5), ("TranslateXAbs", 0.7)):
    pol_l = [("Sharpness", 1.0, 0.9), (second[0], 1.0, second[1])]
    H, W = 48, 64
    n = 3
    pol = CompiledPolicy([pol_l])
    batch = synth_batch(n, (H, W), seed=3)
    seed_all(1)
    want_u8 = np.stack([np.asarray(pil_path.PolicyTransform([pol_l])(PIL.Image.fromarray(a))) for a in batch])
    seed_all(1)
    ss, bb = [], []
    for i in range(n):
        s, b = pol.sample_parity(1, H, W); ss.append(s); bb.append(b)
    samples, boxes = np.concatenate(ss), np.concatenate(bb)
    x = torch.from_numpy(batch).cuda()
    tail = TailSpec(None, 0, False, IMAGENET_MEAN, IMAGENET_STD, 0, torch.float32)
    got = augment_batch(pol, x, tail, samples, boxes).cpu()
    # back to bytes through the exact table
    got_u8 = np.zeros_like(want_u8)
    for c in range(3):
        idx = torch.bucketize(got[:, c].contiguous(), tab[c].contiguous())
        got_u8[..., c] = idx.clamp(0, 255).numpy()
    d = (got_u8 != want_u8)
    print(pol_l, "bad bytes", int(d.sum()))
    ys, xs, cs = np.nonzero(d[0])
    for y, xx, c in list(zip(ys, xs, cs))[:8]:
        print("   img0 y %d x %d ch %d got %d want %d" % (y, xx, c, got_u8[0, y, xx, c], want_u8[0, y, xx, c]))
