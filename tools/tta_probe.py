#!/usr/bin/env python
"""Times the policy search's test-time augmentation over an ImageNet directory: K separate validation loaders (the
reference search.py:87-125 pattern, ``get_dataloaders`` called K times) against one loader's ``tta(K)``.

    python tools/tta_probe.py DIR [--files 4096] [--batch 128] [--replicas 5] [--rounds 3] [--keep]

Writes a SYNTHETIC tree in the reference's layout under DIR (tools/folder_probe.py's writer: DESIGN.md 4.7's size
mixture, 4:2:0, q90) and runs ``get_dataloaders('imagenet', batch, DIR, split=0.15)``'s valid loader (resnet50 -> 224,
fp16 out, Philox) with and without ``faa_jpeg_index``.  The K-loader arm gives its loaders distinct seeds (built in one
process they would otherwise share one seed and yield identical replicas).  Per arm: validation images evaluated with
all K replicas per second, from the index stream to the yielded batches, one warm-up epoch then ``--rounds`` rounds
alternating the arms, each epoch ending in a device synchronise.  Per stage: CUDA-event device times of one b``batch``
batch's decode, of ``train_tta``'s policy, crop-resize, jitter and final launches, of the whole ``train_tta`` and of K
``train`` calls.  Before timing, one epoch checks that the two arms' outputs are equal bit for bit (the K loaders then
use one seed, their Philox keys placed where ``tta`` places replica r's).  The page cache is warm (the files were just
written).  Prints the card's name and power limit with the numbers; removes the tree unless ``--keep``."""
import argparse
import ctypes
import json
import os
import shutil
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from folder_probe import power_limit, write_tree  # noqa: E402

from fast_autoaugment_b200 import _lib, data, engine, jpeg_index  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, TailSpec, decode_jpeg  # noqa: E402


def loaders(root, batch, k, index_dir):
    conf = Config.get()
    conf.clear()
    conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"},
                 "faa_out_dtype": "float16"})
    if index_dir:
        conf["faa_jpeg_index"] = index_dir
    return [data.get_dataloaders("imagenet", batch, root, split=0.15)[2] for _ in range(k)]


def epoch_k_loaders(lds):
    """one epoch of K loaders in lock step, as search.py's loop consumes them"""
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for batches in zip(*lds):
        n += batches[0][0].shape[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def epoch_tta(ld, k):
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for x, _ in ld.tta(k):
        n += x.shape[1]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def arms_equal(root, batch, k, index_dir):
    """one epoch of each arm with the K loaders' keys at tta's layout: replica r of batch j at drawn_j + r * B_j"""
    one = loaders(root, batch, 1, index_dir)[0]
    sep = loaders(root, batch, k, index_dir)
    for ld in sep:
        ld.seed = one.seed
    its = [iter(ld) for ld in sep]
    drawn, n_batches = 0, 0
    for x, y in one.tta(k):
        b = x.shape[1]
        for r, (ld, it) in enumerate(zip(sep, its)):
            ld._drawn = drawn + r * b
            xr, yr = next(it)
            if not (torch.equal(xr, x[r]) and torch.equal(yr, y)):
                return False
        drawn += k * b
        n_batches += 1
    return n_batches == len(one)


def device_ms(fn, iters=5):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def stage_ms(chain, x, k):
    """device time of each of train_tta's stages on a decoded ragged batch x (the calls train_tta makes)"""
    B, s, raw = len(x), chain.input_size, TailSpec.raw_u8()
    pol = chain.aug.compiled
    y = engine.augment_tta(pol, x, raw, k, 1, 0)
    z = engine.crop_resize(y, s, rng=chain.crop.cfg(1, 0))
    recs, rgb = chain._device_records_tta(B, x.device, 1, 0, k)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def jitter():
        _lib.check(_lib.lib.faa_color_jitter(z.data_ptr(), z.data_ptr(), k * B, s, s, recs.data_ptr(), stream))
    return {"policy_ms": device_ms(lambda: engine.augment_tta(pol, x, raw, k, 1, 0, out=y)),
            "crop_resize_ms": device_ms(lambda: engine.crop_resize(y, s, rng=chain.crop.cfg(1, 0))),
            "jitter_ms": device_ms(jitter),
            "final_ms": device_ms(lambda: engine.augment_batch(chain.flip_policy, z, chain.tail,
                                                               rng=engine.make_rng(1, 0, chain.tail), lighting_rgb=rgb))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--files", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--replicas", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--keep", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    torch.cuda.set_device(0)
    host = {"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cores": os.cpu_count(),
            "usable_cores": len(os.sched_getaffinity(0))}
    print(json.dumps(host), flush=True)
    K = a.replicas
    root = os.path.join(a.dir, "q90")
    shutil.rmtree(root, ignore_errors=True)
    write_tree(root, a.files, 90)
    idx_dir = os.path.join(root, "index")
    jpeg_index.main([root, idx_dir])
    # device time per stage, on the first valid batch
    ld = loaders(root, a.batch, 1, None)[0]
    paths = [ld.dataset.paths[i] for i in list(iter(ld.sampler))[:a.batch]]
    enc = EncodedImages.from_bytes([data._read_file(p) for p in paths])
    x, _ = decode_jpeg(enc)
    chain = ld.chain
    stages = {"decode_ms": device_ms(lambda: decode_jpeg(enc, x)), **stage_ms(chain, x, K),
              "train_tta_ms": device_ms(lambda: chain.train_tta(x, K, seed=1)),
              "k_train_ms": device_ms(lambda: [chain.train(x, seed=1, first_index=r * a.batch) for r in range(K)])}
    print(json.dumps({**host, "batch": a.batch, "replicas": K, "distinct_sizes": len(x.groups()),
                      **{k: round(v, 3) for k, v in stages.items()}}), flush=True)
    for index_dir in (None, idx_dir):
        equal = arms_equal(root, a.batch, K, index_dir)
        sep = loaders(root, a.batch, K, index_dir)
        for r, l in enumerate(sep):
            l.seed += r                                   # distinct seeds: distinct replicas
        one = loaders(root, a.batch, 1, index_dir)[0]
        epoch_k_loaders(sep)                              # warm-up: policy tables, allocator, page cache
        epoch_tta(one, K)
        tot = {"k_loaders": [0.0, 0], "tta": [0.0, 0]}
        for _ in range(a.rounds):
            for name, fn in (("k_loaders", lambda: epoch_k_loaders(sep)), ("tta", lambda: epoch_tta(one, K))):
                s, n = fn()
                tot[name][0] += s
                tot[name][1] += n
        print(json.dumps({**host, "quality": 90, "subsampling": "4:2:0", "batch": a.batch, "replicas": K,
                          "jpeg_index": index_dir is not None, "valid_images": len(one.sampler),
                          "outputs_equal": equal,
                          "k_loaders_img_s": round(tot["k_loaders"][1] / tot["k_loaders"][0], 1),
                          "tta_img_s": round(tot["tta"][1] / tot["tta"][0], 1)}), flush=True)
        del sep, one
    if not a.keep:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
