#!/usr/bin/env python
"""Times the policy search's scoring of T candidate policies over an ImageNet directory: one loader's
``tta(K, policies=T candidates)`` (each batch read, staged and decoded once, one launch group per chain stage over
T * K * B images) against T calls of ``tta(K)``, one per candidate (what T hyperopt trials do, one after another).

    python tools/tta_policies_probe.py DIR [--files 4096] [--batch 128] [--replicas 5] [--candidates 1 4 8]
                                           [--rounds 3] [--keep]

Writes a SYNTHETIC tree in the reference's layout under DIR (tools/folder_probe.py's writer: DESIGN.md 4.7's size
mixture, 4:2:0, q90) and runs ``get_dataloaders('imagenet', batch, DIR, split=0.15)``'s valid loader (resnet50 -> 224,
fp16 out, Philox) with and without ``faa_jpeg_index``.  Candidate t is sub-policies [5t, 5t + 5) of the ImageNet archive
policy (num_policy 5, num_op 2, as search.py's policy_decoder gives them).  The T-call arm runs ``tta(K, policies=[p_t])``
for each candidate, which is ``tta(K)`` of a loader with policy p_t (same launches), so both arms share one loader and
its files.  Per arm: validation images x candidates scored per second, from the index stream to the yielded batches,
one warm-up then ``--rounds`` rounds alternating the arms, each ending in a device synchronise; the median and the
spread (min, max) over rounds.  Per stage: CUDA-event device times, on one decoded b``batch`` batch, of the policy,
crop-resize, jitter and final launches of ``train_tta_policies``, of the whole call, and of T ``train_tta`` calls.
Before timing, one epoch checks that both arms give the same bytes (candidate t's block against the single call placed
at its keys).  The page cache is warm (the files were just written).  Nothing here runs a model: the numbers are the
loader side of a trial only.  Prints the card's name and power limit with the numbers; removes the tree unless
``--keep``."""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from folder_probe import power_limit, write_tree  # noqa: E402

from fast_autoaugment_b200 import _lib, archive, data, engine, jpeg_index  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, TailSpec, decode_jpeg  # noqa: E402


def loader(root, batch, index_dir):
    conf = Config.get()
    conf.clear()
    conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"},
                 "faa_out_dtype": "float16"})
    if index_dir:
        conf["faa_jpeg_index"] = index_dir
    return data.get_dataloaders("imagenet", batch, root, split=0.15)[2]


def candidates(T):
    pol = archive.fa_resnet50_rimagenet()
    return engine.compile_policies([pol[5 * t:5 * t + 5] for t in range(T)])


def epoch_multi(ld, k, pols):
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for x, _ in ld.tta(k, policies=pols):
        n += x.shape[2] * x.shape[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def epoch_single(ld, k, pols):
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for p in pols:
        for x, _ in ld.tta(k, policies=[p]):
            n += x.shape[2]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def check_equal(root, batch, k, pols, index_dir):
    """one epoch of the multi-candidate arm; candidate t's block of batch j against a single-candidate call of a second
    loader over the same index stream at drawn_j + t * K * B_j"""
    one, ref = loader(root, batch, index_dir), loader(root, batch, index_dir)
    ref.seed = one.seed
    single = [ref.tta(k, policies=[p]) for p in pols]
    drawn = 0
    for x, y in one.tta(k, policies=pols):
        b = x.shape[2]
        for t, it in enumerate(single):
            ref._drawn = drawn + t * k * b
            xt, yt = next(it)
            if not (torch.equal(xt[0], x[t]) and torch.equal(yt, y)):
                return False
        drawn += len(pols) * k * b
    return True


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


def stage_ms(chain, x, k, pols):
    """device time of each of train_tta_policies' stages on a decoded ragged batch x (the calls it makes)"""
    B, s, raw, n = len(x), chain.input_size, TailSpec.raw_u8(), len(pols) * k
    y = engine.augment_tta_policies(pols, x, raw, k, 1, 0)
    z = engine.crop_resize(y, s, rng=chain.crop.cfg(1, 0))
    recs, rgb = chain._device_records_tta(B, x.device, 1, 0, n)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def jitter():
        _lib.check(_lib.lib.faa_color_jitter(z.data_ptr(), z.data_ptr(), n * B, s, s, recs.data_ptr(), stream))
    return {"policy_ms": device_ms(lambda: engine.augment_tta_policies(pols, x, raw, k, 1, 0, out=y)),
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
    ap.add_argument("--candidates", type=int, nargs="+", default=[1, 4, 8])
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
    ld = loader(root, a.batch, None)
    paths = [ld.dataset.paths[i] for i in list(iter(ld.sampler))[:a.batch]]
    enc = EncodedImages.from_bytes([data._read_file(p) for p in paths])
    x, _ = decode_jpeg(enc)
    chain = ld.chain
    for T in a.candidates:
        pols = candidates(T)
        stages = {"decode_ms": device_ms(lambda: decode_jpeg(enc, x)), **stage_ms(chain, x, K, pols),
                  "train_tta_policies_ms": device_ms(lambda: chain.train_tta_policies(x, pols, K, seed=1)),
                  "t_train_tta_ms": device_ms(lambda: [chain.train_tta_policies(x, [p], K, seed=1,
                                                                                first_index=t * K * a.batch)
                                                       for t, p in enumerate(pols)])}
        print(json.dumps({**host, "candidates": T, "batch": a.batch, "replicas": K, "distinct_sizes": len(x.groups()),
                          **{k: round(v, 3) for k, v in stages.items()}}), flush=True)
    for index_dir in (None, idx_dir):
        for T in a.candidates:
            pols = candidates(T)
            equal = check_equal(root, a.batch, K, pols, index_dir)
            one = loader(root, a.batch, index_dir)
            epoch_multi(one, K, pols)                     # warm-up: policy tables, allocator, page cache
            epoch_single(one, K, pols)
            rates = {"single": [], "multi": []}
            for _ in range(a.rounds):
                for name, fn in (("single", epoch_single), ("multi", epoch_multi)):
                    s, n = fn(one, K, pols)
                    rates[name].append(n / s)
            print(json.dumps({**host, "quality": 90, "subsampling": "4:2:0", "batch": a.batch, "replicas": K,
                              "candidates": T, "jpeg_index": index_dir is not None, "valid_images": len(one.sampler),
                              "outputs_equal": equal,
                              **{"%s_img_cand_s" % k: round(statistics.median(v), 1) for k, v in rates.items()},
                              **{"%s_spread" % k: [round(min(v), 1), round(max(v), 1)] for k, v in rates.items()}}),
                  flush=True)
            del one
    if not a.keep:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
