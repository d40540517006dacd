#!/usr/bin/env python
"""Times the ImageNet train loader over a directory of JPEG files (files stay on disk, ``JpegFileDataset``) against the
same files held on the device (the in-memory ``bytes`` mapping, ``EncodedDeviceDataset``).

    python tools/folder_probe.py DIR [--files 3072] [--batch 256] [--rounds 3] [--keep]

Writes a SYNTHETIC tree in the reference's layout under DIR (``DIR/q75``, ``DIR/q90``: ``imagenet-pytorch/{train,val}``)
with DESIGN.md 4.7's size mixture (40 % 375x500, 25 % 500x375, 20 % 333x500, 15 % random in [64, 1024]^2), 4:2:0,
photo-like content, and times ``get_dataloaders('imagenet', ...)``'s train loader (Philox, resnet50 -> 224, fp32 out)
from the index stream to the yielded batch: one warm-up epoch, then ``--rounds`` rounds that alternate one epoch of the
streamed loader and one of the device-resident loader, each ending in a device synchronise.  Also: the stream alone
(read, stage, copy, decode; no chain) and CUDA-event device times of the decode and of ``ImageNetChain.train`` per batch.
The page cache is warm (the files were just written): reads from a cold disk or a network file system are not measured.
Prints the card's name, its power limit and the host's cores with the numbers; removes the tree unless ``--keep``."""
import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import PIL.Image  # noqa: E402
import torch  # noqa: E402

from fast_autoaugment_b200 import data  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, decode_jpeg  # noqa: E402


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 120 + 70 * np.sin(xx / w * 5 + seed)[..., None] * np.array([1.0, 0.7, 0.4]) + 40 * np.cos(yy / h * 3)[..., None]
    for _ in range(6):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(1, min(h, w) // 4 + 2)
        base[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.integers(0, 256, 3)
    base += 25 * np.sin(xx * 0.9 + yy * 0.4)[..., None] * (xx > w / 2)[..., None] + rng.normal(0, 6, (h, w, 3))
    return np.clip(base, 0, 255).astype(np.uint8)


def mixture(rng, n):
    """SYNTHETIC source sizes (DESIGN.md 4.7, tools/ragged_probe.py)"""
    out = []
    for u in rng.random(n):
        if u < 0.40:
            out.append((375, 500))
        elif u < 0.65:
            out.append((500, 375))
        elif u < 0.85:
            out.append((333, 500))
        else:
            out.append((int(rng.integers(64, 1025)), int(rng.integers(64, 1025))))
    return out


def write_tree(root, n, quality, seed=0, n_classes=16):
    """n train files (and n // 8 val files) cut from a few large photo-like bases at random offsets"""
    rng = np.random.default_rng(seed)
    bases = [photo(1024, 1024, s) for s in range(4)]
    total = 0
    for split, m in (("train", n), ("val", max(1, n // 8))):
        for i, (h, w) in enumerate(mixture(rng, m)):
            b = bases[i % len(bases)]
            y, x = int(rng.integers(0, 1025 - h)), int(rng.integers(0, 1025 - w))
            d = os.path.join(root, "imagenet-pytorch", split, "n%08d" % (i % n_classes))
            os.makedirs(d, exist_ok=True)
            bio = io.BytesIO()
            PIL.Image.fromarray(b[y:y + h, x:x + w]).save(bio, "JPEG", quality=quality, subsampling=2)
            with open(os.path.join(d, "%s_%06d.JPEG" % (split, i)), "wb") as f:
                f.write(bio.getvalue())
            total += len(bio.getvalue())
    return total


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout
        return out.strip().splitlines()[0]
    except Exception:
        return "unknown"


def epoch_s(loader):
    torch.cuda.synchronize()
    t = time.perf_counter()
    n = 0
    for x, _ in loader:
        n += x.shape[0]
    torch.cuda.synchronize()
    return time.perf_counter() - t, n


def device_ms(fn, iters=10):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--files", type=int, default=3072)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--keep", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    torch.cuda.set_device(0)
    host = {"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cores": os.cpu_count(),
            "usable_cores": len(os.sched_getaffinity(0))}
    print(json.dumps(host), flush=True)
    conf = Config.get()
    conf.clear()
    conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}})
    for q in (75, 90):
        root = os.path.join(a.dir, "q%d" % q)
        shutil.rmtree(root, ignore_errors=True)
        t = time.perf_counter()
        nbytes = write_tree(root, a.files, q)
        written_s = time.perf_counter() - t
        paths, targets, _, _ = data._load_arrays("imagenet", root)
        files = []
        for p in paths:
            with open(p, "rb") as f:
                files.append(f.read())
        torch.manual_seed(0)
        streamed = data.get_dataloaders("imagenet", a.batch, root, split=0.0)[1]
        torch.manual_seed(0)
        resident = data.get_dataloaders("imagenet", a.batch, {"train": (files, targets), "test": (files[:8], targets[:8])},
                                        split=0.0)[1]
        for ld in (streamed, resident):                        # warm-up epoch: policy tables, allocator, page cache
            epoch_s(ld)
        tot = {"streamed": [0.0, 0], "resident": [0.0, 0]}
        for _ in range(a.rounds):
            for name, ld in (("streamed", streamed), ("resident", resident)):
                s, n = epoch_s(ld)
                tot[name][0] += s
                tot[name][1] += n
        # the stream alone: read + parse + stage + copy + decode, no chain
        batches = [paths[k:k + a.batch] for k in range(0, len(paths) - a.batch + 1, a.batch)]
        st = data.FileBatchStream()
        for _ in st(batches[:2], "cuda"):
            pass
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in st(batches, "cuda"):
            pass
        torch.cuda.synchronize()
        stream_s = time.perf_counter() - t
        # device time per batch of the decode and of the train chain on one decoded batch
        enc = EncodedImages.from_bytes(files[:a.batch])
        out, _ = decode_jpeg(enc)
        chain = streamed.chain
        dec_ms = device_ms(lambda: decode_jpeg(enc, out))
        chain_ms = device_ms(lambda: chain.train(out, seed=1, first_index=0))
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(5):
            chain.train(out, seed=1, first_index=0)
        torch.cuda.synchronize()
        host_chain_ms = (time.perf_counter() - t) / 5 * 1e3
        print(json.dumps({**host, "quality": q, "subsampling": "4:2:0", "batch": a.batch, "train_files": len(paths),
                          "mean_file_bytes": int(np.mean([len(f) for f in files])), "tree_bytes": nbytes,
                          "tree_written_s": round(written_s, 1),
                          "distinct_sizes_first_batch": len(out.groups()),
                          "streamed_img_s": round(tot["streamed"][1] / tot["streamed"][0], 1),
                          "resident_img_s": round(tot["resident"][1] / tot["resident"][0], 1),
                          "timed_batches_each": tot["streamed"][1] // a.batch,
                          "stream_only_img_s": round(len(batches) * a.batch / stream_s, 1),
                          "decode_device_ms": round(dec_ms, 2), "chain_train_device_ms": round(chain_ms, 2),
                          "chain_train_wall_ms": round(host_chain_ms, 2)}), flush=True)
        del streamed, resident, enc, out
        if not a.keep:
            shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
