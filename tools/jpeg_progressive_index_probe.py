"""Times the device decode of progressive JPEG files with a scan index (``EncodedImages.from_bytes(...,
progressive=True, progressive_index=True)``) against the same files decoded without one and recorded, and the
streamed ImageNet loader learning progressive files' points.

    python tools/jpeg_progressive_index_probe.py [--batch 256] [--iters 20] [--files 1024] [--epochs 2] [--out DIR]

Sets: b256 progressive 375x500 4:2:0 at q75 and q90, and b256 of DESIGN.md 4.9's size mixture at q90 (SYNTHETIC
photo-like content, seeded; tools/jpeg_progressive_probe.py's).  For each set, alternated call by call after warm-up
with CUDA events around each call: the plain decode (reserved-1 headers), the recording decode and the decode from the
recorded index (reserved-3 headers).  The pixels and status of the three are asserted equal byte for byte.  Then the
train loader of ``get_dataloaders('imagenet', ...)`` (ImageNetChain at 224, b128) over trees of --files files with 0 %,
25 % and 100 % progressive files, ``faa_jpeg_index_learn`` on: Pillow for the progressive files
(``faa_jpeg_progressive`` off), the device without the index key, and the device with ``faa_jpeg_progressive_index``;
seconds per epoch for epochs 1 .. --epochs of a fresh loader, median of 3 fresh loaders.  Prints the card's name and
power limit with the numbers, one JSON line per setting."""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from folder_probe import epoch_s, mixture, photo, power_limit  # noqa: E402
from jpeg_progressive_probe import alternated_ms, save, write_tree  # noqa: E402
from fast_autoaugment_b200 import data  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, compact_jpeg_index, decode_jpeg  # noqa: E402


def decode_sets(a):
    rng = np.random.default_rng(0)
    sets = [("375x500 q75", [(375, 500)] * a.batch, 75), ("375x500 q90", [(375, 500)] * a.batch, 90),
            ("size mixture q90", mixture(rng, a.batch), 90)]
    for name, sizes, q in sets:
        prog = [save(photo(h, w, i), quality=q, progressive=True) for i, (h, w) in enumerate(sizes)]
        plain = EncodedImages.from_bytes(prog, progressive=True)
        enc = EncodedImages.from_bytes(prog, progressive=True, progressive_index=True)
        out_p, st_p = decode_jpeg(plain)
        out_r, st_r, count, pts, cap = decode_jpeg(enc, record=True)
        first, points = compact_jpeg_index(cap, count.cpu().numpy(), pts.cpu().numpy())
        indexed = enc.with_index(first, points)
        out_i, st_i = decode_jpeg(indexed)
        torch.cuda.synchronize()
        assert torch.equal(out_p.storage, out_r.storage) and torch.equal(out_p.storage, out_i.storage), name
        assert torch.equal(st_p, st_r) and torch.equal(st_p, st_i), name
        ms = alternated_ms({"plain": lambda: decode_jpeg(plain, out_p),
                            "recording": lambda: decode_jpeg(enc, out_r, record=True),
                            "indexed": lambda: decode_jpeg(indexed, out_i)}, a.iters)
        _, st_i2 = decode_jpeg(indexed, out_i)
        torch.cuda.synchronize()
        assert torch.equal(out_p.storage, out_i.storage) and torch.equal(st_p, st_i2), name
        print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "set": name,
                          "batch": len(prog), "mean_file_bytes": int(np.mean([len(f) for f in prog])),
                          "points_per_file": round(float(np.diff(first).mean()), 1),
                          "files_with_points": int((np.diff(first) > 0).sum()), "device_ms": ms,
                          "outputs_equal": True, "status_nonzero": int((st_p != 0).sum().item())}), flush=True)


def loaders(a):
    modes = {"pillow": {"faa_jpeg_progressive": False},
             "device": {"faa_jpeg_progressive": True},
             "device_index": {"faa_jpeg_progressive": True, "faa_jpeg_progressive_index": True}}
    for share in (0.0, 0.25, 1.0):
        with tempfile.TemporaryDirectory(dir=a.out) as root:
            write_tree(root, a.files, share)
            res = {}
            for mode, keys in modes.items():
                conf = Config.get()
                saved = dict(conf)
                runs = []
                try:
                    for rep in range(3):
                        conf.clear()
                        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True,
                                     "model": {"type": "resnet50"}, "faa_jpeg_index_learn": True, **keys})
                        torch.manual_seed(rep)
                        _, train, _, _ = data.get_dataloaders("imagenet", 128, root, split=0.0)
                        runs.append([epoch_s(train)[0] for _ in range(a.epochs)])
                finally:
                    conf.clear()
                    conf.update(saved)
                runs = np.array(runs)
                res[mode] = {"s_per_epoch": [round(float(x), 3) for x in np.median(runs, 0)],
                             "spread_s": [round(float(x), 3) for x in runs.max(0) - runs.min(0)]}
            print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                              "loader": "train, ImageNetChain 224, b128, faa_jpeg_index_learn", "files": a.files,
                              "progressive_share": share, "epochs": res}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--skip-loaders", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the loader trees (default: the system temp dir)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    decode_sets(a)
    if not a.skip_loaders:
        loaders(a)


if __name__ == "__main__":
    main()
