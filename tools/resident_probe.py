#!/usr/bin/env python
"""Times the ImageNet train loader with the split held in device memory (``conf['faa_jpeg_resident']``,
``ResidentJpegDataset``) against the streamed loader (files on disk, ``JpegFileDataset``, learning its scan index in
the warm-up epoch so the timed epochs decode every file on many threads) and the in-memory ``bytes`` mapping
(``EncodedDeviceDataset``).

    python tools/resident_probe.py DIR [--files 3072] [--batch 256] [--rounds 3] [--keep]

Writes tools/folder_probe.py's SYNTHETIC tree (DESIGN.md 4.7's size mixture, 4:2:0) at q75 and q90 under DIR, then per
quality: one warm-up epoch of each loader, then ``--rounds`` rounds alternating one epoch of each, each ending in a
device synchronise (Philox, resnet50 -> 224, fp32 out).  Also: the resident store's start-up (read + parse + Pillow,
upload, index build), its table count and device bytes per file, and the gather's device time and bytes/s per batch
(CUDA events over repeated ``faa_gather`` launches of one batch's job table).  The page cache is warm.  One process on
one device: shards over several GPUs and NVLink gather rates are not measured.  Prints the card's name and its power
limit with the numbers; removes the tree unless ``--keep``."""
import argparse
import json
import os
import shutil
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from folder_probe import epoch_s, power_limit, write_tree  # noqa: E402

from fast_autoaugment_b200 import _lib, data, engine  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402


def loaders(root, files, targets, batch):
    base = {"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}}
    out = {}
    for name, extra, src in (("streamed_learned", {"faa_jpeg_index_learn": True}, root),
                             ("resident", {"faa_jpeg_resident": True}, root),
                             ("bytes_mapping", {}, {"train": (files, targets), "test": (files[:8], targets[:8])})):
        conf = Config.get()
        conf.clear()
        conf.update({**base, **extra})
        torch.manual_seed(0)
        t = time.perf_counter()
        _, train, _, test = data.get_dataloaders("imagenet", batch, src, split=0.0)
        torch.cuda.synchronize()
        out[name] = (train, test, time.perf_counter() - t)
    return out


def gather_ms(store, batch, iters=20):
    sel = np.arange(min(batch, len(store.paths)))
    p = store.plan(sel)
    out = data.RaggedImages.empty(p.sizes, store.device)
    buf = torch.empty(p.total, dtype=torch.uint8, device=store.device)
    jobs = p.jobs(buf.data_ptr(), out.storage.data_ptr() + out.offsets[p.refused].astype(np.uint64))
    d_jobs = torch.from_numpy(jobs.view(np.uint8).copy()).to(store.device)
    engine.gather(jobs, d_jobs, store.device)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        engine.gather(jobs, d_jobs, store.device)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    nbytes = int(jobs["bytes"].sum())
    return ms, nbytes, len(jobs)


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
    host = {"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cores": os.cpu_count()}
    print(json.dumps(host), flush=True)
    for q in (75, 90):
        root = os.path.join(a.dir, "q%d" % q)
        shutil.rmtree(root, ignore_errors=True)
        write_tree(root, a.files, q)
        paths, targets, _, _ = data._load_arrays("imagenet", root)
        files = [open(p, "rb").read() for p in paths]
        lds = loaders(root, files, targets, a.batch)
        for train, _, _ in lds.values():                       # warm-up epoch (the streamed loader learns its index)
            epoch_s(train)
        tot = {k: [0.0, 0] for k in lds}
        for _ in range(a.rounds):
            for name, (train, _, _) in lds.items():
                s, n = epoch_s(train)
                tot[name][0] += s
                tot[name][1] += n
        ds = lds["resident"][0].dataset
        store = ds.store
        ms, nbytes, n_jobs = gather_ms(store, a.batch)
        print(json.dumps({**host, "quality": q, "batch": a.batch, "train_files": len(paths),
                          "mean_file_bytes": int(np.mean([len(f) for f in files])),
                          **{"%s_img_s" % k: round(v[1] / v[0], 1) for k, v in tot.items()},
                          "timed_batches_each": tot["resident"][1] // a.batch,
                          "resident_build_s": round(lds["resident"][2], 2),
                          "resident_startup_s": {k: round(v, 2) for k, v in store.timing.items()},
                          "resident_device_bytes": int(ds.device_bytes),
                          "resident_device_bytes_per_file": round(ds.device_bytes / len(paths), 1),
                          "tables": int(store.n_tables), "tables_per_file": round(store.n_tables / len(paths), 2),
                          "table_bytes_per_file": round(store.n_tables * _lib.JPEG_TABLE_DTYPE.itemsize / len(paths), 1),
                          "points_per_file": round(float(store.meta["n_points"].mean()), 2),
                          "gather_jobs_per_batch": n_jobs, "gather_bytes_per_batch": nbytes,
                          "gather_device_ms": round(ms, 3), "gather_GB_s": round(nbytes / ms / 1e6, 1)}), flush=True)
        for train, test, _ in lds.values():
            if isinstance(train.dataset, data.ResidentJpegDataset):
                train.dataset.close()
                test.dataset.close()
        del lds, ds, store
        if not a.keep:
            shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
