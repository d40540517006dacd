"""Write the scan indexes of an ImageNet directory: ``python -m fast_autoaugment_b200.jpeg_index DATAROOT OUTDIR``.

For each split of ``DATAROOT/imagenet-pytorch/{train,val}`` (the reference's sample list, ``data.imagenet_index``) it
reads the files as the loaders do, records each file's scan index on the device (``engine.build_jpeg_index``: one
serial decode per file) and writes ``OUTDIR/<split>.npz`` (``data.JpegIndex``).  Give ``OUTDIR`` to
``get_dataloaders('imagenet', ...)`` as ``conf['faa_jpeg_index']``: the files listed there are then decoded on many
threads each, with the same pixels.  The files themselves are not changed.  With ``--progressive`` it also indexes
progressive files (their points come from a recording decode on the device), for loaders run with
``conf['faa_jpeg_progressive']`` and ``conf['faa_jpeg_progressive_index']``; without it they are listed with no points."""
from __future__ import annotations

import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import _lib, data
from .engine import EncodedImages, build_jpeg_index, parse_jpeg_headers

CHUNK_BYTES = 256 << 20           # file bytes on the device at a time


def index_files(paths, folder, device="cuda", workers=4, log=None, progressive=False):
    """The ``data.JpegIndex`` of ``paths`` (files under ``folder``).  Files the device decoder refuses are listed with
    no points; so are progressive files, unless ``progressive`` (``build_jpeg_index`` of files parsed with
    ``progressive_index=True``)."""
    paths = [os.fspath(p) for p in paths]
    sizes, firsts, points = [], [np.zeros(1, np.int64)], []
    t0, done = time.perf_counter(), 0
    with ThreadPoolExecutor(max(1, workers)) as ex:
        k = 0
        while k < len(paths):
            chunk, nbytes = [], 0
            while k < len(paths) and (not chunk or nbytes < CHUNK_BYTES):
                chunk.append(paths[k])
                nbytes += os.path.getsize(paths[k])
                k += 1
            files = list(ex.map(data._read_file, chunk))
            headers, pool, refused = parse_jpeg_headers(files, ex.map, progressive, progressive)[:3]
            bad = {i for i, _ in refused}
            ok = [i for i in range(len(files)) if i not in bad]
            counts = np.zeros(len(files), np.int64)
            if ok:
                enc = EncodedImages.from_bytes([files[i] for i in ok], device, progressive, progressive)
                first, pts = build_jpeg_index(enc)
                counts[ok] = np.diff(first)
                points.append(pts)
            sizes += [len(f) for f in files]
            firsts.append(firsts[-1][-1] + np.cumsum(counts))
            done += len(files)
            if log:
                log("%d / %d files, %.0f files/s" % (done, len(paths), done / max(time.perf_counter() - t0, 1e-9)))
    rel = [os.path.relpath(p, folder) for p in paths]
    pts = np.concatenate(points) if points else np.zeros(0, _lib.JPEG_SYNC_DTYPE)
    return data.JpegIndex(folder, rel, np.array(sizes, np.int64), np.concatenate(firsts), pts)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m fast_autoaugment_b200.jpeg_index", description=__doc__.split("\n\n")[0])
    ap.add_argument("dataroot", help="the reference's dataroot (holds imagenet-pytorch/{train,val})")
    ap.add_argument("outdir", help="directory for train.npz and val.npz (conf['faa_jpeg_index'])")
    ap.add_argument("--splits", default="train,val")
    ap.add_argument("--workers", type=int, default=4, help="reader threads")
    ap.add_argument("--progressive", action="store_true",
                    help="index progressive files too (conf['faa_jpeg_progressive_index'])")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("the scan index is recorded on the device: no CUDA device")
    os.makedirs(a.outdir, exist_ok=True)
    for split in a.splits.split(","):
        samples = data.imagenet_index(a.dataroot, split)
        folder = data.imagenet_split_folder(a.dataroot, split)
        idx = index_files([p for p, _ in samples], folder, workers=a.workers,
                          log=lambda m, s=split: print("[jpeg_index] %s: %s" % (s, m), file=sys.stderr, flush=True),
                          progressive=a.progressive)
        out = os.path.join(a.outdir, "%s.npz" % split)
        idx.save(out)
        print("[jpeg_index] %s: %d files, %d indexed, %d points -> %s" % (
            split, len(samples), int((np.diff(idx.first) > 0).sum()), len(idx.points), out), flush=True)


if __name__ == "__main__":
    main()
