"""Times the JPEG decode that finds its scan index on the device against the plain and the indexed decode, and the
found index against the serial index build.

    python tools/jpeg_find_probe.py [--batch 256] [--iters 20] [--out DIR]

Sets: tools/jpeg_index_probe.py's b256 SYNTHETIC photo-like 375x500 4:2:0 files at q75 and q90 and DESIGN.md 4.9's
size mixture at q90.  For each set, alternated call by call after warm-up with CUDA events around each call:
``decode_jpeg(enc)`` (serial per file), ``decode_jpeg(enc, find=True)`` and ``decode_jpeg`` of the files carrying
``build_jpeg_index``'s index; then ``build_jpeg_index(enc)`` against ``build_jpeg_index(enc, find=True)`` (each
including its copy of the counts back).  Medians are printed with the card's name and power limit read in the same
run, with whether the three decodes' pixels and status are equal byte for byte, how many files' found index converged
(equals the built one) and how many found points equal the built ones.  One JSON line per set (also written to
DIR/jpeg_find_probe.jsonl with --out)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from jpeg_index_probe import sets  # noqa: E402
from jpeg_probe import card  # noqa: E402

from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, decode_jpeg  # noqa: E402


def timed(fns, iters, warmup=3):
    """{name: [ms]} of the callables in ``fns``, alternated call by call (order reversed every other round), and the
    last result of each"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times, res = {k: [] for k in fns}, {}
    names = list(fns)
    for it in range(iters + warmup):
        for k in names if it % 2 == 0 else names[::-1]:
            ev[0].record()
            r = fns[k]()
            ev[1].record()
            torch.cuda.synchronize()
            if it >= warmup:
                times[k].append(ev[0].elapsed_time(ev[1]))
            res[k] = r
    return {k: float(np.median(v)) for k, v in times.items()}, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    torch.cuda.set_device(0)
    name, power = card()
    lines = []
    for label, files in sets(a.batch):
        enc = EncodedImages.from_bytes(files)
        first, points = build_jpeg_index(enc)
        indexed = enc.with_index(first, points)
        dec, r = timed({"plain": lambda: decode_jpeg(enc), "found": lambda: decode_jpeg(enc, find=True),
                        "indexed": lambda: decode_jpeg(indexed)}, a.iters)
        (pa, sa), (pf, sf), (pi, si) = r["plain"], r["found"], r["indexed"]
        idx, ri = timed({"build": lambda: build_jpeg_index(enc), "find": lambda: build_jpeg_index(enc, find=True)},
                        a.iters)
        ff, fp = ri["find"]
        per_file = np.diff(first)
        found_n = np.diff(ff)
        conv = same_pts = 0
        for i in range(len(files)):
            got, want = fp[ff[i]:ff[i + 1]], points[first[i]:first[i + 1]]
            assert got.tobytes() == want[:len(got)].tobytes(), (label, i)        # a prefix, always
            conv += got.tobytes() == want.tobytes()
            same_pts += len(got)
        line = {"set": label, "batch": a.batch, "mean_file_kb": round(float(np.mean([len(f) for f in files])) / 1024, 1),
                "points_per_file": round(float(per_file.mean()), 1),
                "decode_ms_plain": round(dec["plain"], 3), "decode_ms_found": round(dec["found"], 3),
                "decode_ms_indexed": round(dec["indexed"], 3),
                "index_ms_build": round(idx["build"], 3), "index_ms_find": round(idx["find"], 3),
                "outputs_equal": bool(torch.equal(pa.storage, pf.storage) and torch.equal(pa.storage, pi.storage) and
                                      torch.equal(sa, sf) and torch.equal(sa, si)),
                "files_converged": int(conv), "files": len(files),
                "found_points_equal_built": int(same_pts), "built_points": int(per_file.sum()),
                "found_points": int(found_n.sum()), "iters": a.iters, "gpu": name, "power_limit": power}
        lines.append(line)
        print(json.dumps(line), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_find_probe.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
