"""Times the device JPEG decoder with and without a scan index, and the index build rate.

    python tools/jpeg_index_probe.py [--batch 256] [--iters 20] [--out DIR]

Sets: b256 synthetic 375x500 4:2:0 files (photo-like, no restart markers) at q75 and q90, and DESIGN.md 4.9's size
mixture (40 % 375x500, 25 % 500x375, 20 % 333x500, 15 % random in [64, 1024]^2) at q90.  For each set: the index
(``build_jpeg_index``), then ``decode_jpeg`` without and with it, alternated call by call in one run, CUDA events
around each call after warm-up; the two outputs are compared byte for byte.  Prints the card's name and power limit
with the numbers, one JSON line per set (also written to DIR/jpeg_index_probe.jsonl with --out)."""
import argparse
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import PIL.Image  # noqa: E402
import torch  # noqa: E402

from folder_probe import mixture, photo  # noqa: E402
from jpeg_probe import card  # noqa: E402

from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, decode_jpeg  # noqa: E402


def encode(a, q):
    bio = io.BytesIO()
    PIL.Image.fromarray(a).save(bio, "JPEG", quality=q, subsampling=2)
    return bio.getvalue()


def sets(batch):
    bases = [photo(1024, 1024, s) for s in range(4)]
    rng = np.random.default_rng(0)
    fixed = [photo(375, 500, i) for i in range(batch)]
    mixed = []
    for i, (h, w) in enumerate(mixture(rng, batch)):
        y, x = int(rng.integers(0, 1025 - h)), int(rng.integers(0, 1025 - w))
        mixed.append(bases[i % 4][y:y + h, x:x + w])
    return [("375x500-q75", [encode(a, 75) for a in fixed]), ("375x500-q90", [encode(a, 90) for a in fixed]),
            ("mixture-q90", [encode(a, 90) for a in mixed])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    name, power = card()
    lines = []
    for label, files in sets(a.batch):
        enc = EncodedImages.from_bytes(files)
        torch.cuda.synchronize()
        build_jpeg_index(enc)                                 # warm-up
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        build_ms = []
        for _ in range(5):
            ev[0].record()
            first, points = build_jpeg_index(enc)             # (waits for the device: the count comes back)
            ev[1].record()
            torch.cuda.synchronize()
            build_ms.append(ev[0].elapsed_time(ev[1]))
        idx = enc.with_index(first, points)
        idx.device_index()
        outs = {}
        times = {"plain": [], "indexed": []}
        for it in range(a.iters + 3):                         # 3 warm-up rounds, then alternate
            for which, e in (("plain", enc), ("indexed", idx)) if it % 2 == 0 else (("indexed", idx), ("plain", enc)):
                ev[0].record()
                out, st = decode_jpeg(e)
                ev[1].record()
                torch.cuda.synchronize()
                if it >= 3:
                    times[which].append(ev[0].elapsed_time(ev[1]))
                outs[which] = (out.storage.cpu(), st.cpu())
        same = torch.equal(outs["plain"][0], outs["indexed"][0]) and torch.equal(outs["plain"][1], outs["indexed"][1])
        counts = np.diff(first)
        line = {"set": label, "batch": a.batch, "mean_file_kb": round(float(np.mean([len(f) for f in files])) / 1024, 1),
                "indexed_files": int((counts > 0).sum()), "mean_points": round(float(counts.mean()), 1),
                "decode_ms_plain": round(float(np.median(times["plain"])), 3),
                "decode_ms_indexed": round(float(np.median(times["indexed"])), 3),
                "index_build_ms": round(float(np.median(build_ms)), 3),
                "index_build_files_per_s": round(a.batch / (float(np.median(build_ms)) / 1000), 1),
                "outputs_equal": bool(same), "status_zero": int((outs["plain"][1] == 0).sum()),
                "gpu": name, "power_limit": power, "iters": a.iters}
        line["speedup"] = round(line["decode_ms_plain"] / line["decode_ms_indexed"], 2)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_index_probe.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
