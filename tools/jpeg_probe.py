"""Times the device JPEG decoder (``decode_jpeg``: entropy + reconstruct launches) against Pillow on the same files.

    python tools/jpeg_probe.py [--batch 256] [--iters 20] [--files DIR]

Synthetic 375x500 4:2:0 files (photo-like content, seeded) at q75 and q90; CUDA events around the decode call after
warm-up, and Pillow's ``Image.open(f).convert('RGB')`` of the same files on 1 core and with 8 worker processes.
``--files DIR`` also counts how many of the .jpg / .jpeg / .JPEG files under DIR the decoder refuses, and why.
Prints the card's name and power limit with the numbers, one JSON line per setting."""
import argparse
import io
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import PIL.Image  # noqa: E402
import torch  # noqa: E402

from fast_autoaugment_b200 import _lib  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, decode_jpeg  # noqa: E402


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 120 + 70 * np.sin(xx / w * 5 + seed)[..., None] * np.array([1.0, 0.7, 0.4]) + 40 * np.cos(yy / h * 3)[..., None]
    for _ in range(4):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(1, min(h, w) // 3 + 2)
        base[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.integers(0, 256, 3)
    base += 25 * np.sin(xx * 0.9 + yy * 0.4)[..., None] * (xx > w / 2)[..., None] + rng.normal(0, 6, (h, w, 3))
    return np.clip(base, 0, 255).astype(np.uint8)


def pil_decode(b):
    return np.asarray(PIL.Image.open(io.BytesIO(b)).convert("RGB")).shape


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = "unknown"
    return name, q


def refused(directory):
    reasons = {}
    n = 0
    for dp, _, fs in os.walk(directory):
        for f in fs:
            if f.lower().endswith((".jpg", ".jpeg")):
                b = open(os.path.join(dp, f), "rb").read()
                n += 1
                hdr = np.zeros(1, _lib.JPEG_HEADER_DTYPE)
                if _lib.lib.faa_jpeg_parse(b, len(b), hdr.ctypes.data) != _lib.OK:
                    why = (_lib.lib.faa_last_error() or b"").decode()
                    reasons[why] = reasons.get(why, 0) + 1
    return n, reasons


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    name, power = card()
    imgs = [photo(375, 500, i) for i in range(a.batch)]
    for q in (75, 90):
        files = []
        for im in imgs:
            bio = io.BytesIO()
            PIL.Image.fromarray(im).save(bio, "JPEG", quality=q, subsampling=2)
            files.append(bio.getvalue())
        enc = EncodedImages.from_bytes(files)                     # (raises, naming them, if any file is refused)
        out, status = decode_jpeg(enc)
        for _ in range(3):
            decode_jpeg(enc, out)
        torch.cuda.synchronize()
        ok = sum(int(np.array_equal(out.image(i).cpu().numpy(), np.asarray(PIL.Image.open(io.BytesIO(f)).convert("RGB"))))
                 for i, f in enumerate(files[:16]))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            decode_jpeg(enc, out)
        e1.record()
        torch.cuda.synchronize()
        gpu_ms = e0.elapsed_time(e1) / a.iters
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                decode_jpeg(enc, out)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "faa_jpeg" in ev.key:
                kern[ev.key.split("(")[0].split("::")[-1]] = round(ev.device_time_total / 3 / 1000, 3)
        t = time.perf_counter()
        for f in files:
            pil_decode(f)
        one_core_ms = (time.perf_counter() - t) * 1000
        with mp.Pool(8) as pool:
            pool.map(pil_decode, files[:16])
            t = time.perf_counter()
            pool.map(pil_decode, files, chunksize=8)
            eight_ms = (time.perf_counter() - t) * 1000
        print(json.dumps({"card": name, "power_limit": power, "batch": a.batch, "size": "375x500", "subsampling": "4:2:0",
                          "quality": q, "mean_file_bytes": int(np.mean([len(f) for f in files])),
                          "gpu_decode_ms": round(gpu_ms, 3), "kernel_ms": kern,
                          "pillow_1core_ms": round(one_core_ms, 1), "pillow_8workers_ms": round(eight_ms, 1),
                          "status_nonzero": int((status != 0).sum()), "equal_pillow_of_16": ok,
                          "refused": 0}), flush=True)
    if a.files:
        n, reasons = refused(a.files)
        print(json.dumps({"files": n, "refused": sum(reasons.values()), "reasons": reasons}), flush=True)


if __name__ == "__main__":
    main()
