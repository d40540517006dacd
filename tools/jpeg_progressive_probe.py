"""Times the device decode of progressive JPEG files (``decode_jpeg`` of ``EncodedImages.from_bytes(...,
progressive=True)``: the progressive entropy kernel + the reconstruct kernel) against the baseline decode of the same
images saved baseline, and against Pillow on the same progressive files; then the streamed ImageNet loader on trees
with 0 %, 25 % and 100 % progressive files, with ``faa_jpeg_progressive`` on and off.

    python tools/jpeg_progressive_probe.py [--batch 256] [--iters 20] [--files 1024] [--out DIR]

Sets: b256 375x500 4:2:0 at q75 and q90, and b256 of DESIGN.md 4.7's size mixture at q90 (SYNTHETIC photo-like
content, seeded).  Device times are CUDA events around the call after warm-up, the progressive and baseline calls
alternated; kernel times come from a separate torch.profiler run.  The wave schedule's critical path is reported as
the bytes of the largest work item of each wave summed over waves, against all the scan bytes, and by timing the same
images saved progressive with a restart marker every block (every block its own work item).  Pillow is
``Image.open(f).convert('RGB')`` on 1 core and with 8 worker processes.  The loader runs are the train loader of
``get_dataloaders('imagenet', ...)`` (ImageNetChain at 224, b128) over a tree of --files files; seconds per epoch,
median of 3 epochs after one warm-up epoch.  Prints the card's name and power limit with the numbers, one JSON line
per setting."""
import argparse
import io
import json
import multiprocessing as mp
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import PIL.Image  # noqa: E402
import PIL.ImageFile  # noqa: E402
import torch  # noqa: E402

from folder_probe import epoch_s, mixture, photo, power_limit  # noqa: E402
from fast_autoaugment_b200 import data  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import EncodedImages, decode_jpeg, parse_jpeg_headers  # noqa: E402


def save(a, **opts):
    bio = io.BytesIO()
    PIL.ImageFile.MAXBLOCK = max(PIL.ImageFile.MAXBLOCK, a.size * 2 + 65536)
    PIL.Image.fromarray(a).save(bio, "JPEG", subsampling=2, **opts)
    return bio.getvalue()


def pil_decode(b):
    return np.asarray(PIL.Image.open(io.BytesIO(b)).convert("RGB")).shape


def alternated_ms(fns, iters):
    """{name: ms per call} of calls made in turn, CUDA events around each"""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(iters):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
    return {k: round(float(np.median(v)), 3) for k, v in times.items()}


def kernel_ms(fn, reps=3):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return {ev.key.split("(")[0].split("::")[-1]: round(ev.device_time_total / reps / 1000, 3)
            for ev in prof.key_averages() if "faa_jpeg" in ev.key}


def critical_path(files):
    """(bytes of the largest work item of each wave, summed over waves; all scan bytes), over the batch"""
    _, _, _, scans, first = parse_jpeg_headers(files, progressive=True)
    crit = total = 0
    for i in range(len(files)):
        sc = scans[first[i]:first[i + 1]]
        for w in np.unique(sc["wave"]):
            crit += int(sc["len"][sc["wave"] == w].max())
        total += int(sc["len"].sum())
    return crit, total


def decode_sets(a):
    rng = np.random.default_rng(0)
    sets = [("375x500 q75", [(375, 500)] * a.batch, 75), ("375x500 q90", [(375, 500)] * a.batch, 90),
            ("size mixture q90", mixture(rng, a.batch), 90)]
    for name, sizes, q in sets:
        imgs = [photo(h, w, i) for i, (h, w) in enumerate(sizes)]
        base = [save(im, quality=q) for im in imgs]
        prog = [save(im, quality=q, progressive=True) for im in imgs]
        prst = [save(im, quality=q, progressive=True, restart_marker_blocks=1) for im in imgs]
        e_base = EncodedImages.from_bytes(base)
        e_prog = EncodedImages.from_bytes(prog, progressive=True)
        e_prst = EncodedImages.from_bytes(prst, progressive=True)
        outs = {k: decode_jpeg(e)[0] for k, e in (("base", e_base), ("prog", e_prog), ("prst", e_prst))}
        _, st = decode_jpeg(e_prog, outs["prog"])
        torch.cuda.synchronize()
        equal = sum(int(np.array_equal(outs["prog"].image(i).cpu().numpy(), np.asarray(
            PIL.Image.open(io.BytesIO(prog[i])).convert("RGB")))) for i in range(0, len(prog), max(1, len(prog) // 16)))
        ms = alternated_ms({"baseline": lambda: decode_jpeg(e_base, outs["base"]),
                            "progressive": lambda: decode_jpeg(e_prog, outs["prog"]),
                            "progressive_rst1": lambda: decode_jpeg(e_prst, outs["prst"])}, a.iters)
        kern = kernel_ms(lambda: decode_jpeg(e_prog, outs["prog"]))
        t = time.perf_counter()
        for f in prog:
            pil_decode(f)
        one = (time.perf_counter() - t) * 1000
        with mp.Pool(8) as pool:
            pool.map(pil_decode, prog[:16])
            t = time.perf_counter()
            pool.map(pil_decode, prog, chunksize=8)
            eight = (time.perf_counter() - t) * 1000
        crit, total = critical_path(prog)
        print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "set": name,
                          "batch": len(prog), "mean_file_bytes": {"baseline": int(np.mean([len(f) for f in base])),
                                                                  "progressive": int(np.mean([len(f) for f in prog]))},
                          "device_ms": ms, "progressive_kernels_ms": kern,
                          "pillow_progressive_ms": {"1core": round(one, 1), "8workers": round(eight, 1)},
                          "wave_critical_path_bytes": crit, "scan_bytes": total,
                          "status_nonzero": int((st != 0).sum()), "equal_pillow": "%d sampled" % equal}), flush=True)


def write_tree(root, n, share, seed=0, n_classes=16):
    """n train files (and n // 8 val files) of the size mixture at q90, a `share` of them progressive"""
    rng = np.random.default_rng(seed)
    bases = [photo(1024, 1024, s) for s in range(4)]
    for split, m in (("train", n), ("val", max(1, n // 8))):
        for i, (h, w) in enumerate(mixture(rng, m)):
            b = bases[i % len(bases)]
            y, x = int(rng.integers(0, 1025 - h)), int(rng.integers(0, 1025 - w))
            d = os.path.join(root, "imagenet-pytorch", split, "n%08d" % (i % n_classes))
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, "%s_%06d.JPEG" % (split, i)), "wb") as f:
                f.write(save(b[y:y + h, x:x + w], quality=90, progressive=bool(rng.random() < share)))


def loaders(a):
    for share in (0.0, 0.25, 1.0):
        with tempfile.TemporaryDirectory(dir=a.out) as root:
            write_tree(root, a.files, share)
            res = {}
            for key in (False, True):
                conf = Config.get()
                saved = dict(conf)
                conf.clear()
                conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"},
                             "faa_jpeg_progressive": key})
                try:
                    torch.manual_seed(0)
                    _, train, _, _ = data.get_dataloaders("imagenet", 128, root, split=0.0)
                    epoch_s(train)
                    runs = [epoch_s(train) for _ in range(3)]
                finally:
                    conf.clear()
                    conf.update(saved)
                n = runs[0][1]
                res["on" if key else "off"] = {"s_per_epoch": round(float(np.median([r[0] for r in runs])), 3),
                                               "images_per_s": round(n / float(np.median([r[0] for r in runs])), 1)}
            print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                              "loader": "train, ImageNetChain 224, b128", "files": a.files, "progressive_share": share,
                              "faa_jpeg_progressive": res}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--out", default=None, help="directory for the loader trees (default: the system temp dir)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    decode_sets(a)
    loaders(a)


if __name__ == "__main__":
    main()
