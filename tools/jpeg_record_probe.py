"""Times the recording JPEG decode against the plain one, and the ImageNet folder loader learning its scan index.

    python tools/jpeg_record_probe.py DIR [--batch 256] [--iters 20] [--files 2048] [--rounds 3] [--out OUTDIR]

Decode: on tools/jpeg_index_probe.py's b256 375x500 4:2:0 q90 set and DESIGN.md 4.9's size mixture at q90,
``decode_jpeg(enc)`` and ``decode_jpeg(enc, record=True)`` alternate call by call after warm-up, with CUDA events around
each call; the medians and the recording overhead are printed, the outputs compared byte for byte, and the recorded
points compared with ``build_jpeg_index``'s.

Loader: a SYNTHETIC tree of ``--files`` train files (tools/folder_probe.py's mixture, q90) under DIR, then wall time of
full epochs of ``get_dataloaders('imagenet', ...)``'s train loader (Philox, resnet50 -> 224, fp32 out), each ending in a
device synchronise: epochs 1 and 2 of a fresh loader without an index, with ``faa_jpeg_index_learn`` and with a
prebuilt ``faa_jpeg_index``, ``--rounds`` times, and the medians.  A warm-up epoch comes first, so the page cache is
warm.  Prints
the card's name and power limit with the numbers (one JSON line per measurement, also in OUTDIR/jpeg_record_probe.jsonl
with --out); the tree is removed at the end."""
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

from folder_probe import epoch_s, write_tree  # noqa: E402
from jpeg_index_probe import sets  # noqa: E402
from jpeg_probe import card  # noqa: E402

from fast_autoaugment_b200 import data, jpeg_index  # noqa: E402
from fast_autoaugment_b200.conf import Config  # noqa: E402
from fast_autoaugment_b200.engine import (EncodedImages, build_jpeg_index, compact_jpeg_index,  # noqa: E402
                                          decode_jpeg)


def decode_lines(batch, iters, gpu):
    out = []
    for label, files in sets(batch):
        if label == "375x500-q75":
            continue
        enc = EncodedImages.from_bytes(files)
        first, points = build_jpeg_index(enc)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times, res = {"plain": [], "record": []}, {}
        for it in range(iters + 3):                           # 3 warm-up rounds, then alternate
            for which in ("plain", "record") if it % 2 == 0 else ("record", "plain"):
                ev[0].record()
                r = decode_jpeg(enc, record=which == "record")
                ev[1].record()
                torch.cuda.synchronize()
                if it >= 3:
                    times[which].append(ev[0].elapsed_time(ev[1]))
                res[which] = r
        (pa, sa), (pb, sb, cnt, pts, cap_first) = res["plain"], res["record"]
        rf, rp = compact_jpeg_index(cap_first, cnt.cpu().numpy(), pts.cpu().numpy())
        line = {"set": label, "batch": batch, "decode_ms_plain": round(float(np.median(times["plain"])), 3),
                "decode_ms_record": round(float(np.median(times["record"])), 3),
                "outputs_equal": bool(torch.equal(pa.storage, pb.storage) and torch.equal(sa, sb)),
                "points_equal_index_build": bool(np.array_equal(rf, first) and rp.tobytes() == points.tobytes()),
                "recorded_files": int((np.diff(rf) > 0).sum()), "iters": iters, **gpu}
        line["record_overhead_pct"] = round(100 * (line["decode_ms_record"] / line["decode_ms_plain"] - 1), 2)
        out.append(line)
        print(json.dumps(line), flush=True)
    return out


def loader_lines(root, files, batch, rounds, gpu):
    shutil.rmtree(root, ignore_errors=True)
    write_tree(root, files, 90)
    idx_dir = os.path.join(root, "index")
    t = time.perf_counter()
    jpeg_index.main([root, idx_dir])
    index_s = time.perf_counter() - t
    conf = Config.get()
    out = []

    def loader(**kw):
        conf.clear()
        conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}, **kw})
        torch.manual_seed(0)
        return data.get_dataloaders("imagenet", batch, root, split=0.0)[1]

    epoch_s(loader())                                         # warm-up: page cache, allocator
    times = {}
    for r in range(rounds):                                   # fresh loaders each round: epoch 1 is a first epoch
        for name, kw in (("plain", {}), ("learn", {"faa_jpeg_index_learn": True}), ("prebuilt", {"faa_jpeg_index": idx_dir})):
            ld = loader(**kw)
            for epoch in (1, 2):
                s, n = epoch_s(ld)
                times.setdefault((name, epoch), []).append(s)
                line = {"loader": name, "round": r, "epoch": epoch, "files": n, "batch": batch, "epoch_s": round(s, 3),
                        "images_per_s": round(n / s, 1), **gpu}
                if name == "learn":
                    line["learned_files"] = len(ld.dataset.index._added)
                out.append(line)
                print(json.dumps(line), flush=True)
    med = {k: float(np.median(v)) for k, v in times.items()}
    line = {"index_command_s": round(index_s, 3), "train_files": files, "rounds": rounds,
            **{"median_s_%s_epoch%d" % k: round(v, 3) for k, v in med.items()},
            "learn_epoch1_over_plain_epoch1": round(med[("learn", 1)] / med[("plain", 1)], 3),
            "learn_epoch2_over_prebuilt_epoch2": round(med[("learn", 2)] / med[("prebuilt", 2)], 3), **gpu}
    out.append(line)
    print(json.dumps(line), flush=True)
    shutil.rmtree(root, ignore_errors=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    torch.cuda.set_device(0)
    name, power = card()
    gpu = {"gpu": name, "power_limit": power, "host_cores": len(os.sched_getaffinity(0))}
    lines = decode_lines(a.batch, a.iters, gpu) + loader_lines(os.path.join(a.dir, "tree"), a.files, a.batch, a.rounds, gpu)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_record_probe.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
