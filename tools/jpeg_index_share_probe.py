"""Times what sharing the learned JPEG scan index between ranks buys in epoch 2, and what the exchange costs.

    python tools/jpeg_index_share_probe.py DIR [--files 2048] [--batch 128] [--iters 10] [--backend gloo] [--out OUTDIR]

Writes a SYNTHETIC tree of ``--files`` train files under DIR (tools/folder_probe.py's size mixture, q90, 4:2:0) and runs
two ranks (``--backend gloo``: both on device 0; ``nccl``: one device each, needs two) of
``get_dataloaders('imagenet', ..., multinode=True)``'s train loader with ``faa_jpeg_index_learn`` (Philox, resnet50 ->
224, fp32 out) for epochs 1 and 2, with ``set_epoch``.  Measured on each rank:

* the exchange at the start of epoch 2 (``share_jpeg_index``): host wall time, the bytes this rank sent and the entries
  it merged;
* the share of the rank's epoch-2 files that carried points into the decode, with the exchange and with only what the
  rank learned itself;
* the device decode time of each of the rank's epoch-2 batches (``decode_jpeg`` between CUDA events, median of
  ``--iters`` calls after warm-up) with the points the exchange gave and with only the rank's own, the two alternating
  call by call.  The ranks take turns, so no other decode shares the device while one is timed.

Prints one JSON line per rank and a summary from rank 0, with the card's name and power limit (also in
OUTDIR/jpeg_index_share_probe.jsonl with --out); the tree is removed at the end."""
import argparse
import json
import os
import shutil
import socket
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _decode_ms(enc, iters):
    """median device ms per call of the decodes of ``enc`` (a dict of name -> EncodedImages), alternating"""
    from fast_autoaugment_b200.engine import decode_jpeg
    outs = {k: decode_jpeg(e)[0] for k, e in enc.items()}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = {k: [] for k in enc}
    for it in range(iters + 2):
        for k in (list(enc) if it % 2 == 0 else list(enc)[::-1]):
            ev[0].record()
            decode_jpeg(enc[k], outs[k])
            ev[1].record()
            torch.cuda.synchronize()
            if it >= 2:
                times[k].append(ev[0].elapsed_time(ev[1]))
    return {k: float(np.median(v)) for k, v in times.items()}


def _rank(rank, world, port, backend, root, batch, iters, gpu, out_path):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world)
    from fast_autoaugment_b200 import data, distributed
    from fast_autoaugment_b200.conf import Config
    from fast_autoaugment_b200.engine import EncodedImages

    conf = Config.get()
    conf.clear()
    conf.update({"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"},
                 "faa_jpeg_index_learn": True})
    torch.manual_seed(0)
    sampler, loader = data.get_dataloaders("imagenet", batch, root, split=0.0, multinode=True)[:2]
    idx = loader.dataset.index
    staged, ex = [], {}
    read, share, pack = data.read_jpeg_batch, data.share_jpeg_index, distributed._pack_delta

    def read_spy(paths, *a, **kw):
        hb = read(paths, *a, **kw)
        staged.append(hb)
        return hb

    def pack_spy(*delta):
        buf = pack(*delta)
        ex["sent_bytes"] = int(buf.size)
        return buf

    def share_spy(index, *a, **kw):
        torch.cuda.synchronize()
        t = time.perf_counter()
        ex["merged"] = share(index, *a, **kw)
        ex["exchange_s"] = time.perf_counter() - t
        return ex["merged"]
    data.read_jpeg_batch, data.share_jpeg_index, distributed._pack_delta = read_spy, share_spy, pack_spy

    for epoch in (0, 1):
        if epoch == 1:
            own = data.JpegIndex.empty(idx.folder)      # what this rank learned itself, before the exchange
            for rel, (n, q) in idx._added.items():
                own.add([os.path.join(idx.folder, rel)], [n], [0, len(q)], q)
            staged.clear()
        sampler.set_epoch(epoch)
        torch.cuda.synchronize()
        t = time.perf_counter()
        n = sum(x.shape[0] for x, _ in loader)
        torch.cuda.synchronize()
        epoch_s = time.perf_counter() - t
    data.read_jpeg_batch = read
    files = with_points = own_points = 0
    ms = {"exchange": [], "own": []}
    for r in range(world):                              # one rank at a time on the device
        dist.barrier()
        if r != rank:
            continue
        for hb in staged:
            if not len(hb.accepted):
                continue
            paths = [hb.paths[i] for i in hb.accepted]
            lengths = [len(f) for f in hb.files]
            enc = EncodedImages.from_bytes(hb.files)
            of, op = own.gather(paths, lengths)
            files += len(paths)
            with_points += int((np.diff(hb.first) > 0).sum())
            own_points += int((np.diff(of) > 0).sum())
            t = _decode_ms({"exchange": enc.with_index(hb.first, hb.points), "own": enc.with_index(of, op)}, iters)
            for k in ms:
                ms[k].append(t[k])
    dist.barrier()
    line = {"rank": rank, "world": world, "backend": backend, "batch": batch, "epoch2_images": n,
            "epoch2_wall_s": round(epoch_s, 3), "epoch2_files_decoded": files,
            "epoch2_files_with_points_exchange": with_points, "epoch2_files_with_points_own": own_points,
            "decode_ms_per_batch_exchange": round(float(np.mean(ms["exchange"])), 3),
            "decode_ms_per_batch_own": round(float(np.mean(ms["own"])), 3), "batches": len(ms["own"]),
            "exchange_s": round(ex["exchange_s"], 4), "sent_bytes": ex.get("sent_bytes", 0), "merged": ex["merged"],
            "index_files_after_epoch2": len(idx._added) + len(idx._merged), **gpu}
    lines = [None] * world
    dist.all_gather_object(lines, line)
    if rank == 0:
        for x in lines:
            print(json.dumps(x), flush=True)
        summary = {"summary": True, "world": world, "backend": backend, "iters": iters,
                   "decode_ms_per_batch_exchange": round(float(np.mean([x["decode_ms_per_batch_exchange"] for x in lines])), 3),
                   "decode_ms_per_batch_own": round(float(np.mean([x["decode_ms_per_batch_own"] for x in lines])), 3),
                   "exchange_s_max": max(x["exchange_s"] for x in lines), **gpu}
        summary["speedup"] = round(summary["decode_ms_per_batch_own"] / summary["decode_ms_per_batch_exchange"], 2)
        print(json.dumps(summary), flush=True)
        if out_path:
            with open(out_path, "w") as f:
                f.write("".join(json.dumps(x) + "\n" for x in lines + [summary]))
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dir")
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--backend", default="gloo", choices=("gloo", "nccl"))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the GPU path: no CUDA device"
    assert a.backend != "nccl" or torch.cuda.device_count() >= 2, "--backend nccl needs two devices"
    from folder_probe import write_tree
    from jpeg_probe import card
    name, power = card()
    gpu = {"gpu": name, "power_limit": power, "host_cores": len(os.sched_getaffinity(0))}
    root = os.path.join(a.dir, "tree")
    shutil.rmtree(root, ignore_errors=True)
    write_tree(root, a.files, 90)
    out_path = None
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        out_path = os.path.join(a.out, "jpeg_index_share_probe.jsonl")
    try:
        mp.spawn(_rank, args=(2, _free_port(), a.backend, root, a.batch, a.iters, gpu, out_path), nprocs=2, join=True)
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
