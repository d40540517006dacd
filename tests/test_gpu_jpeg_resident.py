"""``conf['faa_jpeg_resident']``: the ImageNet directory held in device memory (``ResidentJpegDataset``) against the
streamed loaders over the same tree, bit for bit, over two epochs (train, valid, test and ``tta``), with progressive
files refused, decoded on the device and taking a scan index; no file read after construction; the store's points
against ``build_jpeg_index`` and the index file; one gather launch per batch; corrupt files; ``faa_gather`` alone;
two processes sharing one device under gloo (NCCL on two devices when present)."""
import json
import os
import re
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from helpers import ROOT, seed_all
from imagenet_tree import write_tree
from test_gpu_imagenet_folder import B, assert_same, conf_set, corrupt_tree, index, run

from fast_autoaugment_b200 import _lib, data, engine

pytestmark = pytest.mark.gpu

MODES = {"refused": {}, "progressive": {"faa_jpeg_progressive": True},
         "progressive_index": {"faa_jpeg_progressive": True, "faa_jpeg_progressive_index": True}}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("imagenet_resident")
    write_tree(root, 21, n_classes=3, per_class=10, n_val=4)             # progressive, CMYK and PNG files included
    from test_gpu_jpeg_record import _bigger_files
    _bigger_files(str(root), 5)                                          # files that take points
    return str(root)


def launches():
    return int(_lib.lib.faa_launch_count())


def tta_run(loader, seed, replicas=2, policies=None):
    seed_all(seed)
    return [(x.cpu(), y.cpu()) for x, y in loader.tta(replicas, policies)]


def no_reads(m):
    def refuse(*a, **kw):
        raise AssertionError("a file was read after construction")
    m.setattr(data, "_read_file", refuse)
    m.setattr(data, "read_jpeg_batch", refuse)


@pytest.mark.parametrize("mode", list(MODES))
def test_resident_loaders_equal_streamed_loaders(tree, mode):
    with conf_set(**MODES[mode]):
        seed_all(3)
        want = data.get_dataloaders("imagenet", B, tree, split=0.2)
    with conf_set(faa_jpeg_resident=True, **MODES[mode]):
        seed_all(3)
        got = data.get_dataloaders("imagenet", B, tree, split=0.2)
    assert isinstance(got[1].dataset, data.ResidentJpegDataset) and isinstance(got[3].dataset, data.ResidentJpegDataset)
    assert got[1].dataset.store is got[2].dataset.store and got[3].dataset.store is not got[1].dataset.store
    assert got[1].dataset.device_bytes > 0 and got[1].dataset.targets == want[1].dataset.targets

    def no_reads_run(fn):
        """``fn()`` with the reader patched to raise: the resident loaders read no file after construction"""
        with pytest.MonkeyPatch.context() as m:
            no_reads(m)
            return fn()
    pols = [data.policy_by_conf_name("fa_reduced_imagenet")] * 2
    try:
        for epoch in range(2):
            for which in (1, 2, 3):
                seed = 10 * epoch + which
                want_b = run(want[which], seed)
                assert_same(no_reads_run(lambda: run(got[which], seed)), want_b, (mode, which, epoch))
        assert_same(no_reads_run(lambda: tta_run(got[2], 40)), tta_run(want[2], 40), (mode, "tta"))
        assert_same(no_reads_run(lambda: tta_run(got[2], 41, policies=pols)), tta_run(want[2], 41, policies=pols),
                    (mode, "tta policies"))
    finally:
        got[1].dataset.close()
        got[3].dataset.close()


def _shard_points(store, i):
    """file i's points read back from its owner's shard (one process: this rank's)"""
    m = store.meta[i]
    n = int(m["n_points"])
    at = int(m["points_at"])
    return store.shard[at:at + 16 * n].cpu().numpy().view(_lib.JPEG_SYNC_DTYPE)


@pytest.mark.parametrize("mode", ["refused", "progressive_index"])
def test_store_points_equal_build_jpeg_index_and_the_index_file(tree, mode, tmp_path):
    kw = MODES[mode]
    paths, _, _, _ = index(tree)
    prog = bool(kw)
    store = data.ResidentJpegStore(paths, "cuda", progressive=prog, progressive_index=prog)
    try:
        acc = np.flatnonzero(store.meta["refused"] == 0)
        files = [open(paths[i], "rb").read() for i in acc]
        first, points = engine.build_jpeg_index(engine.EncodedImages.from_bytes(files, "cuda", prog, prog))
        assert int(first[-1]) > 0
        for k, i in enumerate(acc):
            assert _shard_points(store, i).tobytes() == points[first[k]:first[k + 1]].tobytes(), paths[i]
        assert store.n_tables >= len(acc)
    finally:
        store.close()
    from fast_autoaugment_b200 import jpeg_index
    out = str(tmp_path / "index")
    jpeg_index.main([tree, out] + (["--progressive"] if prog else []))
    idx = data.JpegIndex.load(os.path.join(out, "train.npz"), data.imagenet_split_folder(tree, "train"))
    store = data.ResidentJpegStore(paths, "cuda", index=idx, progressive=prog, progressive_index=prog)
    try:
        for i in np.flatnonzero(store.meta["refused"] == 0):
            want = idx.lookup(paths[i], os.path.getsize(paths[i]))
            assert _shard_points(store, i).tobytes() == want.tobytes(), paths[i]
    finally:
        store.close()


def test_each_batch_adds_one_gather_launch(tree, monkeypatch):
    paths, _, _, _ = index(tree)
    store = data.ResidentJpegStore(paths, "cuda", progressive=True)
    inside = []
    dec = data.decode_jpeg

    def spy(*a, **kw):
        n0 = launches()
        r = dec(*a, **kw)
        inside.append(launches() - n0)
        return r
    monkeypatch.setattr(data, "decode_jpeg", spy)
    try:
        sel = [np.arange(k, min(len(paths), k + B)) for k in range(0, len(paths), B)]
        gen = store.batches(sel)
        for k in range(len(sel)):
            inside.clear()
            n0 = launches()
            next(gen)
            assert len(inside) <= 1 and launches() - n0 == sum(inside) + 1, k
        torch.cuda.synchronize()
    finally:
        store.close()


@pytest.mark.parametrize("pos", [5, 23])
def test_corrupt_file_raises_naming_it(tmp_path, pos):
    bad, n = corrupt_tree(tmp_path, pos)
    with conf_set(faa_jpeg_resident=True):
        _, train, _, test = data.get_dataloaders("imagenet", 4, str(tmp_path), split=0.0)
    seen = []
    try:
        with pytest.raises(OSError, match=re.escape(bad) + r": 0x[0-9a-f]+ \([^)]*scan truncated"):
            for x, _ in test:
                seen.append(x)
        assert len(seen) <= pos // 4 + 1
    finally:
        train.dataset.close()
        test.dataset.close()


def test_gather_copies_exactly_each_job():
    rng = np.random.default_rng(7)
    lens = [400] * 1500 + list(rng.integers(1, 5000, 1500)) + [3 << 20, (5 << 20) + 13, 1, 15, 16, 17, 16385]
    lens = np.array(lens, np.int64)
    n = len(lens)
    src_off = (np.cumsum(lens + 64) - (lens + 64) + 0) // 16 * 16 + 16          # 16-byte aligned sources
    src = torch.from_numpy(rng.integers(0, 256, int(src_off[-1] + lens[-1] + 64), dtype=np.uint8)).cuda()
    shift = rng.integers(0, 16, n)                                               # unaligned destinations
    shift[:1500:3] = 0
    dst_off = np.cumsum(lens + 48) - (lens + 48) + 16 + shift
    dst = torch.full((int(dst_off[-1] + lens[-1] + 64),), 0xA5, dtype=torch.uint8, device="cuda")
    jobs = np.zeros(n, _lib.COPY_DTYPE)
    jobs["src"] = src.data_ptr() + src_off.astype(np.uint64)
    jobs["dst"] = dst.data_ptr() + dst_off.astype(np.uint64)
    jobs["bytes"] = lens
    perm = rng.permutation(n)
    jobs = jobs[perm]
    d_jobs = torch.from_numpy(jobs.view(np.uint8).copy()).cuda()
    n0 = launches()
    engine.gather(jobs, d_jobs, "cuda")
    torch.cuda.synchronize()
    assert launches() - n0 == 1
    want = np.full(dst.numel(), 0xA5, np.uint8)
    s = src.cpu().numpy()
    for o, d, k in zip(src_off, dst_off, lens):
        want[d:d + k] = s[o:o + k]
    got = dst.cpu().numpy()
    assert np.array_equal(got, want)                             # every job exact, every guard byte untouched


# ---- two processes
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, backend, root, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist
    from test_gpu_imagenet_folder import B, assert_same, conf_set, run

    from fast_autoaugment_b200 import data

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world)
    with conf_set():
        torch.manual_seed(0)
        plain = data.get_dataloaders("imagenet", B, root, split=0.2, multinode=True)
    with conf_set(faa_jpeg_resident=True):
        torch.manual_seed(0)
        res = data.get_dataloaders("imagenet", B, root, split=0.2, multinode=True)
    store = res[1].dataset.store
    paths = [p for p, _ in data.imagenet_index(root, "train")]
    assert store.n_local == world and store.local_rank == rank
    own = data.resident_owned(len(paths), rank, world)
    held = np.flatnonzero(store.owner == rank)
    assert np.array_equal(held, own)
    for i in own[store.meta["refused"][own] == 0][:8]:              # the shard holds its owner's bytes
        m = store.meta[i]
        at, n = int(m["hdr"]["offset"]), int(m["hdr"]["len"])
        assert store.shard[at:at + n].cpu().numpy().tobytes() == open(paths[i], "rb").read(), paths[i]
    for epoch in range(2):
        for s in (plain[0], res[0]):
            s.set_epoch(epoch)
        for which in (1, 2, 3):
            assert_same(run(res[which], 70 + 10 * epoch + which), run(plain[which], 70 + 10 * epoch + which),
                        (rank, which, epoch))
    res[1].dataset.close()
    res[3].dataset.close()
    with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
        json.dump({"device_bytes": int(res[1].dataset.device_bytes), "owned": len(own)}, f)
    dist.barrier()
    dist.destroy_process_group()


def _two_ranks(tmp_path, backend):
    root = str(tmp_path / "data")
    write_tree(root, 47, n_classes=3, per_class=12, n_val=4)
    mp.spawn(_worker, args=(2, _free_port(), backend, root, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        with open(os.path.join(tmp_path, "rank%d.json" % r)) as f:
            assert json.load(f)["device_bytes"] > 0


def test_two_processes_share_one_device_gloo(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL needs two devices")
def test_two_processes_nccl(tmp_path):
    _two_ranks(tmp_path, "nccl")
