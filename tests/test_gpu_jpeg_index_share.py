"""``conf['faa_jpeg_index_learn']`` on more than one process: ``get_dataloaders('imagenet', ..., multinode=True)`` over
an ImageNet tree, two ranks, two epochs with ``set_epoch``.  Every batch equals the same run without the key; the
exchange at the start of epoch 2 leaves each rank's index listing exactly the accepted files either rank read that the
placement rule gives points, with the index command's points; in epoch 2 no file either rank learned is recorded again;
only the train loader's epochs exchange.  gloo with both ranks on one device, and NCCL on two devices."""
import json
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

from helpers import ROOT

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, backend, root, ref_dir, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch.distributed as dist
    from test_gpu_imagenet_folder import B, assert_same, conf_set, run

    from fast_autoaugment_b200 import data

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, rank=rank, world_size=world)
    train = data.imagenet_split_folder(root, "train")
    ref = data.JpegIndex.load(os.path.join(ref_dir, "train.npz"), train)
    all_train = [p for p, _ in data.imagenet_index(root, "train")]
    size = {p: os.path.getsize(p) for p in all_train}

    with conf_set():
        torch.manual_seed(0)
        plain = data.get_dataloaders("imagenet", B, root, split=0.2, multinode=True)
    with conf_set(faa_jpeg_index_learn=True):
        torch.manual_seed(0)
        learn = data.get_dataloaders("imagenet", B, root, split=0.2, multinode=True)
    idx = learn[1].dataset.index
    assert isinstance(learn[0], torch.utils.data.distributed.DistributedSampler) and learn[2].dataset.index is idx

    staged, decoded, shares = [], [], []
    read, dec, share = data.read_jpeg_batch, data.decode_jpeg, data.share_jpeg_index

    def read_spy(paths, *a, **kw):
        hb = read(paths, *a, **kw)
        if (a[1] if len(a) > 1 else kw.get("index")) is idx and len(hb.accepted):
            staged.append([hb.paths[i] for i in hb.accepted])
        return hb

    def decode_spy(enc, out=None, record=False, **kw):
        r = dec(enc, out, record=record, **kw)
        if record:
            decoded.append(r[2].cpu().numpy())
        return r

    def share_spy(index, *a, **kw):
        n = share(index, *a, **kw)
        listed = {p: index.lookup(p, size[p]).tobytes() for p in all_train}
        shares.append({p: q for p, q in listed.items() if q})
        return n
    data.read_jpeg_batch, data.decode_jpeg, data.share_jpeg_index = read_spy, decode_spy, share_spy

    # epoch 1: the train loader exchanges (nothing yet), the valid loader (the same SubsetSampler on every rank) and
    # the test loader do not
    for s in (plain[0], learn[0]):
        s.set_epoch(0)
    assert_same(run(learn[1], 51), run(plain[1], 51), "train, epoch 1")
    assert_same(run(learn[2], 52), run(plain[2], 52), "valid, epoch 1")
    assert_same(run(learn[3], 53), run(plain[3], 53), "test")
    assert len(shares) == 1 and not shares[0]
    seen = {p for b in staged for p in b}
    mine = {os.path.join(train, r) for r in idx._added}
    assert mine == {p for p in seen if len(ref.lookup(p, size[p]))} and len(mine) >= 8
    both = [None] * world
    dist.all_gather_object(both, (sorted(seen), sorted(mine)))
    read_any = {p for s, _ in both for p in s}
    others = {p for r, (_, m) in enumerate(both) if r != rank for p in m}
    assert others - mine                                            # the other rank learned files this one did not

    # epoch 2: at its start every rank lists what either rank learned, with the index command's points
    for s in (plain[0], learn[0]):
        s.set_epoch(1)
    staged.clear()
    decoded.clear()
    got = run(learn[1], 61)
    assert len(shares) == 2
    want = {p: ref.lookup(p, size[p]).tobytes() for p in read_any if len(ref.lookup(p, size[p]))}
    assert shares[1] == want and set(want) == mine | others
    assert_same(got, run(plain[1], 61), "train, epoch 2")
    assert len(decoded) == len(staged) and staged
    hit = set()
    for paths, counts in zip(staged, decoded):
        for p, c in zip(paths, counts):
            if p in want:
                hit.add(p)
                assert c == 0, p                                    # carried its points: not recorded again
    assert hit & (others - mine)                                    # files only the other rank had read
    with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
        json.dump({"shared_files": len(want), "hit_from_other": len(hit & (others - mine))}, f)
    dist.barrier()
    dist.destroy_process_group()


def _two_ranks(tmp_path, backend):
    from imagenet_tree import write_tree
    from test_gpu_jpeg_record import _bigger_files

    from fast_autoaugment_b200 import jpeg_index
    root = str(tmp_path / "data")
    write_tree(root, 43, n_classes=3, per_class=20, n_val=4)             # refused files included
    _bigger_files(root, 7)
    ref_dir = str(tmp_path / "index")
    jpeg_index.main([root, ref_dir])
    mp.spawn(_worker, args=(2, _free_port(), backend, root, ref_dir, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        with open(os.path.join(tmp_path, "rank%d.json" % r)) as f:
            assert json.load(f)["hit_from_other"] > 0


def test_learning_loaders_share_the_index_gloo_one_device(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL needs two devices")
def test_learning_loaders_share_the_index_nccl(tmp_path):
    _two_ranks(tmp_path, "nccl")
