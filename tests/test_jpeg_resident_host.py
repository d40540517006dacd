"""The resident JPEG store's host logic without a GPU: ownership, the shard layout's 16-byte boundaries and memory need,
the vectorised batch plan against a per-file loop (refused and progressive files, with and without points), host
grouping, the conf refusals, the metadata exchange and the all-rank failures over gloo with 2 and 3 ranks, and
``faa_gather``'s refusals before any device work."""
import ctypes
import json
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from imagenet_tree import write_tree

from fast_autoaugment_b200 import _lib, data, distributed
from fast_autoaugment_b200.conf import Config as C_

SYNC = _lib.JPEG_SYNC_DTYPE


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("resident_host")
    write_tree(root, 31, n_classes=3, per_class=8, n_val=3)              # progressive, CMYK and PNG files included
    return str(root)


def train_paths(root):
    return [p for p, _ in data.imagenet_index(root, "train")]


class FakeIndex:
    """``JpegIndex.gather``'s form: a few made-up points for every other file"""

    def gather(self, paths, lengths):
        parts = [np.frombuffer(np.arange(16 * (k % 3), dtype=np.uint8).tobytes(), SYNC) if k % 2 == 0 else
                 np.zeros(0, SYNC) for k, _ in enumerate(paths)]
        first = np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int64)
        return first, np.concatenate(parts)


def plan_of(paths, progressive=False, index=None, chunk=5):
    hbs = [data.read_jpeg_batch(paths[k:k + chunk], map, None, progressive, progressive)
           for k in range(0, len(paths), chunk)]
    return data.ShardPlan(hbs, index)


def store_of(shards, n, paths):
    st = data.ResidentJpegStore.__new__(data.ResidentJpegStore)
    st.paths = np.array(paths, dtype=object)
    st._install(shards, list(range(len(shards))))
    return st


def test_ownership_rule():
    for n, L in ((10, 3), (7, 1), (5, 8)):
        parts = [data.resident_owned(n, l, L) for l in range(L)]
        assert sorted(np.concatenate(parts).tolist()) == list(range(n))
        for l, p in enumerate(parts):
            assert all(i % L == l for i in p.tolist())


def test_host_grouping():
    hosts = ["a", "b", "a", "c", "b", "a"]
    assert distributed.local_ranks(hosts, 0) == [0, 2, 5] == distributed.local_ranks(hosts, 5)
    assert distributed.local_ranks(hosts, 4) == [1, 4]
    assert distributed.local_ranks(hosts, 3) == [3]


@pytest.mark.parametrize("progressive", [False, True])
@pytest.mark.parametrize("with_index", [False, True])
def test_shard_items_sit_on_16_byte_boundaries_and_need_adds_up(tree, progressive, with_index):
    paths = train_paths(tree)
    plan = plan_of(paths, progressive, FakeIndex() if with_index else None)
    m = plan.meta
    acc, ref = m["refused"] == 0, m["refused"] != 0
    assert ref.sum() == (2 if progressive else 3)
    offs = [m["hdr"]["offset"][acc], m["points_at"][acc], m["pixels_at"][ref],
            np.array([plan.tables_off, plan.points_off, plan.pixels_off])]
    assert all((o % 16 == 0).all() for o in offs)
    up = lambda x: (x + 15) // 16 * 16                                    # noqa: E731
    if with_index:
        room = m["n_points"][acc]
    else:
        room = np.diff(data.jpeg_index_capacities(m["hdr"][acc]))
    want = int(up(m["hdr"]["len"][acc]).sum()) + _lib.JPEG_TABLE_DTYPE.itemsize * int(m["n_tables"].sum()) + \
        16 * int(room.sum()) + int(up(m["h"][ref].astype(np.int64) * m["w"][ref] * 3).sum())
    assert plan.need == want
    parts = plan.parts()
    ends = [o + len(a) for o, a in parts]
    assert all(ends[k] <= parts[k + 1][0] for k in range(len(parts) - 1)) and ends[-1] <= plan.need
    files = [open(p, "rb").read() for p, r in zip(paths, m["refused"]) if not r]
    for (o, a), f in zip(parts, files):
        assert a.tobytes() == f
    assert (m["n_scans"][acc] > 0).sum() == (1 if progressive else 0)


def loop_plan(store, sel, buf_ptr, image_ptrs):
    """the batch plan of ``ResidentBatch``, one file at a time"""
    jobs, headers, scans, first, tab, at_files, refused = [], [], [], [0], 0, 0, 0
    acc = [i for i in sel if not store.meta["refused"][i]]
    files_at = 400 * sum(int(store.meta["n_tables"][i]) for i in acc)
    pts_at = files_at + sum((int(store.meta["hdr"]["len"][i]) + 15) // 16 * 16 for i in acc)
    tjobs, fjobs, pjobs, xjobs = [], [], [], []
    at_pts = 0
    for i in sel:
        m, s = store.meta[i], store.src[i]
        if m["refused"]:
            xjobs.append((int(s["pixels"]), int(image_ptrs[refused]), int(m["h"]) * int(m["w"]) * 3))
            refused += 1
            continue
        h = m["hdr"].copy()
        h["offset"] = at_files
        h["pool"] = h["pool"] - m["table_at"] + tab
        headers.append(h)
        sc = store.scans[store.scan_first[i]:store.scan_first[i + 1]].copy()
        sc["pool"] = sc["pool"] - m["table_at"] + tab
        scans.append(sc)
        tjobs.append((int(s["tables"]), buf_ptr + 400 * tab, 400 * int(m["n_tables"])))
        fjobs.append((int(s["file"]), buf_ptr + files_at + at_files, int(m["hdr"]["len"])))
        pjobs.append((int(s["points"]), buf_ptr + pts_at + 16 * at_pts, 16 * int(m["n_points"])))
        tab += int(m["n_tables"])
        at_files += (int(m["hdr"]["len"]) + 15) // 16 * 16
        at_pts += int(m["n_points"])
        first.append(first[-1] + int(m["n_points"]))
    jobs = [j for j in tjobs + fjobs + pjobs + xjobs if j[2] > 0]
    return np.array(jobs, np.uint64).reshape(-1, 3), np.array(headers, _lib.JPEG_HEADER_DTYPE), \
        (np.concatenate(scans) if scans else np.zeros(0, _lib.JPEG_SCAN_DTYPE)), np.array(first, np.int64)


@pytest.mark.parametrize("progressive", [False, True])
@pytest.mark.parametrize("with_index", [False, True])
def test_vectorised_batch_plan_equals_a_per_file_loop(tree, progressive, with_index):
    paths = train_paths(tree)
    n, L = len(paths), 2
    shards = []
    for j in range(L):
        own = data.resident_owned(n, j, L)
        plan = plan_of([paths[i] for i in own], progressive, FakeIndex() if with_index else None, chunk=4)
        shards.append((plan.meta, plan.scans, (j + 1) << 40, plan.tables_off))
    st = store_of(shards, n, paths)
    rng = np.random.default_rng(1)
    for sel in (rng.permutation(n)[:11], np.arange(n), rng.permutation(n)[:1]):
        b = st.plan(sel)
        img = (np.arange(len(b.refused), dtype=np.uint64) * 4096 + (7 << 44)).astype(np.uint64)
        jobs = b.jobs(3 << 44, img)
        want_jobs, want_h, want_scans, want_first = loop_plan(st, sel.tolist(), 3 << 44, img)
        got = np.stack([jobs["src"], jobs["dst"], jobs["bytes"]], axis=1)
        assert np.array_equal(got, want_jobs)
        assert b.headers.tobytes() == want_h.tobytes()
        assert (b.first is None and want_first[-1] == 0) or np.array_equal(b.first, want_first)
        assert (b.scans is None and len(want_scans) == 0) or b.scans.tobytes() == want_scans.tobytes()
        assert int(b.total) >= b.points_at
        assert [tuple(s) for s in b.sizes] == [(int(st.meta["h"][i]), int(st.meta["w"][i])) for i in sel]


def test_memory_check_message():
    assert distributed.fit_error([10, 20], [10, 30]) is None
    msg = distributed.fit_error([10, 40], [100, 30])
    assert "rank 0 needs 10 bytes, 100 free" in msg and "rank 1 needs 40 bytes, 30 free (too little)" in msg


class conf_set:
    def __init__(self, **kw):
        self.kw = {"aug": "fa_reduced_imagenet", "faa_crop_resize": True, "model": {"type": "resnet50"}, **kw}

    def __enter__(self):
        self.saved = dict(C_.get())
        C_.get().clear()
        C_.get().update(self.kw)

    def __exit__(self, *a):
        C_.get().clear()
        C_.get().update(self.saved)


@pytest.mark.parametrize("key", ["faa_jpeg_index_learn", "faa_jpeg_index_find"])
def test_learn_and_find_are_refused_before_any_file_is_read(tree, key, monkeypatch):
    def refuse(*a, **kw):
        raise AssertionError("a file was read")
    monkeypatch.setattr(data, "_read_file", refuse)
    with conf_set(faa_jpeg_resident=True, **{key: True}):
        with pytest.raises(ValueError, match="faa_jpeg_resident"):
            data.get_dataloaders("imagenet", 4, tree, split=0.0)


def test_gather_refuses_before_device_work():
    lib = _lib.lib
    buf = (ctypes.c_ubyte * 64)()
    ok = np.zeros(2, _lib.COPY_DTYPE)
    ok["src"], ok["dst"], ok["bytes"] = ctypes.addressof(buf), ctypes.addressof(buf) + 32, 8
    p = ok.ctypes.data
    assert lib.faa_gather(None, p, 2, None) == _lib.ERR_VALUE
    assert lib.faa_gather(p, None, 2, None) == _lib.ERR_VALUE
    assert lib.faa_gather(p, p, 0, None) == _lib.ERR_VALUE
    assert lib.faa_gather(p, p, -1, None) == _lib.ERR_VALUE
    for field in ("src", "dst"):
        bad = ok.copy()
        bad[1][field] = 0
        assert lib.faa_gather(bad.ctypes.data, p, 2, None) == _lib.ERR_VALUE
        assert b"job 1" in lib.faa_last_error()


# ---- the exchange over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, root, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from fast_autoaugment_b200 import data as d, distributed as dd
    paths = [p for p, _ in d.imagenet_index(root, "train")]
    n = len(paths)
    res = {}
    peers = dd.host_ranks()
    res["peers"] = peers
    own = d.resident_owned(n, peers.index(rank), len(peers))
    plan = plan_of([paths[i] for i in own], True, FakeIndex(), chunk=3)
    mine = d.pack_shard_meta(plan.meta, plan.scans, bytes(range(rank, rank + 64)), rank, plan.tables_off)
    bufs, err = dd.gather_bytes(mine, None, chunk_bytes=1000)
    shards = []
    for r in peers:
        meta, scans, h, dev, tables_off = d.unpack_shard_meta(bufs[r])
        assert h == bytes(range(r, r + 64)) and dev == r
        shards.append((meta, scans, (r + 1) << 40, tables_off))
    dd.agree(err)
    st = store_of(shards, n, paths)
    whole = plan_of(paths, True, None, chunk=3)
    res["same_headers"] = bool(np.array_equal(st.meta["hdr"]["h"], whole.meta["hdr"]["h"]) and
                               np.array_equal(st.meta["refused"], whole.meta["refused"]))
    res["owner"] = st.owner.tolist()
    res["scans"] = int(len(st.scans)) == int(len(whole.scans))
    # one rank's shard does not fit: every rank raises naming each rank's need and free memory
    try:
        dd.check_fit(100, 50 if rank == world - 1 else 1000)
        res["fit"] = None
    except RuntimeError as e:
        res["fit"] = str(e)
    # one rank fails before it knows its need
    try:
        dd.check_fit(None if rank == 0 else 10, 1000, OSError("cannot read") if rank == 0 else None)
        res["local"] = None
    except RuntimeError as e:
        res["local"] = str(e)
    # one rank's metadata is malformed: every rank raises
    bad = mine[:-1] if rank == 1 else mine
    bufs, err = dd.gather_bytes(bad, None)
    try:
        for r in range(world):
            d.unpack_shard_meta(bufs[r])
    except ValueError as e:
        err = e
    try:
        dd.agree(err, what="resident JPEG store")
        res["malformed"] = None
    except RuntimeError as e:
        res["malformed"] = str(e)
    dist.barrier()
    with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
        json.dump(res, f)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_metadata_exchange_and_failures_over_gloo(tree, tmp_path, world):
    mp.spawn(_worker, args=(world, _free_port(), tree, str(tmp_path)), nprocs=world, join=True)
    n = len(train_paths(tree))
    for r in range(world):
        with open(os.path.join(tmp_path, "rank%d.json" % r)) as f:
            x = json.load(f)
        assert x["peers"] == list(range(world)) and x["same_headers"] and x["scans"], r
        assert x["owner"] == [i % world for i in range(n)], r
        assert x["fit"] is not None and "rank %d needs 100 bytes, 50 free (too little)" % (world - 1) in x["fit"]
        assert "rank 0 needs 100 bytes, 1000 free" in x["fit"], r
        assert x["local"] is not None and "rank 0: OSError: cannot read" in x["local"], r
        assert x["malformed"] is not None and "resident JPEG store failed" in x["malformed"], r
