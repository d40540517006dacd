"""Sharing learned JPEG scan indexes between ranks without a GPU: ``JpegIndex.delta`` / ``merge`` (round trips through
``save`` / ``load``, replace semantics, lengths, non-ASCII paths, empty and malformed deltas), the packed form the
exchange sends, and ``distributed.share_jpeg_index`` over gloo at world sizes 2 and 3 (``mp.spawn``, as
tests/test_dist_gloo.py): disjoint and overlapping deltas give every rank the same union, a second exchange sends only
sizes, a small chunk size takes several rounds, and one rank's malformed delta or local failure raises on every rank."""
import json
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from fast_autoaugment_b200 import _lib, data, distributed

SYNC = _lib.JPEG_SYNC_DTYPE
FOLDER = os.path.join(os.sep, "data", "imagenet-pytorch", "train")


def pts(seed, n):
    """n fake points (the index never reads them; the decoder checks them)"""
    return np.frombuffer(np.random.default_rng(seed).integers(0, 256, n * 16, dtype=np.uint8).tobytes(), SYNC).copy()


def learn(idx, names, seed=0, length=1000):
    """``add`` the files ``FOLDER/<name>``, one call per file as the loaders' checks make them"""
    for k, name in enumerate(names):
        q = pts(seed + k, 1 + (seed + k) % 7)
        idx.add([os.path.join(FOLDER, name)], [length + k], [0, len(q)], q)


def entries(idx, names, length=1000):
    return {n: idx.lookup(os.path.join(FOLDER, n), length + k).tobytes() for k, n in enumerate(names)}


def test_delta_merge_round_trips_through_save_and_load(tmp_path):
    base = data.JpegIndex(FOLDER, [b"n1/listed.JPEG"], [500], [0, 3], pts(99, 3))
    names = ["n1/a.JPEG", "n1/b.JPEG", "n2/c.JPEG"]
    src = data.JpegIndex.empty(FOLDER)
    learn(src, names)
    paths, lengths, first, points = src.delta()
    assert paths.dtype.kind == "S" and sorted(paths.tolist()) == sorted(os.fsencode(n) for n in names)
    assert lengths.dtype == np.int64 and first.dtype == np.int64 and points.dtype == SYNC and first[-1] == len(points)
    base.merge(paths, lengths, first, points)
    assert entries(base, names) == entries(src, names) and all(entries(base, names).values())
    assert base.lookup(os.path.join(FOLDER, "n1/listed.JPEG"), 500).tobytes() == pts(99, 3).tobytes()
    assert base.gather([os.path.join(FOLDER, n) for n in names], [1000, 1001, 1002])[1].tobytes() == \
        src.gather([os.path.join(FOLDER, n) for n in names], [1000, 1001, 1002])[1].tobytes()
    out = str(tmp_path / "train.npz")
    base.save(out)
    with np.load(out) as z:
        assert int(z["version"]) == data.JPEG_INDEX_VERSION == 1 and len(z["paths"]) == 4
    back = data.JpegIndex.load(out, FOLDER)
    assert entries(back, names) == entries(base, names)
    assert back.lookup(os.path.join(FOLDER, "n1/listed.JPEG"), 500).tobytes() == pts(99, 3).tobytes()
    assert back.delta()[0].size == 0                            # what was loaded is not sent


def test_delta_holds_what_add_entered_since_the_last_delta_and_never_merged_entries():
    idx = data.JpegIndex.empty(FOLDER)
    learn(idx, ["a.JPEG", "b.JPEG"])
    assert sorted(idx.delta()[0].tolist()) == [b"a.JPEG", b"b.JPEG"]
    assert idx.delta()[0].size == 0 and idx.delta()[2].tolist() == [0]
    other = data.JpegIndex.empty(FOLDER)
    learn(other, ["c.JPEG", "a.JPEG"], seed=5)
    idx.merge(*other.delta())
    learn(idx, ["d.JPEG"], seed=7)
    assert idx.delta()[0].tolist() == [b"d.JPEG"]              # merged entries are never sent on
    learn(idx, ["e.JPEG"], seed=8)
    idx.merge(*other_delta_of(["e.JPEG"], seed=9))              # a merge replaces an unsent learned entry
    assert idx.delta()[0].size == 0
    assert "e.JPEG" not in idx._added and idx.lookup(os.path.join(FOLDER, "e.JPEG"), 1000).tobytes() == \
        pts(9, 1 + 9 % 7).tobytes()


def other_delta_of(names, seed):
    o = data.JpegIndex.empty(FOLDER)
    learn(o, names, seed=seed)
    return o.delta()


def test_merge_replaces_entries_and_a_length_mismatch_gets_no_points():
    p = os.path.join(FOLDER, "n1/x.JPEG")
    idx = data.JpegIndex(FOLDER, [b"n1/x.JPEG"], [700], [0, 2], pts(1, 2))
    idx.merge([b"n1/x.JPEG"], [1000], [0, 4], pts(2, 4))        # replaces the listed entry
    assert idx.lookup(p, 1000).tobytes() == pts(2, 4).tobytes() and idx.lookup(p, 700).size == 0
    idx.add([p], [1100], [0, 3], pts(3, 3))                     # learned here: replaces the merged entry
    assert idx.lookup(p, 1100).tobytes() == pts(3, 3).tobytes() and idx.lookup(p, 1000).size == 0
    idx.merge(["n1/x.JPEG"], [1200], [0, 1], pts(4, 1))         # str paths too
    assert idx.lookup(p, 1200).tobytes() == pts(4, 1).tobytes() and idx.lookup(p, 1100).size == 0
    assert idx.delta()[0].size == 0
    first, points = idx.gather([p, p], [1200, 1100])
    assert first.tolist() == [0, 1, 1] and points.tobytes() == pts(4, 1).tobytes()


def test_non_ascii_paths_and_empty_deltas(tmp_path):
    names = ["n01/éclair_ü.JPEG", "n02/猫.JPEG", os.fsdecode(b"n03/\xff\xfe.JPEG")]
    src = data.JpegIndex.empty(FOLDER)
    learn(src, names)
    delta = src.delta()
    buf = distributed._pack_delta(*delta)
    back = distributed._unpack_delta(buf)
    assert back[0] == [bytes(p) for p in delta[0]]
    for a, b in zip(back[1:], delta[1:]):
        assert a.tobytes() == b.tobytes()
    dst = data.JpegIndex.empty(FOLDER)
    dst.merge(*back)
    assert entries(dst, names) == entries(src, names) and all(entries(dst, names).values())
    out = str(tmp_path / "train.npz")
    dst.save(out)
    assert entries(data.JpegIndex.load(out, FOLDER), names) == entries(src, names)
    empty = data.JpegIndex.empty(FOLDER).delta()
    assert empty[0].size == 0 and empty[1].size == 0 and empty[2].tolist() == [0] and empty[3].size == 0
    assert distributed._pack_delta(*empty).size == 0
    dst.merge(*empty)
    dst.merge([], [], [0], np.zeros(0, SYNC))
    assert entries(dst, names) == entries(src, names)


@pytest.mark.parametrize("bad", [
    ([b"a"], [1, 2], [0, 1], 1),                   # a length too many
    ([b"a"], [1], [0], 0),                         # no end offset
    ([b"a", b"b"], [1, 1], [0, 2, 1], 2),          # offsets go back
    ([b"a"], [1], [1, 2], 2),                      # offsets start past 0
    ([b"a"], [1], [0, 3], 2),                      # offsets past the points
    ([b"a"], [-1], [0, 1], 1),                     # a negative length
    ([b""], [1], [0, 1], 1),                       # an empty path
    ([b"/etc/x"], [1], [0, 1], 1),                 # an absolute path
])
def test_malformed_merges_raise_and_enter_nothing(bad):
    paths, lengths, first, n = bad
    idx = data.JpegIndex.empty(FOLDER)
    with pytest.raises(ValueError):
        idx.merge(paths, lengths, first, pts(0, n))
    assert not idx._merged and idx.lookup(os.path.join(FOLDER, "a"), 1).size == 0
    with pytest.raises(ValueError):
        idx.merge([b"a"], [1], [0, 1], np.zeros(16, np.uint8))  # points of another dtype


def test_packed_deltas_of_the_wrong_size_do_not_unpack():
    src = data.JpegIndex.empty(FOLDER)
    learn(src, ["a.JPEG", "bb.JPEG"])
    buf = distributed._pack_delta(*src.delta())
    for cut in (buf[:10], buf[:-1], np.concatenate([buf, buf[:1]])):
        with pytest.raises(ValueError):
            distributed._unpack_delta(cut)
    wrong = buf.copy()
    wrong[24 + 8 * 2:24 + 8 * 3] = np.array([99], np.int64).view(np.uint8)   # a path length past the names
    with pytest.raises(ValueError):
        distributed._unpack_delta(wrong)


# ---- the exchange over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _snapshot(idx, names):
    return {n: idx.lookup(os.path.join(FOLDER, n), 1000).tobytes().hex() for n in names}


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from fast_autoaugment_b200 import data as d, distributed as dd

    calls = []
    real = dd.gather_pool

    def spy(t, group=None):
        calls.append(int(t.numel()))
        return real(t, group)
    dd.gather_pool = spy
    res = {}

    # disjoint and overlapping deltas: rank r learns its own files and the shared ones (same points on every rank, as
    # the placement rule gives them)
    idx = d.JpegIndex.empty(FOLDER)
    own = {r: ["n%d/own_%d.JPEG" % (r, i) for i in range(3 + r)] for r in range(world)}
    shared = ["shared_%d.JPEG" % i for i in range(4)]
    for name in own[rank] + shared[rank % 2::2] + shared[:1]:
        q = pts(hash_name(name), 1 + hash_name(name) % 9)
        idx.add([os.path.join(FOLDER, name)], [1000], [0, len(q)], q)
    everything = [n for r in range(world) for n in own[r]] + shared
    merged = dd.share_jpeg_index(idx)
    res["merged"] = merged
    res["union"] = _snapshot(idx, everything)
    res["want"] = {n: pts(hash_name(n), 1 + hash_name(n) % 9).tobytes().hex() for n in everything}
    res["calls_first"] = list(calls)
    saved = os.path.join(out_dir, "rank%d.npz" % rank)
    idx.save(saved)
    res["saved"] = _snapshot(d.JpegIndex.load(saved, FOLDER), everything)

    # a second exchange with nothing new sends only the sizes
    calls.clear()
    res["merged_second"] = dd.share_jpeg_index(idx)
    res["calls_second"] = list(calls)

    # a chunk size of 40 bytes: several rounds, and only rank 0 learned something
    calls.clear()
    late = ["late_%d.JPEG" % i for i in range(5)]
    if rank == 0:
        for name in late:
            q = pts(hash_name(name), 20)
            idx.add([os.path.join(FOLDER, name)], [1000], [0, len(q)], q)
    res["merged_chunked"] = dd.share_jpeg_index(idx, chunk_bytes=40)
    res["calls_chunked"] = list(calls)
    res["late"] = _snapshot(idx, late)
    res["late_want"] = {n: pts(hash_name(n), 20).tobytes().hex() for n in late}

    # rank 1's delta is malformed (a length too many): every rank raises, naming it
    if rank == 1:
        learn(idx, ["bad.JPEG"])
        good = idx.delta
        idx.delta = lambda: (lambda p, n, f, q: (p, np.concatenate([n, n]), f, q))(*good())
    try:
        dd.share_jpeg_index(idx)
        res["malformed"] = None
    except RuntimeError as e:
        res["malformed"] = str(e)
    res["bad_entered"] = idx.lookup(os.path.join(FOLDER, "bad.JPEG"), 1000).size

    # a local failure before anything is sent: every rank raises, naming the rank
    if rank == world - 1:
        def broken():
            raise OSError("no delta here")
        idx.delta = broken
    try:
        dd.share_jpeg_index(idx)
        res["local"] = None
    except RuntimeError as e:
        res["local"] = str(e)
    dist.barrier()                                                 # the group is still usable
    with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
        json.dump(res, f)
    dist.destroy_process_group()


def hash_name(name):
    return sum((i + 1) * c for i, c in enumerate(name.encode())) % 1000


@pytest.mark.parametrize("world", [2, 3])
def test_share_jpeg_index_over_gloo(tmp_path, world):
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    res = []
    for r in range(world):
        with open(os.path.join(tmp_path, "rank%d.json" % r)) as f:
            res.append(json.load(f))
    late_bytes = 24 + 8 * (3 * 5 + 1) + 16 * 20 * 5 + 5 * len("late_0.JPEG")      # rank 0's packed delta
    for r, x in enumerate(res):
        assert x["union"] == x["want"] == x["saved"], r             # every rank lists every rank's files
        assert len(x["calls_first"]) == 3 and x["calls_first"][0] == x["calls_first"][2] == 1, r   # sizes, data, flags
        assert x["merged"] > 0
        assert x["merged_second"] == 0 and x["calls_second"] == [1], r
        rounds = x["calls_chunked"][1:-1]
        assert x["calls_chunked"][0] == x["calls_chunked"][-1] == 1 and len(rounds) == -(-late_bytes // 40), r
        assert rounds == [40] * (len(rounds) - 1) + [late_bytes - 40 * (len(rounds) - 1)], r   # bytes sent per rank
        assert x["late"] == x["late_want"], r
        assert x["merged_chunked"] == (5 if r else 0)
        assert x["malformed"] is not None and "rank 1's JPEG index delta is malformed" in x["malformed"], r
        assert (x["bad_entered"] > 0) == (r == 1), r                 # learned on rank 1, entered nowhere else
        assert x["local"] is not None and "rank %d: OSError: no delta here" % (world - 1) in x["local"], r
