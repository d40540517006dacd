"""The recording JPEG decode on the device (``decode_jpeg(record=True)``, C ABI ``faa_jpeg_decode`` with its recording outputs): its
pixels and status equal the plain decode's, and its compacted points equal ``build_jpeg_index``'s byte for byte, on the
decoder grid, the geometry streams and a batch mixing used, stale, foreign and absent points; a recording call queued
behind a call that grows the decoder's buffers.  Then ``conf['faa_jpeg_index_learn']`` on an ImageNet tree: the same
batches as without it, the index it learns, its use in epoch 2, and a file rewritten between epochs."""
import os

import numpy as np
import pytest
import torch

import jpeg_index_cases as jic
from imagenet_tree import write, write_tree
from jpeg_cases import content, encode, make
from test_gpu_imagenet_folder import B, assert_same, conf_set, run
from test_gpu_jpeg import sentinel_out, untouched_outside
from test_gpu_jpeg_geometries import GROUPS
from test_gpu_jpeg_index import GRID_BATCHES

from fast_autoaugment_b200 import _lib, data, engine, jpeg_index
from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, compact_jpeg_index, decode_jpeg

pytestmark = pytest.mark.gpu


def plain_and_recorded(enc):
    """(plain pixels, plain status, recorded pixels, recorded status, count, (first, points) compacted)"""
    out_a, out_b = sentinel_out(enc.sizes), sentinel_out(enc.sizes)
    _, st_a = decode_jpeg(EncodedImages(enc.storage, enc.headers, enc.pool), out_a)
    _, st_b, count, points, cap_first = decode_jpeg(enc, out_b, record=True)
    torch.cuda.synchronize()
    assert untouched_outside(out_a) and untouched_outside(out_b)
    count = count.cpu().numpy()
    assert np.array_equal(cap_first, engine.jpeg_index_capacities(enc.headers))
    return (out_a.storage.cpu(), st_a.cpu(), out_b.storage.cpu(), st_b.cpu(), count,
            compact_jpeg_index(cap_first, count, points.cpu().numpy()))


def check_batch(files):
    enc = EncodedImages.from_bytes(files)
    want = build_jpeg_index(enc)
    a, sa, b, sb, count, (first, points) = plain_and_recorded(enc)
    assert torch.equal(sa, sb) and torch.equal(a, b)
    assert np.array_equal(first, want[0]) and points.tobytes() == want[1].tobytes()
    return count


@pytest.mark.parametrize("k", range(len(GRID_BATCHES)))
def test_grid_recording_equals_plain_and_index_build(k):
    check_batch([make(c)[0] for c in GRID_BATCHES[k]])


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_geometry_streams_recording_equals_plain_and_index_build(group):
    files = [b for _, b in GROUPS[group]]
    for k in range(0, len(files), 64):
        check_batch(files[k:k + 64])


def test_mixed_points_record_exactly_the_serial_files():
    a = content("photo", 375, 500, 7)
    own = encode(a, quality=90, subsampling=2)                          # its own points: used
    stale = encode(content("photo", 375, 500, 8), quality=90, subsampling=2)    # another file's points
    restart = encode(a, quality=90, restart_marker_blocks=4)            # points of a restart file: ignored
    absent = encode(content("photo", 240, 320, 3), quality=90)          # no points
    flat = encode(np.full((64, 64, 3), 90, np.uint8), quality=75)       # under 2 KiB: no index
    big = jic.big_file()                                                # garbage points
    files = [own, stale, restart, absent, flat, big]
    enc = EncodedImages.from_bytes(files)
    want_first, want_pts = build_jpeg_index(enc)
    mine = want_pts[want_first[0]:want_first[1]]
    garbage = np.frombuffer(np.random.default_rng(3).integers(0, 256, 40 * 16, dtype=np.uint8).tobytes(), jic.SYNC)
    given = [mine, mine, mine, mine[:0], mine[:0], garbage]
    f = np.concatenate([[0], np.cumsum([len(q) for q in given])]).astype(np.int64)
    x, sx, y, sy, count, (first, points) = plain_and_recorded(enc.with_index(f, np.concatenate(given)))
    assert torch.equal(sx, sy) and torch.equal(x, y) and sx.tolist() == [0] * 6
    serial = [False, True, False, True, False, True]                    # decoded whole by thread 0 with rule points
    assert [int(c) > 0 for c in count] == serial
    for i in range(6):
        got = points[first[i]:first[i + 1]]
        want = want_pts[want_first[i]:want_first[i + 1]] if serial[i] else want_pts[:0]
        assert got.tobytes() == want.tobytes(), i


def test_recording_queued_behind_a_call_that_grows_the_buffers():
    small = [encode(content("photo", 96, 128, s), quality=90) for s in range(3)]
    large = [encode(content("photo", 600, 800, s), quality=95) for s in range(6)]
    e_small, e_large = EncodedImages.from_bytes(small), EncodedImages.from_bytes(large)
    want_s, want_l = build_jpeg_index(e_small), build_jpeg_index(e_large)
    ref_s, _ = decode_jpeg(e_small)
    ref_l, _ = decode_jpeg(e_large)
    torch.cuda.synchronize()
    engine._DECODERS.clear()                                            # a fresh decoder: its buffers start small
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        r1 = decode_jpeg(e_small, record=True)
        out_l, st_l = decode_jpeg(e_large)                              # grows every buffer, in stream order
        r2 = decode_jpeg(e_large, record=True)
        r3 = decode_jpeg(e_small, record=True)
    torch.cuda.synchronize()
    assert torch.equal(out_l.storage, ref_l.storage) and st_l.tolist() == [0] * 6
    for (out, st, cnt, pts, cap), ref, want in ((r1, ref_s, want_s), (r2, ref_l, want_l), (r3, ref_s, want_s)):
        assert torch.equal(out.storage, ref.storage) and st.cpu().tolist() == [0] * len(st)
        first, points = compact_jpeg_index(cap, cnt.cpu().numpy(), pts.cpu().numpy())
        assert np.array_equal(first, want[0]) and points.tobytes() == want[1].tobytes()
    assert int(np.diff(want_l[0]).min()) > 0


def test_abi_refuses_bad_capacity_offsets():
    enc = EncodedImages.from_bytes([encode(content("photo", 96, 128, 2), quality=95)] * 2)
    out = sentinel_out(enc.sizes)
    h_out, d_out = out.descriptors()
    st = torch.empty(2, dtype=torch.int32, device="cuda")
    cnt = torch.empty(2, dtype=torch.int32, device="cuda")
    pts = torch.empty(16 * 64, dtype=torch.uint8, device="cuda")
    decode_jpeg(enc, out)
    dec = engine._DECODERS[enc.device.index]
    for bad in ([1, 0, 2], [-1, 0, 0], [0, 2, 1]):
        f = np.array(bad, np.int64)
        d_f = torch.from_numpy(f).cuda()
        e = _lib.lib.faa_jpeg_decode(dec.handle, enc.headers.ctypes.data, enc.device_headers().data_ptr(),
                                     enc.device_pool().data_ptr(), len(enc.pool), enc.storage.data_ptr(), 2,
                                     h_out.ctypes.data, d_out.data_ptr(), st.data_ptr(), None, None, None,
                                     f.ctypes.data, d_f.data_ptr(), pts.data_ptr(), cnt.data_ptr(), 0, None)
        assert e == _lib.ERR_VALUE
    torch.cuda.synchronize()


# ---- the loaders
def _bigger_files(root, seed):
    """photo-like 240 x 320 files in place of half the train files, so that most of the tree gets points"""
    train = data.imagenet_split_folder(root, "train")
    for k, (dirpath, _, names) in enumerate(sorted(os.walk(train))):
        for j, n in enumerate(sorted(names)):
            if n.startswith("train_") and j % 2 == 0:
                write(os.path.join(dirpath, n), encode(content("photo", 240, 320, seed + 100 * k + j), quality=90,
                                                       subsampling=j % 3))


def test_learning_loaders(tmp_path, monkeypatch):
    root = str(tmp_path / "data")
    write_tree(root, 41, n_classes=3, per_class=10, n_val=6)            # refused files included
    _bigger_files(root, 0)
    train = data.imagenet_split_folder(root, "train")
    with conf_set():
        torch.manual_seed(0)
        plain = data.get_dataloaders("imagenet", B, root, split=0.2)
    with conf_set(faa_jpeg_index_learn=True):
        torch.manual_seed(0)
        learn = data.get_dataloaders("imagenet", B, root, split=0.2)
    idx = learn[1].dataset.index
    assert plain[1].dataset.index is None and learn[2].dataset.index is idx and len(idx._added) == 0
    assert learn[3].dataset.index is not idx

    staged, decoded = [], []
    read, dec = data.read_jpeg_batch, data.decode_jpeg

    def read_spy(paths, *a, **kw):
        hb = read(paths, *a, **kw)
        if len(hb.accepted):
            staged.append([hb.paths[i] for i in hb.accepted])
        return hb

    def decode_spy(enc, out=None, record=False):
        r = dec(enc, out, record=record)
        decoded.append((np.diff(enc.first) if enc.first is not None else None, r[2] if record else None))
        return r
    monkeypatch.setattr(data, "read_jpeg_batch", read_spy)
    monkeypatch.setattr(data, "decode_jpeg", decode_spy)

    # epoch 1 of the train and valid loaders: the same batches; every accepted file they read that the placement
    # rule gives points is learned, with the points the index command writes for it; refused files are not
    got = [run(learn[1], 51), run(learn[2], 52)]
    seen = {p for b in staged for p in b}
    assert_same(got[0], run(plain[1], 51), "train, epoch 1")
    assert_same(got[1], run(plain[2], 52), "valid, epoch 1")
    ref_dir = str(tmp_path / "index")
    jpeg_index.main([root, ref_dir])
    ref = data.JpegIndex.load(os.path.join(ref_dir, "train.npz"), train)
    all_train = [p for p, _ in data.imagenet_index(root, "train")]
    learned = {os.path.join(train, r) for r in idx._added}
    assert learned == {p for p in seen if len(ref.lookup(p, os.path.getsize(p))) > 0} and len(learned) >= 8
    for p in all_train:
        n = os.path.getsize(p)
        assert idx.lookup(p, n).tobytes() == (ref.lookup(p, n).tobytes() if p in learned else b""), p
    refused = [p for p in all_train if engine.parse_jpeg(open(p, "rb").read())[0] is None]
    assert refused and not learned & set(refused)
    saved = str(tmp_path / "learned.npz")
    idx.save(saved)
    back = data.JpegIndex.load(saved, train)
    for p in all_train:
        assert back.lookup(p, os.path.getsize(p)).tobytes() == idx.lookup(p, os.path.getsize(p)).tobytes()

    # a learned file of the valid split rewritten at the same length; epoch 2: the learned files carry their points
    # into the decode and are not recorded again, the rewritten one is decoded serially and gets fresh points
    valid = {learn[2].dataset.paths[int(i)] for i in learn[2].sampler.indices}
    victim = sorted(learned & valid)[0]
    old = open(victim, "rb").read()
    new = encode(content("photo", 240, 320, 4242), quality=60)
    assert len(new) < len(old)
    write(victim, new + b"\x00" * (len(old) - len(new)))
    staged.clear()
    decoded.clear()
    got = [run(learn[1], 61), run(learn[2], 62)]
    assert len(decoded) == len(staged)
    hit = set()
    for (counts, rec), paths in zip(decoded, staged):
        for p, c, r in zip(paths, counts, rec.cpu().numpy()):
            if p in learned:
                hit.add(p)
                assert c > 0 and (r > 0) == (p == victim), p
    assert victim in hit and len(hit) >= 8
    assert_same(got[0], run(plain[1], 61), "train, epoch 2")
    assert_same(got[1], run(plain[2], 62), "valid, epoch 2")
    fresh = build_jpeg_index(EncodedImages.from_bytes([open(victim, "rb").read()]))[1]
    assert len(fresh) > 0 and idx.lookup(victim, len(old)).tobytes() == fresh.tobytes()
    assert idx.lookup(victim, len(old)).tobytes() != ref.lookup(victim, len(old)).tobytes()
    assert_same(run(learn[3], 54), run(plain[3], 54), "test")
