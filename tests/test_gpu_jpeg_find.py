"""The scan index found on the device in parallel (``build_jpeg_index(find=True)``, C ABI ``faa_jpeg_index_find``) and
the decode that finds one first (``decode_jpeg(find=True)``, ``faa_jpeg_decode`` with ``find``).  The found points equal the
host build's (tests/emu/faa_emu_jpeg_find.cpp at the kernel's window and rounds) byte for byte, and
``build_jpeg_index``'s where the chain converged; the found decode's pixels and status equal the plain decode's on the
grid, the geometry streams, the adversarial streams and corrupt files; a batch mixing given, stale, foreign and absent
points with progressive files gets the counts of ``record=True`` right; a call queued behind one that grows the
decoder's buffers; three launches per call; the ABI's refusals; and ``conf['faa_jpeg_index_find']`` in the loaders."""
import os

import numpy as np
import pytest
import torch

import jpeg_index_cases as jic
import jpeg_progressive_cases as jp
from imagenet_tree import write_tree
from jpeg_cases import content, encode, make
from test_gpu_imagenet_folder import B, assert_same, conf_set, run
from test_gpu_jpeg import launches, sentinel_out, untouched_outside
from test_gpu_jpeg_geometries import GROUPS
from test_gpu_jpeg_index import GRID_BATCHES
from test_gpu_jpeg_record import _bigger_files
from test_jpeg_find_host import ADVERSARIAL, CORRUPT, KERNEL_R, KERNEL_W, find, load_emu_find

from fast_autoaugment_b200 import _lib, data, engine
from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, compact_jpeg_index, decode_jpeg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emu():
    return load_emu_find()


def _ranges(first, points, i):
    return points[first[i]:first[i + 1]]


def check_index(emu, files):
    """the device's found index equals the host build's; it is a prefix of the serial build's, all of it when the
    host says the chain converged; returns the number of converged files"""
    enc = EncodedImages.from_bytes(files)
    ff, fp = build_jpeg_index(enc, find=True)
    bf, bp = build_jpeg_index(enc)
    conv = 0
    for i, b in enumerate(files):
        host, (_, _, _, full) = find(emu, b, KERNEL_W, KERNEL_R)
        got, built = _ranges(ff, fp, i), _ranges(bf, bp, i)
        assert got.tobytes() == host.tobytes(), i
        if len(built):                                   # a file whose serial decode is clean
            assert got.tobytes() == built[:len(got)].tobytes(), i
            if full:
                assert got.tobytes() == built.tobytes(), i
                conv += 1
    return conv


def check_decode(files):
    enc = EncodedImages.from_bytes(files)
    out_a, out_b = sentinel_out(enc.sizes), sentinel_out(enc.sizes)
    _, st_a = decode_jpeg(enc, out_a)
    _, st_b = decode_jpeg(enc, out_b, find=True)
    torch.cuda.synchronize()
    assert untouched_outside(out_b)
    assert torch.equal(st_a, st_b) and torch.equal(out_a.storage, out_b.storage)
    return st_a.cpu().numpy()


@pytest.mark.parametrize("k", range(len(GRID_BATCHES)))
def test_grid_found_index_equals_host_and_decodes_the_same(emu, k):
    files = [make(c)[0] for c in GRID_BATCHES[k]]
    check_index(emu, files)
    check_decode(files)


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_geometry_streams_found_index_equals_host_and_decodes_the_same(emu, group):
    files = [b for _, b in GROUPS[group]]
    for k in range(0, len(files), 64):
        check_index(emu, files[k:k + 64])
        check_decode(files[k:k + 64])


def test_adversarial_streams_and_photos(emu):
    files = [b for _, b in ADVERSARIAL] + [b for _, b in jic.indexed_files()]
    assert check_index(emu, files) >= len(jic.indexed_files())
    assert (check_decode(files) == 0).all()


def test_corrupt_files_decode_as_without_a_find(emu):
    files = []
    for _, b in CORRUPT:
        if engine.parse_jpeg(b)[0] is not None:
            files.append(b)
    check_index(emu, files)
    assert (check_decode(files) != 0).sum() > 10


def test_mixed_batch_counts():
    a = content("photo", 375, 500, 7)
    own = encode(a, quality=90, subsampling=2)                          # its own points: used, count 0
    stale = encode(content("photo", 375, 500, 8), quality=90, subsampling=2)    # another file's points: recorded
    restart = encode(a, quality=90, restart_marker_blocks=4)            # a restart interval: nothing
    absent = encode(content("photo", 240, 320, 3), quality=90)          # no points: found, converged
    flat = encode(np.full((64, 64, 3), 90, np.uint8), quality=75)       # under 2 KiB: nothing
    big = jic.big_file()                                                # garbage points: recorded
    prog = jp.encode(content("photo", 120, 160, 5), progressive=True, quality=85, subsampling=2)
    files = [own, stale, restart, absent, flat, big, prog, absent]
    enc = EncodedImages.from_bytes(files, progressive=True)
    want_first, want_pts = build_jpeg_index(enc)
    mine = _ranges(want_first, want_pts, 0)
    garbage = np.frombuffer(np.random.default_rng(3).integers(0, 256, 40 * 16, dtype=np.uint8).tobytes(), jic.SYNC)
    given = [mine, mine, mine, mine[:0], mine[:0], garbage, mine[:0], mine[:0]]
    f = np.concatenate([[0], np.cumsum([len(q) for q in given])]).astype(np.int64)
    idx = enc.with_index(f, np.concatenate(given))
    out_a, out_b = sentinel_out(enc.sizes), sentinel_out(enc.sizes)
    _, st_a = decode_jpeg(EncodedImages.from_bytes(files, progressive=True), out_a)
    _, st_b, count, points, cap_first = decode_jpeg(idx, out_b, record=True, find=True)
    torch.cuda.synchronize()
    assert untouched_outside(out_b)
    assert torch.equal(st_a, st_b) and torch.equal(out_a.storage, out_b.storage) and st_a.tolist() == [0] * 8
    count = count.cpu().numpy()
    first, pts = compact_jpeg_index(cap_first, count, points.cpu().numpy())
    assert [int(c) > 0 for c in count] == [False, True, False, True, False, True, False, True]
    for i in (1, 3, 5, 7):
        assert _ranges(first, pts, i).tobytes() == _ranges(want_first, want_pts, i).tobytes(), i
    # without record the same pixels and status
    out_c = sentinel_out(enc.sizes)
    _, st_c = decode_jpeg(idx, out_c, find=True)
    torch.cuda.synchronize()
    assert torch.equal(st_a, st_c) and torch.equal(out_a.storage, out_c.storage)


def test_found_decode_queued_behind_a_call_that_grows_the_buffers():
    small = [encode(content("photo", 96, 128, s), quality=90) for s in range(3)]
    large = [encode(content("photo", 600, 800, s), quality=95) for s in range(6)]
    e_small, e_large = EncodedImages.from_bytes(small), EncodedImages.from_bytes(large)
    ref_s, _ = decode_jpeg(e_small)
    ref_l, _ = decode_jpeg(e_large)
    torch.cuda.synchronize()
    engine._DECODERS.clear()                                            # a fresh decoder: its buffers start small
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        r1 = decode_jpeg(e_small, find=True)
        r2 = decode_jpeg(e_large)                                       # grows every buffer, in stream order
        r3 = decode_jpeg(e_large, find=True)
        r4 = decode_jpeg(e_small, record=True, find=True)
    torch.cuda.synchronize()
    for r, ref in ((r1, ref_s), (r2, ref_l), (r3, ref_l), (r4, ref_s)):
        assert torch.equal(r[0].storage, ref.storage) and r[1].cpu().tolist() == [0] * len(r[1])


def test_three_launches_per_found_decode_and_one_per_find():
    files = [encode(content("photo", 240, 320, i), quality=90, subsampling=2) for i in range(4)]
    files.append(encode(content("photo", 64, 48, 9), quality=80, restart_marker_blocks=2))
    enc = EncodedImages.from_bytes(files)
    out = engine.RaggedImages.empty(enc.sizes)
    decode_jpeg(enc, out, find=True)
    for kw in ({}, {"record": True}):
        c0 = launches()
        decode_jpeg(enc, out, find=True, **kw)
        assert launches() - c0 == 3
    c0 = launches()
    build_jpeg_index(enc, find=True)
    assert launches() - c0 == 1


def test_abi_refuses_progressive_headers_and_bad_offsets():
    enc = EncodedImages.from_bytes([encode(content("photo", 96, 128, 2), quality=95)] * 2)
    pen = EncodedImages.from_bytes([jp.encode(content("photo", 96, 128, 2), progressive=True, quality=95)] * 2,
                                   progressive=True)
    out = sentinel_out(enc.sizes)
    h_out, d_out = out.descriptors()
    st = torch.empty(2, dtype=torch.int32, device="cuda")
    cnt = torch.empty(2, dtype=torch.int32, device="cuda")
    pts = torch.empty(16 * 64, dtype=torch.uint8, device="cuda")
    decode_jpeg(enc, out)
    dec = engine._DECODERS[enc.device.index]
    good = np.array([0, 8, 16], np.int64)
    d_good = torch.from_numpy(good).cuda()

    def find_call(e, f, d_f):
        return _lib.lib.faa_jpeg_index_find(e.headers.ctypes.data, e.device_headers().data_ptr(),
                                            e.device_pool().data_ptr(), len(e.pool), e.storage.data_ptr(), 2,
                                            f.ctypes.data, d_f.data_ptr(), pts.data_ptr(), cnt.data_ptr(), None)

    def decode_call(e, f, d_f):
        return _lib.lib.faa_jpeg_decode(dec.handle, e.headers.ctypes.data, e.device_headers().data_ptr(),
                                        e.device_pool().data_ptr(), len(e.pool), e.storage.data_ptr(), 2,
                                        h_out.ctypes.data, d_out.data_ptr(), st.data_ptr(), None, None, None,
                                        f.ctypes.data, d_f.data_ptr(), pts.data_ptr(), cnt.data_ptr(), 1, None)
    for call in (find_call, decode_call):
        assert call(enc, good, d_good) == _lib.OK
        assert call(pen, good, d_good) == _lib.ERR_VALUE
        for bad in ([1, 0, 2], [-1, 0, 0], [0, 2, 1]):
            f = np.array(bad, np.int64)
            assert call(enc, f, torch.from_numpy(f).cuda()) == _lib.ERR_VALUE
    torch.cuda.synchronize()


# ---- the loaders
def test_loaders_with_the_key_on_and_off(tmp_path, monkeypatch):
    root = str(tmp_path / "data")
    write_tree(root, 43, n_classes=3, per_class=10, n_val=6)            # refused files included
    _bigger_files(root, 1)
    with conf_set():
        torch.manual_seed(0)
        plain = data.get_dataloaders("imagenet", B, root, split=0.2)
    with conf_set(faa_jpeg_index_find=True):
        torch.manual_seed(0)
        found = data.get_dataloaders("imagenet", B, root, split=0.2)
    with conf_set(faa_jpeg_index_find=True, faa_jpeg_index_learn=True):
        torch.manual_seed(0)
        learn = data.get_dataloaders("imagenet", B, root, split=0.2)
    assert found[1].dataset.find and found[3].dataset.find and not plain[1].dataset.find

    calls = []
    dec = data.decode_jpeg

    def spy(enc, out=None, record=False, find=False):
        calls.append(find)
        return dec(enc, out, record=record, find=find)
    monkeypatch.setattr(data, "decode_jpeg", spy)
    for k, name in ((1, "train"), (2, "valid"), (3, "test")):
        assert_same(run(found[k], 70 + k), run(plain[k], 70 + k), name)
    assert any(calls) and not all(calls)                                # the plain loaders still call without it

    seen = set()
    read = data.read_jpeg_batch

    def read_spy(paths, *a, **kw):
        hb = read(paths, *a, **kw)
        seen.update(hb.paths[i] for i in hb.accepted)
        return hb
    monkeypatch.setattr(data, "read_jpeg_batch", read_spy)
    calls.clear()
    got = [run(learn[1], 81), run(learn[2], 82)]
    assert calls and all(calls)
    with conf_set():                          # fresh loaders: a loader's Philox counter runs on across epochs
        torch.manual_seed(0)
        plain = data.get_dataloaders("imagenet", B, root, split=0.2)
    assert_same(got[0], run(plain[1], 81), "learn, train")
    assert_same(got[1], run(plain[2], 82), "learn, valid")
    idx = learn[1].dataset.index
    train = data.imagenet_split_folder(root, "train")
    paths = [p for p, _ in data.imagenet_index(root, "train")]
    files = [open(p, "rb").read() for p in paths]
    ok = [i for i, b in enumerate(files) if engine.parse_jpeg(b)[0] is not None]
    enc = EncodedImages.from_bytes([files[i] for i in ok])
    bf, bp = build_jpeg_index(enc)
    emu = load_emu_find()
    learned = {os.path.join(train, r) for r in idx._added}
    for j, i in enumerate(ok):                # the files epoch 1 of train + valid read
        if paths[i] not in seen:
            continue
        got = idx.lookup(paths[i], len(files[i]))
        host, (_, _, _, full) = find(emu, files[i], KERNEL_W, KERNEL_R)
        if full and len(host):                # converged: learned (a file found nothing for is recorded serially)
            assert paths[i] in learned, paths[i]
        elif len(host):                       # a prefix that did not converge: decoded with it, not learned
            assert paths[i] not in learned, paths[i]
        assert got.tobytes() == (_ranges(bf, bp, j).tobytes() if paths[i] in learned else b""), paths[i]
    assert len(learned) >= 8

    # EncodedDeviceDataset carries the key too
    ds = data.EncodedDeviceDataset([files[i] for i in ok], [0] * len(ok), find=True)
    assert ds.subset([0, 1]).find
