"""The JPEG scan index on the device: ``build_jpeg_index`` (C ABI ``faa_jpeg_index_build``) equals the host build's
index byte for byte, and ``decode_jpeg`` with an index (``faa_jpeg_decode``'s input points) equals the decode without one, in
pixels and status, on the decoder grid, the geometry streams, fuzzed indexes, 1, 2 and 128 segments and a batch that
mixes indexed, stale, restart-marker and point-less files.  Then the index command on an ImageNet tree, and
``get_dataloaders('imagenet', ...)`` with and without ``conf['faa_jpeg_index']``."""
import os

import numpy as np
import pytest
import torch

import jpeg_index_cases as jic
from imagenet_tree import baseline_file, write, write_tree
from jpeg_cases import GRID, content, encode, make
from test_gpu_imagenet_folder import B, assert_same, conf_set, run
from test_gpu_jpeg import sentinel_out, untouched_outside
from test_gpu_jpeg_geometries import GROUPS

from fast_autoaugment_b200 import _lib, data, engine, jpeg_index
from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, decode_jpeg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emu():
    return jic.load_emu_index()


def host_first_points(emu, files):
    first, pts = [0], []
    for b in files:
        q = jic.host_index(emu, b)[0]
        first.append(first[-1] + len(q))
        pts.append(q)
    return np.array(first, np.int64), np.concatenate(pts) if pts else np.zeros(0, jic.SYNC)


def decode_both(enc, first, points):
    """(pixels, status) of the decode without and with the index, each into sentinel-filled storage"""
    out_a, out_b = sentinel_out(enc.sizes), sentinel_out(enc.sizes)
    _, st_a = decode_jpeg(enc, out_a)
    _, st_b = decode_jpeg(enc.with_index(first, points), out_b)
    torch.cuda.synchronize()
    assert untouched_outside(out_a) and untouched_outside(out_b)
    return out_a.storage.cpu(), st_a.cpu(), out_b.storage.cpu(), st_b.cpu()


def check_batch(emu, files):
    enc = EncodedImages.from_bytes(files)
    first, points = build_jpeg_index(enc)
    hf, hp = host_first_points(emu, files)
    assert np.array_equal(first, hf) and points.tobytes() == hp.tobytes()
    a, sa, b, sb = decode_both(enc, first, points)
    assert torch.equal(sa, sb) and torch.equal(a, b)
    return first


def _grid_batches(n=64):
    return [GRID[k:k + n] for k in range(0, len(GRID), n)]


GRID_BATCHES = _grid_batches()


@pytest.mark.parametrize("k", range(len(GRID_BATCHES)))
def test_grid_device_index_equals_host_and_decodes_the_same(emu, k):
    files = [make(c)[0] for c in GRID_BATCHES[k]]
    check_batch(emu, files)


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_geometry_streams_device_index_equals_host_and_decodes_the_same(emu, group):
    files = [b for _, b in GROUPS[group]]
    for k in range(0, len(files), 64):
        check_batch(emu, files[k:k + 64])


def test_one_two_and_128_segments(emu):
    small = encode(content("noise", 48, 48, 0), quality=95)                  # scan of 2 - 3 KiB: 1 point
    flat = encode(np.full((64, 64, 3), 90, np.uint8), quality=75)            # under 2 KiB: none
    big = jic.big_file()                                                     # 127 points
    first = check_batch(emu, [flat, small, big, small, flat])
    assert np.diff(first).tolist() == [0, 1, 127, 1, 0]


def test_fuzzed_indexes_decode_as_without_one(emu):
    files = [b for _, b in jic.indexed_files()]
    enc = EncodedImages.from_bytes(files)
    first, points = build_jpeg_index(enc)
    for k, b in enumerate(files):
        pts = points[first[k]:first[k + 1]]
        other = points[first[(k + 1) % len(files)]:first[(k + 1) % len(files) + 1]]
        hdr = enc.headers[k]
        cases = jic.fuzzed(pts, other, (int(hdr["scan_off"]), int(hdr["scan_len"])),
                           int(hdr["mcu_x"]) * int(hdr["mcu_y"]), b,
                           jic.host_states(emu, b, int(hdr["mcu_x"]) * int(hdr["mcu_y"])))
        # every fuzzed list of this file in one batch of copies of it
        one = EncodedImages.from_bytes([b] * len(cases))
        f = np.concatenate([[0], np.cumsum([len(q) for _, q in cases])]).astype(np.int64)
        p = np.concatenate([q for _, q in cases])
        a, sa, c, sc = decode_both(one, f, p)
        assert torch.equal(sa, sc) and torch.equal(a, c), k
        assert sa.tolist() == [0] * len(cases)


def test_mixed_batch_only_the_stale_file_falls_back(emu):
    a = content("photo", 375, 500, 7)
    indexed = encode(a, quality=90, subsampling=2)
    stale_src = encode(content("photo", 375, 500, 8), quality=90, subsampling=2)
    restart = encode(a, quality=90, restart_marker_blocks=4)
    pointless = encode(content("photo", 48, 64, 1), quality=75)
    files = [indexed, stale_src, restart, pointless]
    enc = EncodedImages.from_bytes(files)
    first, points = build_jpeg_index(enc)
    assert np.diff(first).tolist()[2:] == [0, 0]
    # the stale file gets the indexed file's points; the restart file gets them too (ignored)
    own = points[first[0]:first[1]]
    n = len(own)
    f = np.array([0, n, 2 * n, 3 * n, 3 * n], np.int64)              # the point-less file gets none
    p = np.concatenate([own, own, own])
    assert [jic.linked(emu, b, p[f[i]:f[i + 1]]) for i, b in enumerate(files)] == [1, 0, 0, 0]
    x, sx, y, sy = decode_both(enc, f, p)
    assert torch.equal(sx, sy) and torch.equal(x, y) and sx.tolist() == [0] * 4


def test_abi_refuses_bad_point_offsets():
    b = [encode(content("photo", 96, 128, 2), quality=95)] * 2
    enc = EncodedImages.from_bytes(b)
    first, points = build_jpeg_index(enc)
    out = sentinel_out(enc.sizes)
    h_out, d_out = out.descriptors()
    st = torch.empty(2, dtype=torch.int32, device="cuda")
    decode_jpeg(enc, out)
    dec = engine._DECODERS[enc.device.index]
    for bad in ([1, 0, 2], [-1, 0, 0], [0, 2, 1]):
        f = np.array(bad, np.int64)
        d_f = torch.from_numpy(f).cuda()
        e = _lib.lib.faa_jpeg_decode(dec.handle, enc.headers.ctypes.data, enc.device_headers().data_ptr(),
                                     enc.device_pool().data_ptr(), len(enc.pool), enc.storage.data_ptr(), 2,
                                     h_out.ctypes.data, d_out.data_ptr(), st.data_ptr(),
                                     enc.with_index(first, points).device_index()[1].data_ptr(),
                                     f.ctypes.data, d_f.data_ptr(), *(None,) * 8, 0, None)
        assert e == _lib.ERR_VALUE
        cnt = torch.empty(2, dtype=torch.int32, device="cuda")
        e = _lib.lib.faa_jpeg_index_build(enc.headers.ctypes.data, enc.device_headers().data_ptr(),
                                          enc.device_pool().data_ptr(), len(enc.pool), enc.storage.data_ptr(), 2,
                                          f.ctypes.data, d_f.data_ptr(), None, cnt.data_ptr(), st.data_ptr(), None)
        assert e == _lib.ERR_VALUE
    torch.cuda.synchronize()


def test_index_command_and_loaders_with_and_without_the_index(tmp_path):
    root = str(tmp_path / "data")
    write_tree(root, 31, n_classes=3, per_class=10, n_val=6)
    # bigger files, so that most of the tree is indexed
    train = data.imagenet_split_folder(root, "train")
    for k, (dirpath, _, names) in enumerate(sorted(os.walk(train))):
        for j, n in enumerate(sorted(names)):
            if n.startswith("train_") and j % 2 == 0:
                write(os.path.join(dirpath, n), encode(content("photo", 240, 320, 100 * k + j), quality=90,
                                                       subsampling=j % 3))
    out = str(tmp_path / "index")
    jpeg_index.main([root, out])
    idx = data.JpegIndex.load(os.path.join(out, "train.npz"), train)
    assert len(idx.points) > 0 and (np.diff(idx.first) > 0).sum() >= 10
    # after indexing: one indexed file rewritten with other content (same length would be caught on the device; a
    # new length is caught by the lookup), and one file added
    paths = [p for p, _ in data.imagenet_index(root, "train")]
    victim = next(p for p in paths if len(idx.lookup(p, os.path.getsize(p))) > 0)
    write(victim, encode(content("photo", 240, 320, 999), quality=85))
    write(os.path.join(train, "n00001000", "added.JPEG"), baseline_file(3, 77))
    for parity in (False, True):
        with conf_set(faa_parity=parity):
            torch.manual_seed(0)
            plain = data.get_dataloaders("imagenet", B, root, split=0.2)
        with conf_set(faa_parity=parity, faa_jpeg_index=out):
            torch.manual_seed(0)
            indexed = data.get_dataloaders("imagenet", B, root, split=0.2)
        assert indexed[1].dataset.index is not None and plain[1].dataset.index is None
        assert list(indexed[0].indices) == list(plain[0].indices)
        for which in (1, 2, 3):
            assert_same(run(indexed[which], 40 + which), run(plain[which], 40 + which), (parity, which))
