"""The progressive JPEG decoder on the device (``decode_jpeg`` of ``EncodedImages.from_bytes(..., progressive=True)``,
C ABI ``faa_jpeg_decode`` with scans): pixels and status equal the host build's and Pillow's on the Pillow grid, at
every reconstruct-tile residue, at restart segment counts 1, 127 to 129 and thousands (waves with more work items than
threads); corrupt streams give the host build's status; batches mixing progressive files with baseline, indexed and
restart-interval files give every file the pixels and status of its decode alone; a call on a second stream grows
every buffer while the first is still queued."""
import numpy as np
import pytest
import torch

import jpeg_progressive_cases as jp
from jpeg_cases import content, encode
from test_gpu_jpeg import sentinel_out, untouched_outside
from test_jpeg_progressive_host import _sos_offsets

from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, decode_jpeg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emu():
    return jp.load_emu()


def device_decode(files, **kw):
    enc = EncodedImages.from_bytes(files, progressive=True)
    if kw.get("index"):
        enc = enc.with_index(*build_jpeg_index(enc))
    out = sentinel_out(enc.sizes)
    _, st = decode_jpeg(enc, out)
    torch.cuda.synchronize()
    assert untouched_outside(out)
    return [out.image(i).cpu().numpy() for i in range(len(files))], st.cpu().numpy()


def _chunks(items, n):
    return [items[i:i + n] for i in range(0, len(items), n)]


@pytest.mark.parametrize("chunk", _chunks(jp.GRID, 24), ids=lambda c: "%s..%s" % (c[0][0], c[-1][0]))
def test_grid_equals_host_build_and_pillow(emu, chunk):
    files = [jp.grid_files(e) for e in chunk]
    px, st = device_decode(files)
    for b, p, s in zip(files, px, st):
        hs, hp, _ = jp.decode(emu, b)
        assert s == hs == 0
        assert np.array_equal(p, hp) and np.array_equal(p, jp.pillow(b))


def _geometry_files():
    # every residue of the 64 x 32 reconstruct tile, each sampling, and restart segment counts 1, 127-129, thousands
    files = []
    for k, (h, w) in enumerate([(32 + r, 64 + 4 * r) for r in range(16)] + [(31 - r, 63 - 4 * r) for r in range(16)]):
        files.append(jp.encode(content("photo", h, w, k), progressive=True, quality=85, subsampling=k % 3))
    for n in (127, 128, 129):
        files.append(jp.encode(content("noise", 8, 8 * n, n), gray=True, progressive=True, quality=90,
                               restart_marker_blocks=1))
    files.append(jp.encode(content("photo", 375, 500, 9), progressive=True, quality=90, subsampling=2,
                           restart_marker_blocks=1))
    return files


def test_geometries_and_restart_segment_counts(emu):
    files = _geometry_files()
    px, st = device_decode(files)
    for b, p, s in zip(files, px, st):
        hs, hp, _ = jp.decode(emu, b)
        assert s == hs == 0
        assert np.array_equal(p, hp) and np.array_equal(p, jp.pillow(b))


def test_corrupt_streams_give_the_host_status(emu):
    rng = np.random.default_rng(11)
    bases = [jp.encode(content("photo", 48, 72, 2), progressive=True, quality=85, subsampling=2, restart_marker_blocks=2),
             jp.encode(content("photo", 40, 40, 3), progressive=True, quality=70, subsampling=0)]
    files = []
    for k in range(160):
        base = bases[k % 2]
        b = bytearray(base)
        lo = _sos_offsets(base)[0] + 12
        for _ in range(1 + k % 4):
            b[int(rng.integers(lo, len(b) - 2))] = int(rng.integers(0, 256))
        if jp.parse(emu, bytes(b))[0] == 0:
            files.append(bytes(b))
    files.append(bases[0][:len(bases[0]) - 40] + b"\xff\xd9")          # cut inside its last scan
    px, st = device_decode(files)
    bad = 0
    for b, p, s in zip(files, px, st):
        hs, hp, _ = jp.decode(emu, b)
        assert s == hs
        bad += s != 0
        if s == 0:
            assert np.array_equal(p, hp)
    assert bad > 0


def _mixed_files():
    a = content("photo", 120, 152, 5)
    return [encode(a, quality=90), jp.encode(a, progressive=True, quality=90, subsampling=2),
            encode(content("photo", 200, 260, 6), quality=90, restart_marker_blocks=3),
            jp.encode(content("noise", 75, 93, 7), progressive=True, quality=75, subsampling=1, restart_marker_rows=1),
            encode(content("photo", 375, 500, 8), quality=90),
            jp.encode(content("photo", 64, 64, 9), gray=True, progressive=True, quality=60)]


@pytest.mark.parametrize("index", [False, True])
def test_mixed_batches_equal_each_file_alone(index):
    files = _mixed_files()
    px, st = device_decode(files, index=index)
    for i, b in enumerate(files):
        p1, s1 = device_decode([b], index=index)
        assert st[i] == s1[0] == 0
        assert np.array_equal(px[i], p1[0]) and np.array_equal(px[i], jp.pillow(b))


def test_mixed_record_and_index_give_progressive_files_nothing():
    files = _mixed_files()
    enc = EncodedImages.from_bytes(files, progressive=True)
    first, points = build_jpeg_index(enc)
    counts = np.diff(first)
    assert (counts[enc.progressive()] == 0).all() and counts[4] > 0
    out, st, count, pts, cap_first = decode_jpeg(enc, record=True)
    count = count.cpu().numpy()
    assert (count[enc.progressive()] == 0).all() and count[4] > 0
    assert (np.diff(cap_first)[enc.progressive()] == 0).all()
    assert (st.cpu().numpy() == 0).all()
    for i, b in enumerate(files):
        assert np.array_equal(out.image(i).cpu().numpy(), jp.pillow(b))


def test_second_stream_grows_every_buffer_while_first_is_queued():
    small = EncodedImages.from_bytes([jp.encode(content("photo", 40, 40, 1), progressive=True, quality=80)],
                                     progressive=True)
    large_files = [jp.encode(content("photo", 1536, 2048, 2), progressive=True, quality=90, subsampling=2,
                             restart_marker_blocks=1)]
    large = EncodedImages.from_bytes(large_files, progressive=True)
    out_s, st_s = decode_jpeg(small)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out_l, st_l = decode_jpeg(large)
    torch.cuda.synchronize()
    assert st_s.item() == 0 and st_l.item() == 0
    assert np.array_equal(out_l.image(0).cpu().numpy(), jp.pillow(large_files[0]))


@pytest.mark.parametrize("chunk", [0, 1])
def test_hand_built_streams_equal_host_build_and_pillow(emu, chunk):
    import jpeg_progressive_streams as ps
    cases = ps.cases()[chunk::2]
    files = [c[1] for c in cases]
    px, st = device_decode(files)
    for b, p, s in zip(files, px, st):
        hs, hp, _ = jp.decode(emu, b)
        assert s == hs == 0
        assert np.array_equal(p, hp) and np.array_equal(p, jp.pillow(b))


def test_loaders_decode_progressive_files_on_the_device(tmp_path, monkeypatch):
    """the key on: the same train / valid / test / tta batches as with it off, the progressive file decoded on the
    device (not by Pillow), and with ``faa_jpeg_index_learn`` no point learned for it"""
    from imagenet_tree import write_tree
    from test_gpu_imagenet_folder import B, assert_same, conf_set, run

    from fast_autoaugment_b200 import data

    root = str(tmp_path / "data")
    write_tree(root, 23, n_classes=3, per_class=10, n_val=6)          # a progressive, a CMYK and a PNG-named file
    pillowed = []
    real = data._pillow_rgb

    def spy(pb):
        pillowed.append(pb[0].rsplit("/", 1)[1])
        return real(pb)
    monkeypatch.setattr(data, "_pillow_rgb", spy)
    loaders = {}
    for key in (False, True):
        with conf_set(faa_jpeg_progressive=key, faa_jpeg_index_learn=key):
            torch.manual_seed(0)
            loaders[key] = data.get_dataloaders("imagenet", B, root, split=0.2)
    on, off = set(), set()
    for which in (1, 2, 3):
        pillowed.clear()
        got = run(loaders[True][which], 70 + which)
        on |= set(pillowed)
        pillowed.clear()
        want = run(loaders[False][which], 70 + which)
        off |= set(pillowed)
        assert_same(got, want, which)
    assert "progressive.JPEG" in off and "progressive.JPEG" not in on
    assert on == off - {"progressive.JPEG"} and "cmyk.JPEG" in on
    assert any(p.endswith("progressive.JPEG") for p in loaders[True][1].dataset.paths)
    for key in (False, True):
        torch.manual_seed(5)
        out = [(x.cpu(), y.cpu()) for x, y in loaders[key][2].tta(2)]
        loaders[key] = loaders[key] + (out,)
    assert_same(loaders[True][4], loaders[False][4], "tta")
    idx = loaders[True][1].dataset.index
    assert len(idx._added) > 0 and not any(r.endswith("progressive.JPEG") for r in idx._added)
