"""The scan index of progressive JPEG files on the device (``EncodedImages.from_bytes(..., progressive=True,
progressive_index=True)``, C ABI ``faa_jpeg_decode`` with reserved-3 headers): a recording decode places the host
build's points byte for byte; a decode from them, or from a fuzzed or stale index, gives the pixels and status of the
plain decode and Pillow's; batches mixing scan-indexed progressive files with reserved-1 progressive, baseline indexed,
baseline found and restart-interval files give every file its result alone with the launches they made before; a call
on a second stream grows every buffer while the first is queued; and the loaders with
``conf['faa_jpeg_progressive_index']`` yield the batches they yield without it while learning progressive points."""
import numpy as np
import pytest
import torch

import jpeg_progressive_cases as jp
from jpeg_cases import content, encode
from test_gpu_jpeg import launches, sentinel_out, untouched_outside
from test_jpeg_progressive_index_host import FILES, STREAMS, decode as host_decode, load_emu, rule

from fast_autoaugment_b200 import _lib
from fast_autoaugment_b200.engine import EncodedImages, build_jpeg_index, compact_jpeg_index, decode_jpeg

pytestmark = pytest.mark.gpu

SYNC = _lib.JPEG_SYNC_DTYPE


@pytest.fixture(scope="module")
def emu():
    return load_emu()


def run(enc, **kw):
    out = sentinel_out(enc.sizes)
    r = decode_jpeg(enc, out, **kw)
    torch.cuda.synchronize()
    assert untouched_outside(out)
    px = [out.image(i).cpu().numpy() for i in range(len(enc))]
    if kw.get("record"):
        _, st, count, pts, cap = r
        first, points = compact_jpeg_index(cap, count.cpu().numpy(), pts.cpu().numpy())
        return px, st.cpu().numpy(), (first, points)
    return px, r[1].cpu().numpy(), None


def _chunks(items, n):
    return [items[i:i + n] for i in range(0, len(items), n)]


@pytest.mark.parametrize("chunk", range(4))
def test_device_recording_equals_host_build_and_indexed_decode_the_plain_one(emu, chunk):
    files = [f[1] for f in FILES[chunk::4]]
    plain = EncodedImages.from_bytes(files, progressive=True)
    enc = EncodedImages.from_bytes(files, progressive=True, progressive_index=True)
    px0, st0, _ = run(plain)
    px, st, (first, points) = run(enc, record=True)
    assert (st == 0).all() and (st0 == 0).all()
    for i, b in enumerate(files):
        want = rule(emu, b)
        assert points[first[i]:first[i + 1]].tobytes() == want.tobytes(), i
        assert np.array_equal(px[i], px0[i]) and np.array_equal(px[i], jp.pillow(b))
    assert np.array_equal(build_jpeg_index(enc)[0], first)
    px2, st2, (f2, _) = run(enc.with_index(first, points), record=True)
    assert (st2 == 0).all() and (np.diff(f2) == 0).all()             # used as they stand: nothing recorded
    for i in range(len(files)):
        assert np.array_equal(px2[i], px0[i])


def test_fuzzed_and_stale_indexes_give_the_plain_pixels_and_status(emu):
    b = [f[1] for f in FILES if f[0] == "p375x500_2_q90"][0]
    pts = rule(emu, b)
    rng = np.random.default_rng(3)
    variants = []
    for f in ("mcu", "byte", "bit"):
        q = pts.copy()
        q[f][len(q) // 2] += 1
        variants.append(q)
    q = pts.copy()
    q["pred"][1, 0] += 1
    variants += [q, rng.permutation(pts), pts[:-1], np.concatenate([pts[:2], pts[1:]]), rule(emu, STREAMS[1][1])]
    files = [b] * len(variants)
    # a corrupt copy of the file with the intact file's points
    bad = bytearray(b)
    _, _, h, scans = jp.parse(jp.load_emu(), b)
    at = int(scans[2]["off"] + scans[2]["len"] // 3)
    bad[at] ^= 0x5A
    files.append(bytes(bad))
    variants.append(pts)
    first = np.concatenate([[0], np.cumsum([len(v) for v in variants])]).astype(np.int64)
    enc = EncodedImages.from_bytes(files, progressive=True, progressive_index=True)
    px, st, _ = run(enc.with_index(first, np.concatenate(variants)))
    px0, st0, _ = run(EncodedImages.from_bytes(files, progressive=True))
    for i, b in enumerate(files):
        hs, hp, _, _ = host_decode(emu, b, indexed=0)
        assert st[i] == st0[i] == hs, i
        assert np.array_equal(px[i], px0[i]) and np.array_equal(px[i], hp), i


def _mixed():
    """scan-indexed progressive, reserved-1 progressive, baseline (indexed / found), baseline with restarts"""
    big = content("photo", 375, 500, 8)
    files = [jp.encode(big, progressive=True, quality=90, subsampling=2),
             jp.encode(content("photo", 300, 420, 3), progressive=True, quality=75, subsampling=0),
             encode(big, quality=90),
             encode(content("photo", 200, 260, 6), quality=90, restart_marker_blocks=3),
             jp.encode(content("noise", 160, 200, 7), progressive=True, quality=90, subsampling=1),
             encode(content("photo", 320, 400, 4), quality=85)]
    enc = EncodedImages.from_bytes(files, progressive=True, progressive_index=True)
    h = enc.headers.copy()
    h["reserved"][1], h["scan_len"][1] = _lib.JPEG_PROGRESSIVE, 0                       # file 1 takes no index
    enc = EncodedImages(enc.storage, h, enc.pool, scans=enc.scans, scan_first=enc.scan_first)
    return files, enc


@pytest.mark.parametrize("mode", ["plain", "indexed", "record", "indexed_record", "find"])
def test_mixed_batches_give_every_file_its_result_alone(mode):
    files, enc = _mixed()
    first, points = build_jpeg_index(enc)
    counts = np.diff(first)
    assert counts[0] > 0 and counts[4] > 0 and counts[2] > 0 and counts[1] == 0 and counts[3] == 0
    if mode.startswith("indexed"):
        enc = enc.with_index(first, points)
    kw = {"record": mode.endswith("record") or mode == "find", "find": mode == "find"}
    n0 = launches()
    px, st, rec = run(enc, **kw)
    assert launches() - n0 == (4 if mode == "find" else 3)             # (find,) entropy, progressive, reconstruct
    assert (st == 0).all()
    for i, b in enumerate(files):
        assert np.array_equal(px[i], jp.pillow(b)), i
        one = enc.select([i])
        p1, s1, r1 = run(one, **kw)
        assert s1[0] == st[i] and np.array_equal(p1[0], px[i]), i
        if rec is not None:
            assert rec[1][rec[0][i]:rec[0][i + 1]].tobytes() == r1[1].tobytes(), i
    if rec is not None:
        got = np.diff(rec[0])
        assert got[1] == 0 and got[3] == 0
        if mode == "record":
            assert rec[1].tobytes() == points.tobytes()                 # every file recorded, as the index build
        elif mode == "indexed_record":
            assert got[0] == 0 and got[4] == 0                          # progressive points used as they stood
        else:                                                           # find: progressive files recorded serially
            for i in (0, 4):
                assert rec[1][rec[0][i]:rec[0][i + 1]].tobytes() == points[first[i]:first[i + 1]].tobytes()


def test_build_jpeg_index_with_find_gives_progressive_files_nothing():
    _, enc = _mixed()
    first, _ = build_jpeg_index(enc, find=True)
    counts = np.diff(first)
    assert counts[0] == counts[1] == counts[4] == 0 and counts[2] > 0


def test_second_stream_grows_every_buffer_while_first_is_queued():
    small = EncodedImages.from_bytes([jp.encode(content("photo", 40, 40, 1), progressive=True, quality=80)],
                                     progressive=True, progressive_index=True)
    large_files = [jp.encode(content("photo", 1536, 2048, 2), progressive=True, quality=90, subsampling=2)]
    large = EncodedImages.from_bytes(large_files, progressive=True, progressive_index=True)
    large = large.with_index(*build_jpeg_index(large))
    assert len(large.points) > 0
    out_s, st_s = decode_jpeg(small)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out_l, st_l, count, _, _ = decode_jpeg(large, record=True)
    torch.cuda.synchronize()
    assert st_s.item() == 0 and st_l.item() == 0 and count.item() == 0
    assert np.array_equal(out_l.image(0).cpu().numpy(), jp.pillow(large_files[0]))


def test_loaders_learn_progressive_points_with_the_same_batches(tmp_path, monkeypatch):
    """``faa_jpeg_progressive`` + ``faa_jpeg_index_learn``, with and without ``faa_jpeg_progressive_index``: epochs 1
    and 2 yield the same batches bit for bit; with the key the progressive files are learned in epoch 1 with the
    command's points and, in epoch 2, decoded from them and not entered again; ``tta`` batches are unchanged"""
    import os

    from imagenet_tree import write, write_tree
    from test_gpu_imagenet_folder import B, assert_same, conf_set
    from test_gpu_imagenet_folder import run as run_loader

    from fast_autoaugment_b200 import data, jpeg_index

    root = str(tmp_path / "data")
    base = write_tree(root, 29, n_classes=3, per_class=10, n_val=6)
    big = {}
    for k, (split, c) in enumerate((("train", 1), ("train", 2), ("val", 0))):
        p = os.path.join(base, split, "n%08d" % (1000 + 7 * c), "big_progressive_%d.JPEG" % k)
        big[p] = jp.encode(content("photo", 300 + 20 * k, 420, 40 + k), progressive=True, quality=90,
                           subsampling=2 * (k % 2))
        write(p, big[p])
    added = []
    real_add = data.JpegIndex.add

    def spy(self, paths, *a):
        added.append([os.path.basename(p) for p in paths])
        return real_add(self, paths, *a)
    monkeypatch.setattr(data.JpegIndex, "add", spy)
    loaders, learned = {}, {}
    for key in (False, True):
        with conf_set(faa_jpeg_progressive=True, faa_jpeg_index_learn=True, faa_jpeg_progressive_index=key):
            torch.manual_seed(0)
            loaders[key] = data.get_dataloaders("imagenet", B, root, split=0.2)
        for epoch in (1, 2):
            added.clear()
            got = run_loader(loaders[key][1], 90 + epoch), run_loader(loaders[key][2], 80 + epoch)
            loaders[key] = loaders[key] + (got,)
            learned[key, epoch] = {n for batch in added for n in batch}
    for epoch in (1, 2):
        for which in (0, 1):
            assert_same(loaders[True][3 + epoch][which], loaders[False][3 + epoch][which], (epoch, which))
    train_big = {os.path.basename(p) for p in big if "/train/" in p}
    assert not any(n.startswith("big_progressive") for e in (1, 2) for n in learned[False, e])
    assert any(n in learned[True, 1] for n in train_big)
    assert not any(n.startswith("big_progressive") for n in learned[True, 2])      # decoded from the points
    idx = loaders[True][1].dataset.index
    want = jpeg_index.index_files(list(big), os.path.join(base, "train"), progressive=True)
    for p in big:
        q = idx.lookup(p, len(big[p]))
        if len(q):
            assert q.tobytes() == want.lookup(p, len(big[p])).tobytes()
    assert sum(len(idx.lookup(p, len(big[p]))) > 0 for p in big) >= 1
    for key in (False, True):
        torch.manual_seed(5)
        loaders[key] = loaders[key] + ([(x.cpu(), y.cpu()) for x, y in loaders[key][2].tta(2)],)
    assert_same(loaders[True][-1], loaders[False][-1], "tta")
