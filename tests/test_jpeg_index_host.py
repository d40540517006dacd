"""The JPEG scan index without a GPU: the host build of the recording decode and of the indexed decode
(tests/emu/faa_emu_jpeg_index.cpp, the same faa_jpeg.cuh the kernels run) on every file of the decoder grid and on the
restart-free hand-built streams.  The points follow the placement rule and equal the serial decoder's state at their
MCU; the indexed decode equals the serial decode and Pillow; any broken index gives the serial result without touching
a byte outside its buffers.  Also the index files (``data.JpegIndex``) and how a batch's points are staged."""
import functools
import os

import numpy as np
import pytest

import jpeg_index_cases as jic
from imagenet_tree import write_tree
from jpeg_cases import GRID, emu_decode, encode, content, load_emu_jpeg, make, pillow
from test_jpeg_host import MUTATIONS

from fast_autoaugment_b200 import _lib, data
from fast_autoaugment_b200.engine import parse_jpeg

SYNC = jic.SYNC


@pytest.fixture(scope="module")
def emu():
    return jic.load_emu_index()


@pytest.fixture(scope="module")
def emu_jpeg():
    return load_emu_jpeg()


def header(b):
    hdr, _ = parse_jpeg(b)
    assert hdr is not None
    return hdr[0]


def check_file(emu, b, want=None):
    """placement rule, points == serial states, indexed decode == Pillow.  A file the rule gives no points decodes
    through the serial path itself (test_jpeg_host holds that to Pillow): only its empty index is checked."""
    h = header(b)
    mcus = int(h["mcu_x"]) * int(h["mcu_y"])
    pts, st, (_, scan_len) = jic.host_index(emu, b)
    assert st == 0
    assert scan_len == int(h["scan_len"])
    parts = jic.parts(scan_len, int(h["restart"]))
    assert _lib.lib.faa_jpeg_index_capacity(h.tobytes()) == max(parts - 1, 0)
    if parts == 0:
        assert len(pts) == 0
        return pts
    states = jic.host_states(emu, b, mcus)
    assert len(states) == mcus
    assert pts.tobytes() == jic.rule_points(states, scan_len, 0).tobytes()
    if len(pts):
        assert (np.diff(pts["mcu"]) > 0).all() and pts["mcu"][0] > 0 and pts["mcu"][-1] < mcus
        assert jic.linked(emu, b, pts) == 1
        st1, got = jic.decode_indexed(emu, b, pts)
        assert st1 == 0 and np.array_equal(got, pillow(b) if want is None else want)
    return pts


@functools.lru_cache(maxsize=8)
def _content(kind, h, w):
    return content(kind, h, w, h * 7 + w)


def grid_bytes(case):
    """the file of a GRID case, as make(case) writes it (without Pillow's decode; the pixels of one size and content
    are made once for all its settings, GRID being ordered by size)"""
    _, h, w, kind, opts = case
    opts = dict(opts)
    gray = opts.pop("gray", False)
    return encode(_content(kind, h, w), gray=gray, **opts)


GRID_CHUNKS = [GRID[k:k + 32] for k in range(0, len(GRID), 32)]


@pytest.mark.parametrize("k", range(len(GRID_CHUNKS)), ids=lambda k: GRID_CHUNKS[k][0][0])
def test_grid_index_follows_the_rule_and_decodes_as_pillow(emu, k):
    """every GRID case; Pillow's decode is compared where the file has points (without them the indexed decode is the
    serial one, which test_jpeg_host holds to Pillow)"""
    for case in GRID_CHUNKS[k]:
        b = grid_bytes(case)
        h = header(b)
        pts = check_file(emu, b)
        assert (len(pts) > 0) == (int(h["restart"]) == 0 and int(h["scan_len"]) >= 2048), case[0]
    assert grid_bytes(GRID_CHUNKS[k][0]) == make(GRID_CHUNKS[k][0])[0]


STREAMS = jic.stream_cases()


@pytest.mark.parametrize("k", range(0, len(STREAMS), 16), ids=lambda k: STREAMS[k][0])
def test_streams_index_follows_the_rule_and_decodes_as_pillow(emu, k):
    for name, b in STREAMS[k:k + 16]:
        check_file(emu, b)


def test_large_scan_gets_127_points(emu):
    b = jic.big_file()
    assert int(header(b)["scan_len"]) >= 128 * 1024
    pts = check_file(emu, b)
    assert len(pts) == 127


def test_restart_files_and_short_scans_get_no_points(emu, emu_jpeg):
    a = content("photo", 375, 500, 1)
    for opts in ({"restart_marker_blocks": 4}, {"restart_marker_rows": 1}):
        b = encode(a, quality=90, **opts)
        assert int(header(b)["scan_len"]) > 4096 and int(header(b)["restart"]) > 0
        assert len(jic.host_index(emu, b)[0]) == 0
        # the points of the same image without markers are ignored: the decode is the serial one
        pts = jic.host_index(emu, encode(a, quality=90))[0]
        assert len(pts) > 0 and jic.linked(emu, b, pts) == 0
        st, got = jic.decode_indexed(emu, b, pts)
        assert st == 0 and np.array_equal(got, pillow(b))
    flat = encode(np.full((64, 64, 3), 100, np.uint8), quality=75)
    assert int(header(flat)["scan_len"]) < 2048 and len(jic.host_index(emu, flat)[0]) == 0
    # just under and at 2 KiB of scan
    for b in (encode(content("noise", 24, 40, s), quality=q) for s in range(3) for q in (60, 80, 95)):
        n = len(jic.host_index(emu, b)[0])
        assert (n > 0) == (int(header(b)["scan_len"]) >= 2048)


def test_capacity_limits_the_points(emu):
    b = jic.indexed_files()[0][1]
    full = jic.host_index(emu, b)[0]
    assert len(full) > 4
    assert jic.host_index(emu, b, cap=3)[0].tobytes() == full[:3].tobytes()
    assert len(jic.host_index(emu, b, cap=0)[0]) == 0


FILES = jic.indexed_files()


@pytest.mark.parametrize("k", range(len(FILES)), ids=[f[0] for f in FILES])
def test_fuzzed_indexes_give_the_serial_decode(emu, emu_jpeg, k):
    name, b = FILES[k]
    h = header(b)
    mcus = int(h["mcu_x"]) * int(h["mcu_y"])
    pts, _, scan = jic.host_index(emu, b)
    assert len(pts) >= 3, name
    other = jic.host_index(emu, FILES[(k + 1) % len(FILES)][1])[0]
    e, st0, serial = emu_decode(emu_jpeg, b)
    assert e == 0 and st0 == 0
    cases = jic.fuzzed(pts, other, scan, mcus, b, jic.host_states(emu, b, mcus))
    assert any(n == "on-stuffed-zero" for n, _ in cases)
    for what, q in cases:
        st, got = jic.decode_indexed(emu, b, q)
        assert st == st0 and np.array_equal(got, serial), (name, what)
    # a byte, bit or predictor off by one always breaks the chain (grayscale has no predictors 1 and 2 to break)
    for what, q in cases:
        if what.startswith(("byte", "bit", "pred")) and "@" in what and not (what.startswith("pred") and
                                                                           int(h["ncomp"]) == 1 and what[4] != "0"):
            assert jic.linked(emu, b, q) == 0, (name, what)


def _mutated(b, seed):
    """corruptions of a restart-free file in the manner of test_jpeg_host._mutations: cuts, bit flips, a bad code"""
    h = header(b)
    s0, n = int(h["scan_off"]), int(h["scan_len"])
    rng = np.random.default_rng(seed)
    out = [("trunc-%g" % f, b[:s0 + int(n * f)]) for f in (0.1, 0.5, 0.9, 0.99)]
    for j in range(8):
        m = bytearray(b)
        m[s0 + int(rng.integers(0, n))] ^= 1 << int(rng.integers(0, 8))
        out.append(("flip-%d" % j, bytes(m)))
    m = bytearray(b)
    m[s0 + n // 3:s0 + n // 3 + 8] = b"\xff\x00" * 4
    out.append(("badcode", bytes(m)))
    return out


def test_corrupt_streams_with_the_intact_index_give_the_serial_decode(emu, emu_jpeg):
    # test_jpeg_host's corruptions (their files are small: mostly no index), then the same kinds on indexed files
    intact, cases = {}, []
    for k, (h_, w_, sub, extra) in enumerate([(64, 80, 2, {}), (48, 48, 0, {"restart_marker_blocks": 2}),
                                              (40, 72, 1, {"restart_marker_rows": 1}), (33, 17, 2, {})]):
        intact[k] = encode(content("photo", h_, w_, k), quality=85, subsampling=sub, **extra)
    for name, b, _ in MUTATIONS:
        k = int(name.split("-")[0][-1])
        cases.append((name, b, intact[k]))
    for fname, b in FILES:
        cases += [(fname + "-" + n, m, b) for n, m in _mutated(b, len(b))]
    flagged = 0
    for name, bad, good in cases:
        pts = jic.host_index(emu, good)[0]
        e, st0, serial = emu_decode(emu_jpeg, bad)
        assert e == 0, name
        st, got = jic.decode_indexed(emu, bad, pts)
        assert st == st0 and np.array_equal(got, serial), name
        flagged += st0 != 0
    assert flagged > 10


# ---- index files and staging
def _tree_index(emu, root):
    """a JpegIndex of the train split of a tree, from the host build"""
    folder = data.imagenet_split_folder(root, "train")
    paths = [p for p, _ in data.imagenet_index(root, "train")]
    rel, sizes, first, pts = [], [], [0], []
    for p in paths:
        b = open(p, "rb").read()
        q = jic.host_index(emu, b)[0] if parse_jpeg(b)[0] is not None else np.zeros(0, SYNC)
        rel.append(os.path.relpath(p, folder))
        sizes.append(len(b))
        first.append(first[-1] + len(q))
        pts.append(q)
    return paths, data.JpegIndex(folder, rel, sizes, first, np.concatenate(pts))


def test_index_file_round_trip_and_lookup(emu, tmp_path):
    write_tree(tmp_path, 21, n_classes=2, per_class=3, n_val=1, refused=False)
    paths, idx = _tree_index(emu, str(tmp_path))
    assert len(idx.points) > 0
    out = os.path.join(str(tmp_path), "idx", "train.npz")
    os.makedirs(os.path.dirname(out))
    idx.save(out)
    back = data.JpegIndex.load(out, idx.folder)
    assert back.points.tobytes() == idx.points.tobytes() and np.array_equal(back.first, idx.first)
    for p in paths:
        n = os.path.getsize(p)
        assert back.lookup(p, n).tobytes() == idx.lookup(p, n).tobytes()
    some = next(p for p in paths if len(idx.lookup(p, os.path.getsize(p))))
    assert len(back.lookup(some, os.path.getsize(some) + 1)) == 0                    # length differs: no points
    assert len(back.lookup(os.path.join(idx.folder, "n99", "absent.JPEG"), 10)) == 0   # not listed: no points
    z = dict(np.load(out))
    z["version"] = np.int64(99)
    np.savez(out, **z)
    with pytest.raises(ValueError, match="version"):
        data.JpegIndex.load(out, idx.folder)


def test_staged_points_land_at_their_offsets(emu, tmp_path):
    write_tree(tmp_path, 22, n_classes=2, per_class=4, n_val=1)
    paths, idx = _tree_index(emu, str(tmp_path))
    rng = np.random.default_rng(1)
    batch = [paths[int(i)] for i in rng.permutation(len(paths))]
    stale = batch[2]                                               # rewritten after indexing: another length
    b = open(stale, "rb").read()
    open(stale, "wb").write(b + b"\x00" * 7)
    hb = data.read_jpeg_batch(batch, index=idx)
    plain = data.read_jpeg_batch(batch)
    assert hb.headers.tobytes() == plain.headers.tobytes() and plain.first is None
    accepted = [batch[i] for i in hb.accepted]
    assert len(hb.first) == len(accepted) + 1 and hb.first[0] == 0
    for k, p in enumerate(accepted):
        want = idx.lookup(p, os.path.getsize(p))
        assert hb.points[hb.first[k]:hb.first[k + 1]].tobytes() == want.tobytes()
        if p == stale:
            assert hb.first[k + 1] == hb.first[k]
    assert int(hb.first[-1]) > 0
    lay = data._Layout(hb)
    lay0 = data._Layout(plain)
    assert (lay.pool, lay.files, lay.files_end, lay.pixels) == (lay0.pool, lay0.files, lay0.files_end, lay0.pixels)
    assert lay.first % 16 == 0 and lay.points % 16 == 0 and lay.first >= (lay0.pixels or [lay0.files_end])[-1]
    buf = np.full(lay.total, 0xA5, np.uint8)
    lay.pack(hb, buf)
    assert buf[lay.first:lay.first + hb.first.nbytes].view(np.int64).tolist() == hb.first.tolist()
    assert buf[lay.points:lay.points_end].tobytes() == hb.points.tobytes()
    assert lay.points_end <= lay.total
