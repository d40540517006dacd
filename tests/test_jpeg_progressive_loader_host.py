"""The loaders' host half with and without ``progressive``: ``read_jpeg_batch`` sends progressive files to Pillow
without it, and with it accepts them with their scans (offsets into the accepted files' scans, parsed as
``parse_jpeg_headers`` parses them alone); ``_Layout`` of a batch without progressive files is the same with the
option on and off, and with them it carries the scans after everything else."""
import numpy as np

import jpeg_progressive_cases as jp
from imagenet_tree import baseline_file, refused_files, write

from fast_autoaugment_b200 import data
from fast_autoaugment_b200.engine import parse_jpeg_headers


def _tree(tmp_path):
    files = {"a.JPEG": baseline_file(0, 3), "b.JPEG": baseline_file(1, 3), **refused_files(3),
             "c.JPEG": jp.encode(jp.content("photo", 50, 70, 1), progressive=True, quality=90, subsampling=1)}
    paths = []
    for name, b in files.items():
        write(str(tmp_path / name), b)
        paths.append(str(tmp_path / name))
    return paths, files


def test_read_batch_with_and_without_progressive(tmp_path):
    paths, files = _tree(tmp_path)
    names = [p.rsplit("/", 1)[1] for p in paths]
    off = data.read_jpeg_batch(paths)
    on = data.read_jpeg_batch(paths, progressive=True)
    prog = [i for i, n in enumerate(names) if n in ("progressive.JPEG", "c.JPEG")]
    assert set(prog) <= set(off.refused.tolist()) and off.scans is None
    assert not set(prog) & set(on.refused.tolist())
    assert set(on.refused.tolist()) == set(off.refused.tolist()) - set(prog)
    assert np.array_equal(on.sizes(), off.sizes())
    acc = on.accepted.tolist()
    assert len(on.scan_first) == len(acc) + 1 and on.scan_first[-1] == len(on.scans)
    for k, i in enumerate(acc):
        n = int(on.scan_first[k + 1] - on.scan_first[k])
        if i in prog:
            _, _, _, sc, _ = parse_jpeg_headers([files[names[i]]], progressive=True)
            got = on.scans[on.scan_first[k]:on.scan_first[k + 1]]
            for f in ("off", "len", "restart", "ns", "comp", "ss", "se", "ah", "al", "wave"):
                assert np.array_equal(got[f], sc[f]), f
            assert on.headers["reserved"][k] == 1
        else:
            assert n == 0 and on.headers["reserved"][k] == 0
    assert np.array_equal(on.headers["offset"], np.cumsum([len(f) for f in on.files]) - [len(f) for f in on.files])


def test_layout_unchanged_without_progressive_files(tmp_path):
    paths, _ = _tree(tmp_path)
    base = [p for p in paths if p.endswith(("a.JPEG", "b.JPEG", "cmyk.JPEG"))]
    off, on = data.read_jpeg_batch(base), data.read_jpeg_batch(base, progressive=True)
    assert on.scans is None and on.scan_first is None
    lo, ln = data._Layout(off), data._Layout(on)
    assert vars(lo) == vars(ln)
    bo, bn = np.zeros(lo.total, np.uint8), np.zeros(ln.total, np.uint8)
    lo.pack(off, bo)
    ln.pack(on, bn)
    assert np.array_equal(bo, bn)


def test_layout_carries_the_scans(tmp_path):
    paths, _ = _tree(tmp_path)
    hb = data.read_jpeg_batch(paths, progressive=True)
    lay = data._Layout(hb)
    assert lay.scan_first >= (lay.pixels[-1] if lay.pixels else lay.files_end) and lay.scan_first % 16 == 0
    assert lay.scans % 16 == 0 and lay.total >= lay.scans_end
    buf = np.zeros(lay.total, np.uint8)
    lay.pack(hb, buf)
    assert np.array_equal(buf[lay.scan_first:lay.scans].view(np.int64)[:len(hb.scan_first)], hb.scan_first)
    assert buf[lay.scans:lay.scans_end].tobytes() == hb.scans.tobytes()
    assert buf[lay.files:lay.files_end].tobytes() == b"".join(hb.files)
