"""faa_jpeg_decode's argument checks on a machine without a GPU.  Every refusal comes before the call looks for a
device, so the device pointers here are dummies the host never reads, and a call that passes every check returns
FAA_ERR_NO_DEVICE."""
import itertools

import numpy as np
import pytest
import torch

import jpeg_progressive_cases as jp
from jpeg_cases import content, encode

from fast_autoaugment_b200 import _lib, engine

DEV = 0x1000                                   # a dummy device pointer


def _batch(kinds="bb"):
    """(headers, n_tables, h_out, scans, scan_first) of 96 x 128 files, "b" baseline and "p" progressive"""
    a = content("photo", 96, 128, 2)
    files = [jp.encode(a, progressive=True, quality=95) if k == "p" else encode(a, quality=95) for k in kinds]
    headers, pool, _, scans, scan_first = engine.parse_jpeg_headers(files, progressive=True)
    out = np.zeros(len(kinds), dtype=_lib.IMAGE_DTYPE)
    out["data"], out["h"], out["w"] = DEV, 96, 128
    return headers, len(pool), out, scans, scan_first


@pytest.mark.skipif(torch.cuda.is_available(), reason="a call that passes its checks would launch on the dummy pointers")
def test_index_and_recording_refusals_come_before_the_device():
    dec = engine._JpegDecoder()
    headers, n_tables, h_out = _batch()[:3]
    first = np.array([0, 8, 16], np.int64)
    empty = np.zeros(3, np.int64)

    def call(index=(None,) * 3, rec=(None,) * 4, find=0, batch=2, headers=headers):
        return _lib.lib.faa_jpeg_decode(dec.handle, headers.ctypes.data, DEV, DEV, n_tables, DEV, batch,
                                        h_out.ctypes.data, DEV, DEV, *index, *rec, *(None,) * 4, find, None)

    def index(f=first, d_points=DEV):                  # (d_points, h_first, d_first)
        return (d_points, f.ctypes.data, DEV)

    def rec(f=first, d_points_out=DEV):                # (h_cap_first, d_cap_first, d_points_out, d_count)
        return (f.ctypes.data, DEV, d_points_out, DEV)

    # well-formed: no group, either group, both, find; a points array may be null where the offsets give no point
    for kw in ({}, {"index": index()}, {"rec": rec()}, {"index": index(), "rec": rec()}, {"rec": rec(), "find": 1},
               {"index": index(), "rec": rec(), "find": 1}, {"index": index(empty, None)},
               {"rec": rec(empty, None), "find": 1}):
        assert call(**kw) == _lib.ERR_NO_DEVICE, kw
    assert call(batch=0) == _lib.ERR_NO_DEVICE
    # a group given in part
    for group, full in (("index", index()), ("rec", rec())):
        for keep in itertools.product((False, True), repeat=len(full)):
            if any(keep) and not all(keep):
                assert call(**{group: tuple(p if k else None for p, k in zip(full, keep))}) == _lib.ERR_VALUE, keep
    # find without the recording outputs
    assert call(find=1) == _lib.ERR_VALUE
    assert call(index=index(), find=1) == _lib.ERR_VALUE
    # offsets that are out of order or negative, in either array
    for bad in ([1, 0, 2], [-1, 0, 0], [0, 2, 1]):
        f = np.array(bad, np.int64)
        assert call(index=index(f)) == _lib.ERR_VALUE
        assert call(rec=rec(f)) == _lib.ERR_VALUE
        assert call(rec=rec(f), find=1) == _lib.ERR_VALUE
    # a progressive header without the scans group
    assert call(headers=_batch("pp")[0]) == _lib.ERR_VALUE
    assert b"progressive" in _lib.lib.faa_last_error()
    # batch bounds
    assert call(batch=-1) == _lib.ERR_VALUE
    assert call(batch=65536) == _lib.ERR_UNSUPPORTED


@pytest.mark.skipif(torch.cuda.is_available(), reason="a call that passes its checks would launch on the dummy pointers")
def test_scans_group_refusals_come_before_the_device():
    dec = engine._JpegDecoder()

    def call(kinds, scans=None, first=None, headers=None, group=None, rec=(None,) * 4, find=0):
        hdr, n_tables, h_out, s, f = _batch(kinds)
        hdr = hdr if headers is None else headers
        s = s if scans is None else scans
        f = np.asarray(f if first is None else first, np.int64)
        if group is None:
            group = (s.ctypes.data, DEV, f.ctypes.data, DEV)
        return _lib.lib.faa_jpeg_decode(dec.handle, hdr.ctypes.data, DEV, DEV, n_tables, DEV, len(kinds),
                                        h_out.ctypes.data, DEV, DEV, None, None, None, *rec, *group, find, None)

    def refused(why, *a, **kw):
        assert call(*a, **kw) == _lib.ERR_VALUE, why
        assert why.encode() in _lib.lib.faa_last_error(), _lib.lib.faa_last_error()

    hdr, _, _, scans, first = _batch("bp")
    n = int(first[-1])
    assert 1 < n <= 64 and list(first) == [0, 0, n]
    cap = np.zeros(3, np.int64)
    # well-formed: all progressive, mixed either way round, mixed with the recording outputs and find
    for kinds in ("pp", "bp", "pb"):
        assert call(kinds) == _lib.ERR_NO_DEVICE, kinds
    assert call("bp", rec=(cap.ctypes.data, DEV, None, DEV), find=1) == _lib.ERR_NO_DEVICE
    # a group given in part
    full = (scans.ctypes.data, DEV, first.ctypes.data, DEV)
    for keep in itertools.product((False, True), repeat=4):
        if any(keep) and not all(keep):
            refused("null argument", "bp", group=tuple(p if k else None for p, k in zip(full, keep)))
    # a baseline image that owns scans
    refused("a baseline image owns no scans", "bp", scans=np.concatenate([scans[:1], scans]), first=[0, 1, n + 1])
    # 0 and 65 scans
    refused("1 to 64 scans", "pp", first=[0, 0, n])
    many = np.resize(scans, 65 + n)
    refused("1 to 64 scans", "pp", scans=many, first=[0, 65, 65 + n])
    # scan offsets out of order
    refused("point offsets", "pp", first=[0, 2 * n, n])
    # a wrong wave, a scan past the file, a scan's pool slot out of range
    s = scans.copy()
    s["wave"][n - 1] += 1
    refused("wave", "bp", scans=s)
    s = scans.copy()
    s["off"][0] = hdr["len"][1]
    refused("byte range", "bp", scans=s)
    s = scans.copy()
    s["pool"][0, 0] = 1 << 20
    refused("table pool index", "bp", scans=s)
    # a progressive header with a scan range of its own
    h = hdr.copy()
    h["scan_len"][1] = 1
    refused("no scan range or restart interval", "bp", headers=h)
