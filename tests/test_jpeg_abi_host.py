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


def _batch(progressive=False):
    """(headers, n_tables, h_out) of two 96 x 128 files"""
    a = content("photo", 96, 128, 2)
    b = jp.encode(a, progressive=True, quality=95) if progressive else encode(a, quality=95)
    headers, pool = engine.parse_jpeg_headers([b, b], progressive=progressive)[:2]
    out = np.zeros(2, dtype=_lib.IMAGE_DTYPE)
    out["data"], out["h"], out["w"] = DEV, 96, 128
    return headers, len(pool), out


@pytest.mark.skipif(torch.cuda.is_available(), reason="a call that passes its checks would launch on the dummy pointers")
def test_decode_refusals_come_before_the_device():
    dec = engine._JpegDecoder()
    headers, n_tables, h_out = _batch()
    first = np.array([0, 8, 16], np.int64)
    empty = np.zeros(3, np.int64)

    def call(index=(None,) * 3, rec=(None,) * 4, find=0, batch=2, headers=headers):
        return _lib.lib.faa_jpeg_decode(dec.handle, headers.ctypes.data, DEV, DEV, n_tables, DEV, batch,
                                        h_out.ctypes.data, DEV, DEV, *index, *rec, find, None)

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
    # a progressive header is faa_jpeg_decode_progressive's
    assert call(headers=_batch(progressive=True)[0]) == _lib.ERR_VALUE
    assert b"progressive" in _lib.lib.faa_last_error()
    # batch bounds
    assert call(batch=-1) == _lib.ERR_VALUE
    assert call(batch=65536) == _lib.ERR_UNSUPPORTED
