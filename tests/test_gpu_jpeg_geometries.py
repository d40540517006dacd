"""The JPEG decoder on the device at every geometry its two kernels split the work by: the hand-built streams of
tests/jpeg_streams.py (edge coefficients, header layouts, narrow sizes, restart markers on the entropy kernel's chunk
edges, images on every reconstruct-tile edge, restart segment counts around its 128 threads and past 10^4) decoded as
mixed ragged batches into sentinel-filled storage.  Every image must equal Pillow and the host build, and the bytes
between images must keep the sentinel.  Also: a small call on one stream, then a call on a second stream that grows
every buffer of the decoder, with no host wait between them."""
import numpy as np
import pytest
import torch

import jpeg_streams as js
from jpeg_cases import emu_decode, load_emu_jpeg, pillow
from test_gpu_jpeg import sentinel_out, untouched_outside

from fast_autoaugment_b200 import engine
from fast_autoaugment_b200.engine import EncodedImages, decode_jpeg

pytestmark = pytest.mark.gpu

ACCEPTED = [(n, b) for n, b, ok in js.REFUSALS if ok]
GROUPS = {"random-edge": js.RANDOM + js.EDGE, "layouts": js.LAYOUTS + ACCEPTED, "narrow": js.NARROW,
          "restarts": js.RESTARTS, "tile-edges": js.TILE_EDGES, "segment-counts": js.SEGMENT_COUNTS}


def _batches(n_per=40):
    """every group in mixed batches: shuffled, so each batch mixes sizes, subsamplings and restart layouts"""
    out = []
    for g, cases in GROUPS.items():
        order = np.random.default_rng(len(cases)).permutation(len(cases))
        for k in range(0, len(order), n_per):
            out.append(("%s-%d" % (g, k // n_per), [cases[int(i)] for i in order[k:k + n_per]]))
    return out


BATCHES = _batches()


@pytest.fixture(scope="module")
def emu_jpeg():
    return load_emu_jpeg()


def _check(emu, cases, out, status):
    assert status.cpu().tolist() == [0] * len(cases)
    host = out.storage.cpu().numpy()
    want = {}                                     # (a file repeated in a call is decoded once on the host)
    for i, (name, b) in enumerate(cases):
        o, (h, w) = int(out.offsets[i]), out.sizes[i]
        img = host[o:o + int(h) * int(w) * 3].reshape(int(h), int(w), 3)
        if b not in want:
            want[b] = pillow(b)
            assert np.array_equal(want[b], emu_decode(emu, b)[2]), name
        assert np.array_equal(img, want[b]), name
    assert untouched_outside(out)


@pytest.mark.parametrize("k", range(len(BATCHES)), ids=[b[0] for b in BATCHES])
def test_streams_in_ragged_batches_equal_pillow_and_host(emu_jpeg, k):
    cases = BATCHES[k][1]
    enc = EncodedImages.from_bytes([b for _, b in cases])
    out = sentinel_out(enc.sizes)
    got, status = decode_jpeg(enc, out)
    assert got is out
    _check(emu_jpeg, cases, out, status)


def test_second_stream_grows_every_buffer():
    """a small call on stream 1, then on stream 2 a call with more blocks, restart segments and images than the first
    call's buffers hold (a fresh decoder: 64 KiB each, i.e. 512 blocks, 16 384 segments, 4 096 jobs), queued with no
    host wait; both outputs right"""
    small = js.NARROW[:3]
    large = js.SEGMENT_COUNTS * 2 + js.TILE_EDGES[:40] + js.NARROW * 13      # 23 k segments, 4 284 images
    assert len(large) > 4096
    enc_s = EncodedImages.from_bytes([b for _, b in small])
    enc_l = EncodedImages.from_bytes([b for _, b in large])
    dev = enc_s.device
    saved = engine._DECODERS.get(dev.index)
    engine._DECODERS[dev.index] = engine._JpegDecoder()
    try:
        out_s, out_l = sentinel_out(enc_s.sizes), sentinel_out(enc_l.sizes)
        enc_s.device_headers(), enc_s.device_pool(), enc_l.device_headers(), enc_l.device_pool()
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(s1):
            _, st_s = decode_jpeg(enc_s, out_s)
        with torch.cuda.stream(s2):
            _, st_l = decode_jpeg(enc_l, out_l)
        torch.cuda.synchronize()
        emu = load_emu_jpeg()
        _check(emu, small, out_s, st_s)
        _check(emu, large, out_l, st_l)
    finally:
        engine._DECODERS[dev.index] = saved
