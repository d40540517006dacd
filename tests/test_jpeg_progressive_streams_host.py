"""The progressive decoder's host build on hand-built streams (``jpeg_progressive_streams``): non-interleaved and
partially interleaved DC scans, single-coefficient bands, several refinement levels, EOB runs up to 32767 across
block rows and restart intervals, refinement with ZRL and correction bits, DHT / DQT / DRI redefined between scans and
coefficients at the ends of their range.  The decoded coefficients equal the blocks written, inside each component's
own extent, and the pixels equal Pillow's."""
import numpy as np
import pytest

import jpeg_progressive_cases as jp
import jpeg_progressive_streams as ps

CASES = ps.cases()


@pytest.fixture(scope="module")
def emu():
    return jp.load_emu()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stream_coefficients_and_pixels(emu, case):
    name, b, blocks, sampling = case
    e, why, h, scans = jp.parse(emu, b)
    assert e == 0, why
    st, px, coef = jp.decode(emu, b)
    assert st == 0
    at = 0
    for c, blk in enumerate(blocks):
        n = blk.shape[0] * blk.shape[1]
        got = coef[at:at + n].reshape(blk.shape)
        m = ps.extent_mask(int(h["h"]), int(h["w"]), sampling, c)
        assert np.array_equal(got[m], blk[m]), (name, c)
        at += n
    assert at == len(coef)
    assert np.array_equal(px, jp.pillow(b))
    assert [int(s["wave"]) for s in scans] == jp.brute_waves(scans)


def test_eobrun_reaches_its_maximum():
    name, b, blocks, _ = [c for c in CASES if c[0] == "eobrun_32767"][0]
    assert blocks[0].shape[0] * blocks[0].shape[1] > 32767
