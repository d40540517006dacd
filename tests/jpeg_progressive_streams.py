"""Hand-built progressive streams (``jpeg_progressive_writer``) of the progressive decoder tests: (name, file bytes,
given blocks, sampling).  Each covers something Pillow's one scan script never writes."""
import numpy as np

import jpeg_progressive_writer as pw
from jpeg_writer import block_grid, random_blocks

Q1 = np.ones(64, np.int64)
QA = np.arange(1, 65, dtype=np.int64) % 13 + 1
QB = np.arange(64, 0, -1, dtype=np.int64) % 9 + 2


def _blocks(rng, h, w, sampling, quant, qsel, density=0.3):
    """random in-range blocks of every component, AC zero outside each component's own extent (no scan writes them)"""
    out = []
    for c in range(len(sampling)):
        rows, cols = block_grid(h, w, sampling, c)
        b = random_blocks(rng, (rows, cols), quant[qsel[c]], density)
        er, ec = pw.extent(h, w, sampling, c)
        b[er:, :, 1:] = 0
        b[:, ec:, 1:] = 0
        out.append(b)
    return out


def _sc(comps, ss, se, ah=0, al=0, **kw):
    return dict(comps=list(comps), ss=ss, se=se, ah=ah, al=al, **kw)


def _case(name, h, w, sampling, scans, rng, quant=None, qsel=None, density=0.3, blocks=None):
    quant = quant or {0: QA, 1: QB}
    qsel = qsel or ([0] + [1] * (len(sampling) - 1))
    blocks = blocks if blocks is not None else _blocks(rng, h, w, sampling, quant, qsel, density)
    b = pw.write(h, w, blocks, quant, pw.script(scans), sampling=sampling, qsel=qsel)
    return name, b, blocks, sampling


def cases():
    rng = np.random.default_rng(2024)
    s420, s422, s444, gray = [(2, 2), (1, 1), (1, 1)], [(2, 1), (1, 1), (1, 1)], [(1, 1)] * 3, [(1, 1)]
    out = []
    # spectral selection without successive approximation, interleaved DC
    for name, samp in (("spectral_420", s420), ("spectral_422", s422), ("spectral_444", s444)):
        sc = [_sc([0, 1, 2], 0, 0)] + [_sc([c], a, b) for c in range(3) for a, b in ((1, 5), (6, 20), (21, 63))]
        out.append(_case(name, 37, 45, samp, sc, rng))
    # several refinement levels of DC and AC
    sc = [_sc([0, 1, 2], 0, 0, 0, 3)] + [_sc([c], 1, 63, 0, 4) for c in range(3)] + \
        [_sc([0, 1, 2], 0, 0, a + 1, a) for a in (2, 1, 0)] + \
        [_sc([c], 1, 63, a + 1, a) for a in (3, 2, 1, 0) for c in (2, 0, 1)]
    out.append(_case("refine_levels_420", 41, 30, s420, sc, rng))
    # non-interleaved DC scans (luma's own extent inside its padded grid) and a partially interleaved one
    sc = [_sc([0], 0, 0, 0, 1), _sc([1, 2], 0, 0, 0, 1)] + [_sc([c], 1, 63, 0, 1) for c in range(3)] + \
        [_sc([0], 0, 0, 1, 0), _sc([2], 0, 0, 1, 0), _sc([1], 0, 0, 1, 0)] + [_sc([c], 1, 63, 1, 0) for c in range(3)]
    out.append(_case("noninterleaved_dc_420", 25, 19, s420, sc, rng))
    out.append(_case("noninterleaved_dc_422", 9, 33, s422, sc, rng))
    # single-coefficient bands: 64 scans of a grayscale image
    sc = [_sc([0], 0, 0)] + [_sc([0], k, k) for k in range(1, 64)]
    out.append(_case("single_bands_gray", 23, 29, gray, sc, rng, density=0.6))
    # long EOB runs: up to 32767 blocks, across block rows, with and without restart intervals
    h, w = 1536, 1400
    blk = [np.zeros(block_grid(h, w, gray, 0) + (64,), np.int16)]
    blk[0][..., 0] = rng.integers(-60, 60, blk[0].shape[:2])
    blk[0][0, 0, 5], blk[0][-1, -1, 7], blk[0][100, 3, 1] = 9, -7, 3
    sc = [_sc([0], 0, 0), _sc([0], 1, 63, 0, 1), _sc([0], 1, 63, 1, 0)]
    out.append(_case("eobrun_32767", h, w, gray, sc, rng, quant={0: QA}, blocks=blk))
    sc = [_sc([0], 0, 0, restart=7), _sc([0], 1, 63, 0, 1, restart=1000), _sc([0], 1, 63, 1, 0, restart=333)]
    out.append(_case("eobrun_restarts", 400, 640, gray, sc, rng, quant={0: QA},
                     blocks=[b[:50, :80] for b in blk]))
    # refinement with ZRL and correction bits: sparse blocks, long zero runs between coefficients with history
    sc = [_sc([0], 0, 0), _sc([0], 1, 63, 0, 2), _sc([0], 1, 63, 2, 1), _sc([0], 1, 63, 1, 0)]
    out.append(_case("refine_zrl", 48, 48, gray, sc, rng, quant={0: QA}, density=0.12))
    # DHT (every scan), DQT and DRI redefined between scans: the DQT after a component's first scan changes nothing
    sc = [_sc([0, 1, 2], 0, 0, 0, 1, restart=3), _sc([0], 1, 63, 0, 1, restart=0, dqt={0: QB, 1: QA}),
          _sc([1], 1, 63, restart=5), _sc([2], 1, 63), _sc([0, 1, 2], 0, 0, 1, 0, restart=2),
          _sc([0], 1, 63, 1, 0, restart=0)]
    out.append(_case("redefined_tables", 40, 56, s420, sc, rng))
    # coefficients at the ends of their range (unit quantisation: |DC| <= 1024, |AC| <= 1023)
    ends = _blocks(rng, 16, 16, gray, {0: Q1}, [0], density=0.0)
    ends[0][0, 0, 0], ends[0][0, 1, 0], ends[0][1, 0, 0], ends[0][1, 1, 0] = 1024, -1024, 1023, -1023
    ends[0][0, 0, 63], ends[0][0, 1, 1], ends[0][1, 0, 8], ends[0][1, 1, 62] = 1023, -1023, 1, -1
    sc = [_sc([0], 0, 0, 0, 1), _sc([0], 1, 63, 0, 2), _sc([0], 0, 0, 1, 0), _sc([0], 1, 63, 2, 1),
          _sc([0], 1, 63, 1, 0)]
    out.append(_case("range_ends", 16, 16, gray, sc, rng, quant={0: Q1}, blocks=ends))
    return out


def extent_mask(h, w, sampling, c):
    rows, cols = block_grid(h, w, sampling, c)
    er, ec = pw.extent(h, w, sampling, c)
    m = np.zeros((rows, cols), bool)
    m[:er, :ec] = True
    return m
