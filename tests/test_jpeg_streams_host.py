"""The JPEG decoder's host build on hand-built streams (tests/jpeg_streams.py): coefficients at the ends of their
range and of the entropy code, every header layout the parser reads, narrow images, restart markers around the
entropy kernel's 128-chunk search and images on every reconstruct-tile edge.  Each must equal Pillow byte for byte,
decoded serially and with the kernels' split of the work (restart markers found per chunk; every 64 x 32 tile built
only from the blocks of its windows, the rest of each plane poisoned)."""
import io

import numpy as np
import PIL.Image
import pytest

import jpeg_streams as js
import jpeg_writer as jw
from jpeg_cases import SERIAL, TILED, TILED_TRIMMED, emu_decode, load_emu_jpeg

from fast_autoaugment_b200 import _lib


@pytest.fixture(scope="module")
def emu_jpeg():
    return load_emu_jpeg()


def pillow(b):
    return np.asarray(PIL.Image.open(io.BytesIO(b)).convert("RGB"))


def equal_pillow(lib, b, modes=(SERIAL, TILED)):
    want = pillow(b)
    for mode in modes:
        e, status, got = emu_decode(lib, b, mode)
        assert e == 0 and status == 0, (mode, e, status)
        assert got.shape == want.shape
        assert np.array_equal(got, want), "mode %d differs from Pillow at %d pixels" % (
            mode, int((got != want).any(-1).sum()))
    return want


def _ids(cases):
    return [c[0] for c in cases]


@pytest.mark.parametrize("name,b", js.RANDOM, ids=_ids(js.RANDOM))
def test_random_in_range_blocks_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


@pytest.mark.parametrize("name,b", js.EDGE, ids=_ids(js.EDGE))
def test_edge_blocks_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


def test_random_blocks_stay_in_range():
    rng = np.random.default_rng(1)
    for q in (1, 3, 255):
        qt = np.full(64, q)
        blocks = jw.random_blocks(rng, (50, 64), qt)
        assert jw.in_range(blocks, qt)
        assert int(np.abs(blocks[..., 1:]).max()) == 1023 // q            # the range is reached, not only its middle
        assert int(np.abs(blocks[..., 0]).max()) == 1024 // q
    for _, blocks in js._edge_blocks():
        assert jw.in_range(blocks, np.ones(64))


@pytest.mark.parametrize("name,b", js.LAYOUTS, ids=_ids(js.LAYOUTS))
def test_layouts_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


def test_layouts_of_the_same_coefficients_decode_alike():
    """the writer's self-check: every layout of one image's coefficients decodes to the same pixels in Pillow"""
    layouts = dict(js.LAYOUTS)
    want = pillow(layouts[js.LAYOUT_BASE])
    for name, b in js.LAYOUTS:
        if not name.startswith("gray-declares"):
            assert np.array_equal(pillow(b), want), name
    gray = [pillow(b) for name, b in js.LAYOUTS if name.startswith("gray-declares")]
    assert all(np.array_equal(g, gray[0]) for g in gray)


def test_long_code_tables_leave_the_lookup():
    """the long-code tables give every symbol, the most frequent first, a code longer than the 9-bit lookup"""
    bits, vals = jw.long_codes({0: 100, 1: 50, 2: 1, 0x11: 7})
    assert sum(bits[:9]) == 0 and sum(bits) == 4 and vals[-1] == 0
    assert sum(jw.optimal({s: 1 for s in range(162)})[0]) == 162


@pytest.mark.parametrize("name,b", js.NARROW, ids=_ids(js.NARROW))
def test_narrow_sizes_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


@pytest.mark.parametrize("name,b", js.RESTARTS, ids=_ids(js.RESTARTS))
def test_restart_layouts_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


def test_restart_markers_sit_on_chunk_edges():
    """the chunk-edge files put what they claim where they claim it"""
    big = js.content("photo", 48, 160, 7)
    for residue in (-1, 0, 1):
        mk = lambda fill, info: js.from_pixels(big, "420", restart=1, rst_fill=fill, info=info)  # noqa: E731
        b, info, _ = js.place_marker(mk, 5, residue)
        c = js.chunk(info["scan_len"])
        at = info["scan_off"] + info["rst_ff"][5]
        assert b[at] == 0xFF and 0xD0 <= b[at + 1] <= 0xD7 and info["rst_ff"][5] % c == residue % c
    short = dict(js.RESTARTS)["rst-short-scan-gray"]
    st, hdr = _parse(short)
    assert st == _lib.OK and int(hdr["scan_len"]) < js.CHUNKS and int(hdr["restart"]) == 1


@pytest.mark.parametrize("name,b", js.TILE_EDGES, ids=_ids(js.TILE_EDGES))
def test_tile_edges_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)


@pytest.mark.parametrize("name,b", js.SEGMENT_COUNTS, ids=_ids(js.SEGMENT_COUNTS))
def test_segment_counts_equal_pillow(emu_jpeg, name, b):
    equal_pillow(emu_jpeg, b)
    st, hdr = _parse(b)
    n = int(name.split("-")[0][3:]) if not name.startswith("seg1-") else 1
    mcus = int(hdr["mcu_x"]) * int(hdr["mcu_y"])
    assert -(-mcus // int(hdr["restart"])) == n


def test_narrow_windows_show_in_the_tiled_model(emu_jpeg):
    """the tiled model reads nothing outside a tile's windows: chroma windows one block too narrow change the output"""
    changed = 0
    for name, b in js.TILE_EDGES:
        if "gray" in name:
            continue
        e, _, got = emu_decode(emu_jpeg, b, TILED_TRIMMED)
        changed += not np.array_equal(got, pillow(b))
    assert changed >= len([n for n, _ in js.TILE_EDGES if "gray" not in n]) // 2


def _parse(b):
    hdr = np.zeros(1, _lib.JPEG_HEADER_DTYPE)
    st = _lib.lib.faa_jpeg_parse(b, len(b), hdr.ctypes.data)
    return st, hdr[0]


@pytest.mark.parametrize("name,b,ok", js.REFUSALS, ids=_ids(js.REFUSALS))
def test_parser_takes_what_pillow_takes(emu_jpeg, name, b, ok):
    try:
        pillow(b)
        pillow_ok = True
    except OSError:
        pillow_ok = False
    assert pillow_ok == ok
    st, _ = _parse(b)
    assert (st == _lib.OK) == ok, (lib_error(), st)
    if ok:
        equal_pillow(emu_jpeg, b)
    else:
        assert st == _lib.ERR_VALUE


def lib_error():
    return (_lib.lib.faa_last_error() or b"").decode()


def test_standard_tables_in_pool_form():
    """a scan without DHT gets T.81 K.3's tables in faa_jpeg_tables"""
    b = dict((n, x) for n, x, _ in js.REFUSALS)["no-dht"]
    st, hdr = _parse(b)
    assert st == _lib.OK and list(hdr["table_at"][3:7:3]) == [-2, -4]
    tabs = np.zeros(9, _lib.JPEG_TABLE_DTYPE)
    _lib.check(_lib.lib.faa_jpeg_tables(b, len(b), np.array([hdr]).ctypes.data, tabs.ctypes.data))
    for slot, key in ((3, ("dc", 0)), (6, ("ac", 0))):
        bits, vals = jw.STANDARD[key]
        assert list(tabs[slot]["bits"]) == bits and list(tabs[slot]["vals"][:len(vals)]) == vals
