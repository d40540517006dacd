"""The baseline JPEG decoder without a GPU: the host build of its arithmetic (tests/emu/faa_emu_jpeg.cpp, the same
faa_jpeg.cuh the kernels run) against Pillow's decode byte for byte, the header parser of the C ABI, and corrupt
streams that must come back with a status, never outside their buffers."""
import io

import numpy as np
import PIL.Image
import pytest

from jpeg_cases import GRID, content, emu_decode, encode, load_emu_jpeg, make

from fast_autoaugment_b200 import _lib


@pytest.fixture(scope="module")
def emu_jpeg():
    return load_emu_jpeg()


def parse(b):
    hdr = np.zeros(1, _lib.JPEG_HEADER_DTYPE)
    st = _lib.lib.faa_jpeg_parse(b, len(b), hdr.ctypes.data)
    return st, hdr[0], (_lib.lib.faa_last_error() or b"").decode()


@pytest.mark.parametrize("case", GRID, ids=[c[0] for c in GRID])
def test_host_decode_equals_pillow(emu_jpeg, case):
    b, want = make(case)
    e, status, got = emu_decode(emu_jpeg, b)
    assert e == 0 and status == 0
    assert got.shape == want.shape
    assert np.array_equal(got, want), "differs from Pillow at %d pixels" % int((got != want).any(-1).sum())


@pytest.mark.parametrize("h,w,sub,hs,vs", [(7, 9, 0, 1, 1), (33, 17, 1, 2, 1), (375, 500, 2, 2, 2), (1, 1, 2, 2, 2)])
def test_parse_reports_size_and_sampling(h, w, sub, hs, vs):
    b = encode(content("photo", h, w, 1), subsampling=sub, quality=80, restart_marker_blocks=2)
    st, hdr, _ = parse(b)
    assert st == _lib.OK
    assert (int(hdr["h"]), int(hdr["w"]), int(hdr["ncomp"]), int(hdr["hs"]), int(hdr["vs"])) == (h, w, 3, hs, vs)
    assert int(hdr["restart"]) == 2
    assert int(hdr["mcu_x"]) == -(-w // (8 * hs)) and int(hdr["mcu_y"]) == -(-h // (8 * vs))
    assert 0 < int(hdr["scan_off"]) and int(hdr["scan_off"]) + int(hdr["scan_len"]) <= len(b) - 2
    assert b[int(hdr["scan_off"]) + int(hdr["scan_len"]):][:2] == b"\xff\xd9"
    assert list(hdr["pool"]) == [-1] * 9
    g = encode(content("photo", h, w, 1), gray=True)
    st, hdr, _ = parse(g)
    assert st == _lib.OK and int(hdr["ncomp"]) == 1 and (int(hdr["hs"]), int(hdr["vs"])) == (1, 1)
    assert int(hdr["restart"]) == 0


def test_parse_refuses_progressive_and_cmyk():
    a = content("photo", 40, 56, 3)
    st, _, why = parse(encode(a, quality=80, progressive=True))
    assert st == _lib.ERR_UNSUPPORTED and "progressive" in why
    bio = io.BytesIO()
    PIL.Image.fromarray(a).convert("CMYK").save(bio, "JPEG", quality=80)
    st, _, why = parse(bio.getvalue())
    assert st == _lib.ERR_UNSUPPORTED and "CMYK" in why


def _sof_at(b):
    i = b.index(b"\xff\xc0")
    return i


def test_parse_refuses_arithmetic_and_12_bit_headers():
    b = bytearray(encode(content("gradient", 24, 24, 0), quality=75))
    i = _sof_at(bytes(b))
    arith = bytearray(b)
    arith[i + 1] = 0xC9                                    # SOF9: extended sequential, arithmetic coding
    st, _, why = parse(bytes(arith))
    assert st == _lib.ERR_UNSUPPORTED and "arithmetic" in why
    twelve = bytearray(b)
    twelve[i + 4] = 12                                     # sample precision
    st, _, why = parse(bytes(twelve))
    assert st == _lib.ERR_UNSUPPORTED and "12-bit" in why


def test_parse_refuses_other_sampling_and_malformed_headers():
    b = encode(content("gradient", 24, 24, 0), quality=75, subsampling=2)
    i = _sof_at(b)
    odd = bytearray(b)
    odd[i + 11] = 0x12                                     # luma 1x2
    st, _, why = parse(bytes(odd))
    assert st == _lib.ERR_UNSUPPORTED and "sampling" in why
    st, _, _ = parse(b"\x00\x01garbage")
    assert st == _lib.ERR_VALUE
    st, _, _ = parse(b[:i + 5])                            # cut inside the frame header
    assert st == _lib.ERR_VALUE


def _mutations():
    """deterministic corrupt streams: (name, bytes, whether the status must be non-zero)"""
    rng = np.random.default_rng(7)
    out = []
    for k, (h, w, sub, extra) in enumerate([(64, 80, 2, {}), (48, 48, 0, {"restart_marker_blocks": 2}),
                                            (40, 72, 1, {"restart_marker_rows": 1}), (33, 17, 2, {})]):
        b = encode(content("photo", h, w, k), quality=85, subsampling=sub, **extra)
        st, hdr, _ = parse(b)
        s0, n = int(hdr["scan_off"]), int(hdr["scan_len"])
        for frac in (0.0, 0.1, 0.5, 0.9, 0.99):
            out.append(("trunc%d-%g" % (k, frac), b[:s0 + int(n * frac)], True))
        for j in range(6):
            m = bytearray(b)
            pos = s0 + int(rng.integers(0, n))
            m[pos] ^= 1 << int(rng.integers(0, 8))
            out.append(("flip%d-%d" % (k, j), bytes(m), False))
        m = bytearray(b)
        m[s0 + n // 3:s0 + n // 3 + 8] = b"\xff\x00" * 4           # all-ones bits: no code of a JPEG table
        out.append(("badcode%d" % k, bytes(m), True))
    return out


MUTATIONS = _mutations()


@pytest.mark.parametrize("name,b,must_flag", MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_corrupt_streams_report_a_status_inside_their_buffers(emu_jpeg, name, b, must_flag):
    guard = 64
    src = np.full(len(b) + 2 * guard, 0x5A, np.uint8)
    src[guard:guard + len(b)] = np.frombuffer(b, np.uint8)
    st, hdr, _ = parse(b)
    assert st == _lib.OK
    h, w = int(hdr["h"]), int(hdr["w"])
    out = np.full(h * w * 3 + 2 * guard, 0xA5, np.uint8)
    status = np.zeros(1, np.int32)
    hw = np.zeros(2, np.int32)
    e = emu_jpeg.faa_emu_jpeg_decode(src.ctypes.data + guard, len(b), out.ctypes.data + guard, h * w * 3,
                                     status.ctypes.data, hw.ctypes.data)
    assert e == 0
    assert (src[:guard] == 0x5A).all() and (src[guard + len(b):] == 0x5A).all()
    assert np.array_equal(src[guard:guard + len(b)], np.frombuffer(b, np.uint8))
    assert (out[:guard] == 0xA5).all() and (out[guard + h * w * 3:] == 0xA5).all()
    if must_flag:
        assert int(status[0]) != 0
    else:
        assert int(status[0]) & ~0xF == 0
    # the same stream decodes to the same bytes every time (the output is defined)
    again = np.zeros(h * w * 3, np.uint8)
    emu_jpeg.faa_emu_jpeg_decode(src.ctypes.data + guard, len(b), again.ctypes.data, again.size, status.ctypes.data,
                                 hw.ctypes.data)
    assert np.array_equal(again, out[guard:guard + h * w * 3])


def test_table_pool_form(emu_jpeg):
    """faa_jpeg_tables gives the quantisation tables in natural order and the Huffman tables as BITS / HUFFVAL"""
    b = encode(content("photo", 32, 48, 2), quality=50, subsampling=2)
    st, hdr, _ = parse(b)
    hdr = np.array([hdr])
    tabs = np.zeros(9, _lib.JPEG_TABLE_DTYPE)
    _lib.check(_lib.lib.faa_jpeg_tables(b, len(b), hdr.ctypes.data, tabs.ctypes.data))
    im = PIL.Image.open(io.BytesIO(b))
    q = im.quantization                                     # Pillow: tables in natural order
    for c, t in ((0, 0), (1, 1), (2, 1)):
        assert np.array_equal(tabs[c]["q"], np.asarray(q[t]))
    for slot in range(3, 9):
        assert int(tabs[slot]["bits"].sum()) > 0 and not tabs[slot]["q"].any()
