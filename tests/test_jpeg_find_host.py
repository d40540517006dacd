"""The scan index found in parallel, without a GPU: the host build of ``jpeg_index_find``
(tests/emu/faa_emu_jpeg_find.cpp, the same faa_jpeg.cuh steps faa_jpeg_find_kernel runs on one thread per part), with
the window W and the round cap R as parameters.

Found points are always a prefix of the serial decode's index (``jpeg_index_record``) and equal it wherever the chain
converged: on the decoder's Pillow grid, on the restart-free hand-built streams, and on adversarial streams (identical
blocks in every component, so a parse one block off stays one block off; thresholds on a stuffed 0xFF or its 0x00;
scans of exactly 2 KiB and at the 128-part cap; one-MCU-wide images; every sampling).  On corrupt and truncated scans
every found point is the serial decoder's state at its MCU, and the indexed decode over the found points gives the
plain decode's pixels and status.  Nothing is written outside a file's point range."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_index_cases as jic
import jpeg_streams as js
import jpeg_writer as jw
from helpers import ROOT
from test_jpeg_host import MUTATIONS
from test_jpeg_index_host import FILES, GRID_CHUNKS, STREAMS, _mutated, grid_bytes, header

SYNC = jic.SYNC
GUARD = 64
WINDOWS = (0, 512, 4096)              # none, the kernel's, and more than a part
ROUNDS = (1, 8, 128)                  # one round, the kernel's cap, and enough for any chain
KERNEL_W, KERNEL_R = 512, 8


def load_emu_find():
    so = os.path.join(ROOT, "tests", "emu", "libfaa_emu_jpeg_find.so")
    src = os.path.join(ROOT, "tests", "emu", "faa_emu_jpeg_find.cpp")
    hdr = os.path.join(ROOT, "fast_autoaugment_b200", "csrc", "faa_jpeg.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    lib = C.CDLL(so)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int32
    lib.faa_emu_jpeg_find.argtypes = [vp, i64, i32, i32, vp, i32, vp]
    return lib


@pytest.fixture(scope="module")
def emu():
    return load_emu_find()


@pytest.fixture(scope="module")
def emu_index():
    return jic.load_emu_index()


def find(lib, b, window=KERNEL_W, rounds=KERNEL_R, cap=jic.MAX_PARTS - 1):
    """(points, stats) of the host build's find: stats = (links, held in round 1, rounds run, converged).  Guard bytes
    around the point range must keep their value."""
    src = np.frombuffer(b, np.uint8).copy()
    raw = np.full((cap + 2 * GUARD) * 16, 0x3C, np.uint8)
    st = np.full(4, -7, np.int32)
    n = lib.faa_emu_jpeg_find(src.ctypes.data, src.size, window, rounds, raw.ctypes.data + GUARD * 16, cap,
                              st.ctypes.data)
    assert 0 <= n <= cap
    assert (raw[:GUARD * 16] == 0x3C).all() and (raw[(GUARD + n) * 16:] == 0x3C).all()
    return raw[GUARD * 16:(GUARD + n) * 16].view(SYNC).copy(), tuple(int(x) for x in st)


def check_found(lib, emu_index, b, windows=WINDOWS, rounds=ROUNDS):
    """found points are a prefix of the serial index and all of it when converged; returns {(W, R): converged}"""
    want, st, _ = jic.host_index(emu_index, b)
    h = header(b)
    parts = jic.parts(int(h["scan_len"]), int(h["restart"]))
    out = {}
    for w in windows:
        for r in rounds:
            got, (links, held, ran, full) = find(lib, b, w, r)
            assert links == max(parts - 1, 0) and 0 <= held <= links and ran <= r
            if parts == 0:
                assert len(got) == 0 and not full
                continue
            if st == 0:
                assert got.tobytes() == want[:len(got)].tobytes(), (w, r)
                if full:
                    assert got.tobytes() == want.tobytes(), (w, r)
            if r >= parts and len(want) == parts - 1:      # each round verifies at least one more link
                assert full or st != 0, (w, r)
            out[(w, r)] = bool(full)
    return out


@pytest.mark.parametrize("k", range(len(GRID_CHUNKS)), ids=lambda k: GRID_CHUNKS[k][0][0])
def test_grid_found_points_are_a_prefix_and_all_when_converged(emu, emu_index, k):
    for case in GRID_CHUNKS[k]:
        check_found(emu, emu_index, grid_bytes(case), windows=(0, 4096), rounds=(1, 128))


@pytest.mark.parametrize("k", range(0, len(STREAMS), 16), ids=lambda k: STREAMS[k][0])
def test_streams_found_points_are_a_prefix_and_all_when_converged(emu, emu_index, k):
    for _, b in STREAMS[k:k + 16]:
        check_found(emu, emu_index, b)


def test_photo_files_converge_at_the_kernel_window_and_rounds(emu, emu_index):
    """the parameters the kernel uses converge on these photo-like files (DESIGN §4.8 has the sweep)"""
    for name, b in FILES:
        if name.startswith("noise"):
            continue
        conv = check_found(emu, emu_index, b, windows=(KERNEL_W,), rounds=(KERNEL_R,))
        assert conv[(KERNEL_W, KERNEL_R)], name


# ------------------------------------------------------------------------------------------------ adversarial streams
QUANT2 = {0: np.full(64, 2), 1: np.full(64, 2)}


def _identical(sub, h, w, seed):
    """every block of every component the same, one quantisation table and one pair of Huffman tables: a parse that
    starts one block off inside an MCU decodes the same symbols and stays one block off"""
    samp = js.SAMPLINGS[sub]
    blk = jw.random_blocks(np.random.default_rng(seed), (1, 1), QUANT2[0], density=0.6)[0, 0]
    blocks = [np.broadcast_to(blk, jw.block_grid(h, w, samp, c) + (64,)).copy() for c in range(len(samp))]
    return jw.write(h, w, blocks, QUANT2, sampling=samp, qsel=[0] * len(samp), tsel=[(0, 0)] * len(samp))


def _padded(b, scan_len):
    """b with zero bytes after its entropy-coded data so that the scan is exactly scan_len bytes"""
    h = header(b)
    end = int(h["scan_off"]) + int(h["scan_len"])
    assert int(h["scan_len"]) <= scan_len
    return b[:end] + bytes(scan_len - int(h["scan_len"])) + b[end:]


def _stuffed_thresholds(b):
    """(parts, thresholds on the 0xFF of a stuffed pair, thresholds on its 0x00)"""
    h = header(b)
    s0, n = int(h["scan_off"]), int(h["scan_len"])
    p = jic.parts(n, 0)
    zeros = set(jic.stuffed_offsets(b, s0, n))
    ts = [k * n // p for k in range(1, p)]
    return p, [t for t in ts if t + 1 in zeros], [t for t in ts if t in zeros]


def adversarial():
    out = []
    for sub in ("gray", "444", "422", "420"):
        out.append(("identical-%s" % sub, _identical(sub, 96, 128, 1)))
    rng = np.random.default_rng(7)
    for sub, w in (("gray", 8), ("444", 8), ("422", 16), ("420", 16)):      # one MCU wide
        out.append(("one-mcu-wide-%s" % sub, js.random_file(rng, 1024, w, sub, QUANT2)))
    for sub, h, w in (("gray", 48, 64), ("420", 48, 40)):                 # exactly 2 KiB: P = 2
        base = js.random_file(np.random.default_rng(3), h, w, sub, QUANT2)
        assert 1100 < int(header(base)["scan_len"]) <= 2048, sub
        out.append(("2KiB-%s" % sub, _padded(base, 2048)))
    # a scan of exactly 2 KiB whose data ends before the threshold: the rule places nothing past the last MCU
    short = js.random_file(np.random.default_rng(3), 8, 16, "444", QUANT2)
    out.append(("2KiB-mostly-padding", _padded(short, 2048)))
    big = js.random_file(np.random.default_rng(11), 256, 256, "444", QUANT2)
    assert jic.parts(int(header(big)["scan_len"]), 0) >= 64
    out.append(("many-parts-444", big))
    out.append(("128-parts", jic.big_file()))
    for seed in range(40):                      # thresholds on each byte of a stuffed pair
        b = js.random_file(np.random.default_rng(100 + seed), 128, 128, "420", {0: np.full(64, 1), 1: np.full(64, 1)})
        _, on_ff, on_00 = _stuffed_thresholds(b)
        if on_ff and not any(n.startswith("threshold-on-ff") for n, _ in out):
            out.append(("threshold-on-ff", b))
        if on_00 and not any(n.startswith("threshold-on-00") for n, _ in out):
            out.append(("threshold-on-00", b))
    return out


ADVERSARIAL = adversarial()


def test_adversarial_set_covers_what_it_claims():
    names = [n for n, _ in ADVERSARIAL]
    assert "threshold-on-ff" in names and "threshold-on-00" in names
    assert jic.parts(int(header(dict(ADVERSARIAL)["128-parts"])["scan_len"]), 0) == 128
    for n in ("2KiB-gray", "2KiB-420", "2KiB-mostly-padding"):
        assert int(header(dict(ADVERSARIAL)[n])["scan_len"]) == 2048


@pytest.mark.parametrize("k", range(len(ADVERSARIAL)), ids=[a[0] for a in ADVERSARIAL])
def test_adversarial_streams_end_in_a_verified_prefix(emu, emu_index, k):
    name, b = ADVERSARIAL[k]
    conv = check_found(emu, emu_index, b, windows=(0, 1, 64, KERNEL_W, 4096), rounds=(1, 2, KERNEL_R, 128))
    st0, px0 = jic.decode_indexed(emu_index, b, np.zeros(0, SYNC))
    for w in (0, KERNEL_W):
        got, _ = find(emu, b, w, KERNEL_R)
        assert jic.decode_indexed(emu_index, b, got)[0] == st0
        assert np.array_equal(jic.decode_indexed(emu_index, b, got)[1], px0), name
    if name.startswith("identical-") and name != "identical-gray":
        # every candidate is a block boundary, most at the wrong block of their MCU: one round verifies one link
        _, (links, held, _, full) = find(emu, b, KERNEL_W, 1)
        assert links > 2 and held < links and not full
    else:
        assert conv[(4096, 128)] or name == "2KiB-mostly-padding"


def test_one_round_verifies_at_least_one_link_per_round(emu, emu_index):
    _, b = ADVERSARIAL[[n for n, _ in ADVERSARIAL].index("identical-420")]
    want = jic.host_index(emu_index, b)[0]
    prev = -1
    for r in range(1, len(want) + 2):
        got, (_, _, _, full) = find(emu, b, KERNEL_W, r)
        assert len(got) >= min(r, len(want)) and len(got) >= prev
        prev = len(got)
    assert full and got.tobytes() == want.tobytes()


def test_capacity_short_gives_the_first_points(emu, emu_index):
    b = jic.big_file()
    want = jic.host_index(emu_index, b)[0]
    for cap in (1, 5, 126):
        got, (_, _, _, full) = find(emu, b, KERNEL_W, 128, cap=cap)
        assert got.tobytes() == want[:cap].tobytes() and not full
    got, (_, _, _, full) = find(emu, b, KERNEL_W, 128, cap=127)
    assert got.tobytes() == want.tobytes() and full


# ------------------------------------------------------------------------------------------------ corrupt scans
def _corrupt():
    return [("mutation-%d" % i, b) for i, (_, b, _) in enumerate(MUTATIONS)] + \
        [("%s-%s" % (name, what), m) for name, good in FILES for what, m in _mutated(good, len(good))]


CORRUPT = _corrupt()


def test_corrupt_and_truncated_scans_find_only_true_points(emu, emu_index):
    flagged = 0
    for name, b in CORRUPT:
        try:
            h = header(b)
        except AssertionError:
            continue
        st0, px0 = jic.decode_indexed(emu_index, b, np.zeros(0, SYNC))
        flagged += st0 != 0
        mcus = int(h["mcu_x"]) * int(h["mcu_y"])
        states = jic.host_states(emu_index, b, mcus)
        for w in (0, KERNEL_W):
            got, _ = find(emu, b, w, KERNEL_R)
            for p in got:                        # the serial decoder's state at that MCU, decoded cleanly up to it
                assert int(p["mcu"]) < len(states) and states[int(p["mcu"])].tobytes() == p.tobytes(), name
            st, px = jic.decode_indexed(emu_index, b, got)
            assert st == st0 and np.array_equal(px, px0), name
    assert flagged > 10
