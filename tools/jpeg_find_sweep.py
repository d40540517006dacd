"""Measures, on the CPU, how often a scan index found in parallel converges: the window W and round cap R of
``jpeg_index_find`` (fast_autoaugment_b200/csrc/faa_jpeg.cuh, DESIGN.md 4.8).

    python tools/jpeg_find_sweep.py [--batch 256] [--windows 0,64,128,256,512,1024] [--out OUTDIR]

Whether a parse started at an arbitrary byte falls onto the true code boundaries and the true block of its MCU is a
property of the bytes, so the host build of the find (tests/emu/faa_emu_jpeg_find.cpp, compiled into a temporary
directory) measures it exactly.  Sets: the restart-free files of the decoder's Pillow grid (tests/jpeg_cases.py) with a
scan of at least 2 KiB, tools/jpeg_index_probe.py's b256 SYNTHETIC photo-like 375x500 4:2:0 q75 and q90 sets, and its
b256 size mixture at q90 (DESIGN.md 4.9).  For each set and W: the share of links that hold in round 1, and the share
of files whose chain converges within R = 1, 2, 3, 4, 6, 8 rounds.  Every found prefix is checked against the serial
decode's index (``jpeg_index_record``).  One JSON line per (set, W), also in OUTDIR/jpeg_find_sweep.jsonl."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from fast_autoaugment_b200 import _lib  # noqa: E402

SYNC = _lib.JPEG_SYNC_DTYPE
ROUNDS = (1, 2, 3, 4, 6, 8)


def load(tmp):
    libs = []
    for name in ("faa_emu_jpeg_find", "faa_emu_jpeg_index"):
        so = os.path.join(tmp, "lib%s.so" % name)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so,
                               os.path.join(ROOT, "tests", "emu", name + ".cpp")])
        libs.append(C.CDLL(so))
    find, index = libs
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int32
    find.faa_emu_jpeg_find.argtypes = [vp, i64, i32, i32, vp, i32, vp]
    index.faa_emu_jpeg_index.argtypes = [vp, i64, vp, i32, vp, vp]
    return find, index


def found(lib, b, window, rounds):
    src = np.frombuffer(b, np.uint8).copy()
    out = np.zeros(128, SYNC)
    st = np.zeros(4, np.int32)
    n = lib.faa_emu_jpeg_find(src.ctypes.data, src.size, window, rounds, out.ctypes.data, 127, st.ctypes.data)
    return out[:max(n, 0)].copy(), st


def recorded(lib, b):
    src = np.frombuffer(b, np.uint8).copy()
    out = np.zeros(128, SYNC)
    st = np.zeros(1, np.int32)
    scan = np.zeros(2, np.int64)
    n = lib.faa_emu_jpeg_index(src.ctypes.data, src.size, out.ctypes.data, 127, st.ctypes.data, scan.ctypes.data)
    return out[:max(n, 0)].copy(), int(st[0])


def grid_files():
    from test_jpeg_index_host import GRID, grid_bytes
    out = []
    for case in GRID:
        b = grid_bytes(case)
        if "restart_marker_blocks" in case[4] or "restart_marker_rows" in case[4]:
            continue
        out.append(b)
    return out


def sweep(find, index, label, files, windows):
    want = [recorded(index, b) for b in files]
    keep = [(b, w) for b, w in zip(files, want) if len(w[0]) and w[1] == 0]
    lines = []
    for window in windows:
        links = held = 0
        conv = {r: 0 for r in ROUNDS}
        for b, (pts, _) in keep:
            for r in ROUNDS:
                got, st = found(find, b, window, r)
                assert got.tobytes() == pts[:len(got)].tobytes(), (label, window, r)    # always a prefix
                if st[3]:
                    assert got.tobytes() == pts.tobytes(), (label, window, r)
                conv[r] += int(st[3])
                if r == 1:
                    links += int(st[0])
                    held += int(st[1])
        line = {"set": label, "files": len(keep), "window": window, "links": links,
                "held_round1_pct": round(100 * held / max(links, 1), 2),
                **{"converged_R%d_pct" % r: round(100 * conv[r] / max(len(keep), 1), 2) for r in ROUNDS}}
        lines.append(line)
        print(json.dumps(line), flush=True)
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--windows", default="0,64,128,256,512,1024")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    windows = [int(w) for w in a.windows.split(",")]
    from jpeg_index_probe import sets
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        find, index = load(tmp)
        lines += sweep(find, index, "pillow-grid", grid_files(), windows)
        for label, files in sets(a.batch):
            lines += sweep(find, index, label, files, windows)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_find_sweep.jsonl"), "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
