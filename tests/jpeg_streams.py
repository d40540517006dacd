"""Hand-built JPEG streams of the decoder tests (written by tests/jpeg_writer.py), shared by the host tests
(test_jpeg_streams_host.py) and the device tests (test_gpu_jpeg_geometries.py).  Every list holds (name, file bytes)
and is built deterministically at import.

- ``RANDOM``: random in-range coefficient blocks at q in {1, 2, 3, 8, 16, 255} and under a random table, grayscale
  and 4:2:0, serial and with restart markers.
- ``EDGE``: blocks at the ends of the coefficient range and of the entropy code: DC differences of category 11,
  AC values of category 10, ZRL runs up to coefficient 63, a last coefficient at 63 (no EOB), flat DC +-1024.
- ``LAYOUTS``: one image's coefficients in every header layout the parser must read (``LAYOUT_BASE`` names the plain
  one; all decode to the same pixels).
- ``NARROW``: every size w, h in 1..9 with each subsampling.
- ``RESTARTS``: restart intervals around the entropy kernel's 128 threads and mid-row, restart markers whose 0xFF
  sits on a chunk's first or last byte, fill runs across a chunk edge and scans shorter than 128 bytes.
- ``TILE_EDGES``: images of 1x1 to 3x3 reconstruct tiles (64 x 32) with every residue that moves a tile edge or a
  chroma halo, in each subsampling.
- ``SEGMENT_COUNTS``: restart segment counts 1, 2, 127, 128, 129, 255, 256, 257 and one image of more than 10^4.
- ``REFUSALS``: (name, bytes, whether Pillow and the parser take it): an all-ones Huffman code, stray bytes between
  segments, a scan without DHT (standard tables) or without DQT."""
import numpy as np
import PIL.Image

import jpeg_writer as jw
from jpeg_cases import content

SAMPLINGS = {"gray": [(1, 1)], "444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "420": [(2, 2), (1, 1), (1, 1)]}
QUANT = {0: np.full(64, 4), 1: np.full(64, 6)}
CHUNKS = 128                                   # threads of the entropy kernel's restart-marker search


def planes(a, sub):
    """sample planes of RGB pixels for a subsampling: Y (and Cb, Cr averaged over the chroma sample's pixels)"""
    if sub == "gray":
        return [np.asarray(PIL.Image.fromarray(a).convert("L"))]
    ycc = np.asarray(PIL.Image.fromarray(a).convert("YCbCr")).astype(np.float64)
    hs, vs = SAMPLINGS[sub][0]
    h, w = a.shape[:2]
    out = [ycc[..., 0]]
    for c in (1, 2):
        p = np.pad(ycc[..., c], ((0, (-h) % vs), (0, (-w) % hs)), mode="edge")
        out.append(p.reshape(p.shape[0] // vs, vs, p.shape[1] // hs, hs).mean(axis=(1, 3)))
    return out


def from_pixels(a, sub, quant=QUANT, **kw):
    """a file of RGB pixels `a` in subsampling `sub` (components use table 0, chroma 1 unless qsel says otherwise)"""
    h, w = a.shape[:2]
    samp = SAMPLINGS[sub]
    qsel = kw.get("qsel", [0] + [1] * (len(samp) - 1))
    blocks = [jw.coefs_from_plane(p, quant[qsel[c]], jw.block_grid(h, w, samp, c)) for c, p in enumerate(planes(a, sub))]
    return jw.write(h, w, blocks, quant, sampling=samp, **kw)


def random_file(rng, h, w, sub, quant, **kw):
    samp = SAMPLINGS[sub]
    qsel = kw.get("qsel", [0] + [1] * (len(samp) - 1))
    blocks = [jw.random_blocks(rng, jw.block_grid(h, w, samp, c), quant[qsel[c]]) for c in range(len(samp))]
    return jw.write(h, w, blocks, quant, sampling=samp, **kw)


def _random():
    rng = np.random.default_rng(101)
    out = []
    for q in (1, 2, 3, 8, 16, 255):
        quant = {0: np.full(64, q), 1: np.full(64, q)}
        out.append(("random-q%d-gray" % q, random_file(rng, 48, 64, "gray", quant)))
        out.append(("random-q%d-420-rst" % q, random_file(rng, 40, 56, "420", quant, restart=2)))
    quant = {0: rng.integers(1, 256, 64), 1: rng.integers(1, 40, 64)}
    out.append(("random-qrand-444", random_file(rng, 24, 40, "444", quant)))
    out.append(("random-qrand-422-16bit", random_file(rng, 24, 40, "422", {0: rng.integers(1, 2000, 64),
                                                                          1: rng.integers(1, 700, 64)}, qbits=16)))
    return out


def _edge_blocks():
    """(name, [n, 64] natural-order blocks at q = 1)"""
    zz = jw.ZIGZAG
    out = []
    dc = np.zeros((16, 64), np.int64)
    dc[:, 0] = [-1024, 1023] * 8                                   # differences of 2047: category 11
    out.append(("dc-cat11", dc))
    flat = np.zeros((8, 64), np.int64)
    flat[:, 0] = [1024, 1024, 0, -1024, -1024, 0, 1024, 0]
    out.append(("flat-dc-1024", flat))
    ac = np.zeros((12, 64), np.int64)
    for i in range(12):                                            # category 10: 512..1023
        k = zz[[1, 2, 5, 9, 20, 35, 50, 62, 63, 3, 14, 27][i]]
        ac[i, k] = [1023, -1023, 512, -512][i % 4]
        ac[i, zz[(i * 7) % 63 + 1]] = [-1023, 700, -600, 1023][i % 4]
    out.append(("ac-cat10", ac))
    zrl = np.zeros((4, 64), np.int64)
    zrl[0, zz[63]] = 5                                             # run 62 = 3 ZRL + 14, then coefficient 63
    zrl[1, zz[14]] = -3
    zrl[1, zz[63]] = 1023                                          # 48 zeros = 3 ZRL, then coefficient 63
    zrl[2, zz[15]] = 2                                             # 3 ZRL then EOB-less end at 63
    zrl[2, zz[63]] = -1
    zrl[3, zz[47]] = 9                                             # 2 ZRL, run 14, then EOB
    out.append(("zrl-to-63", zrl))
    last = np.zeros((6, 64), np.int64)
    last[:, zz[63]] = [1, -1, 1023, -1023, 300, -2]
    last[:, 0] = [10, -10, 0, 1024, -1024, 5]
    out.append(("last-63-no-eob", last))
    ex = np.zeros((1, 64), np.int64)
    ex[0, 0] = 1016                                                # IDCT outputs past 511: saturate, not wrap
    ex[0, [1, 8, 9]] = 1023
    out.append(("saturating-idct", ex))
    return out


def _edge():
    out = []
    ones = np.ones(64, np.int64)
    for name, blocks in _edge_blocks():
        n = len(blocks)
        g = blocks.reshape(1, n, 64)
        out.append(("edge-%s-gray" % name, jw.write(8, 8 * n, [g], {0: ones})))
        out.append(("edge-%s-gray-rst" % name, jw.write(8, 8 * n, [g], {0: ones}, restart=1)))
        out.append(("edge-%s-long-codes" % name, jw.write(8, 8 * n, [g], {0: ones},
                                                          huff={("dc", 0): jw.long_codes, ("ac", 0): jw.long_codes})))
        # 4:2:0: the blocks as luma, and again as both chroma planes
        mx = n
        y = np.concatenate([g, g[:, ::-1]], axis=0).repeat(2, axis=1)[:, :2 * mx]
        out.append(("edge-%s-420" % name, jw.write(16, 16 * mx, [y, g, g[:, ::-1]], {0: ones, 1: ones},
                                                   sampling=SAMPLINGS["420"])))
    return out


def _layouts():
    rng = np.random.default_rng(202)
    a = content("photo", 37, 45, 3)
    h, w = a.shape[:2]
    samp = SAMPLINGS["420"]
    q3 = {0: rng.integers(1, 30, 64), 1: rng.integers(2, 40, 64), 2: rng.integers(2, 40, 64)}
    ps = planes(a, "420")
    blocks = [jw.coefs_from_plane(ps[c], q3[c], jw.block_grid(h, w, samp, c)) for c in range(3)]
    base = dict(quant=q3, sampling=samp, qsel=[0, 1, 2], restart=5)
    W = lambda **kw: jw.write(h, w, blocks, **dict(base, **kw))  # noqa: E731
    out = [
        (LAYOUT_BASE, W()),
        ("merged-tables", W(merge_dqt=True, merge_dht=True)),
        ("tables-after-sof", W(segments=["app0", "sof", "dht", "dri", "dqt"])),
        ("no-jfif", W(jfif=False)),
        ("com-app1-app2", W(segments=[(0xFE, b"a comment"), "app0", (0xE1, b"Exif\x00\x00" + bytes(40)),
                                      (0xE2, b"ICC_PROFILE\x00" + bytes(20)), "dqt", "sof", (0xFE, b""), "dht", "dri"])),
        ("fill-before-markers", W(before={0: b"\xff", 1: b"\xff" * 3, 2: b"\xff" * 2, 3: b"\xff", 4: b"\xff" * 7,
                                          "sos": b"\xff" * 2, "eoi": b"\xff" * 4})),
        ("fill-before-rst", W(rst_fill={0: 1, 1: 5, 2: 2})),
        ("stray-bytes", W(before={1: b"\x00", 2: b"\x12\x34\x56", 4: b"\x00\xfe", "sos": b"\x80"})),
        ("trailing-bytes", W(trailing=b"\x00\x00\xff\xd8 trailing garbage")),
        ("ids-0-1-2", W(ids=[0, 1, 2])),
        ("ids-odd", W(ids=[7, 200, 255])),
        ("quant-16bit-sof1", W(qbits=16)),
        ("huff-ids-2-3-sof1", W(tsel=[(2, 3), (3, 2), (2, 3)], sof=0xC1)),
        ("huff-ids-2-3-sof0", W(tsel=[(3, 3), (2, 2), (3, 3)])),
        ("huff-per-component", W(tsel=[(0, 1), (1, 0), (2, 3)], sof=0xC1, merge_dht=True)),
        ("huff-long-codes", W(huff={(k, i): jw.long_codes for k in ("dc", "ac") for i in (0, 1)})),
        ("standard-tables-no-dht", W(huff=dict(jw.STANDARD), segments=["app0", "dqt", "sof", "dri"])),
        ("standard-tables-dht", W(huff=dict(jw.STANDARD))),
    ]
    return out


LAYOUT_BASE = "layout-base"


def _gray_sampling():
    a = content("photo", 21, 27, 4)
    out = []
    for s in ((2, 2), (2, 1), (1, 2), (4, 4), (3, 1)):
        out.append(("gray-declares-%dx%d" % s, jw.write(21, 27, [jw.coefs_from_plane(planes(a, "gray")[0], QUANT[0],
                                                                                      (3, 4))],
                                                        QUANT, sampling=[s], restart=2)))
    return out


def _narrow():
    out = []
    for sub in SAMPLINGS:
        for h in range(1, 10):
            for w in range(1, 10):
                a = content("noise", h, w, 10 * h + w)
                out.append(("narrow-%s-%dx%d" % (sub, h, w), from_pixels(a, sub, restart=1 if (h + w) % 3 == 0 else 0)))
    return out


def chunk(scan_len):
    return -(-scan_len // CHUNKS)


def place_marker(make, k, residue, limit=600):
    """a file from make(rst_fill) whose k-th restart marker's 0xFF (the one before its code) is at a scan offset
    congruent to `residue` (mod the chunk size; -1: a chunk's last byte), found by adding fill bytes before it"""
    info = {}
    make({}, info)
    for n in range(limit):                     # n fill bytes move the marker and lengthen the scan by n
        c = chunk(info["scan_len"] + n)
        if (info["rst_ff"][k] + n) % c == residue % c:
            info = {}
            b = make({k: n}, info)
            assert (info["rst_ff"][k] - residue) % chunk(info["scan_len"]) == 0
            return b, info, n
    raise AssertionError("no fill puts marker %d at residue %d" % (k, residue))


def _restarts():
    out = []
    a = content("photo", 64, 96, 5)
    for sub in ("gray", "420", "422"):
        for r in (1, 2, 3, 5, 7, 13):                             # intervals that end mid-row
            out.append(("rst-%s-r%d" % (sub, r), from_pixels(a, sub, restart=r)))
    # restart segment counts around the 128 threads: gray 8 x 8n, one MCU per interval
    g = content("noise", 8, 8 * 130, 6)
    for n in (127, 128, 129):
        out.append(("rst-gray-%dseg" % n, from_pixels(g[:, :8 * n], "gray", restart=1)))
        out.append(("rst-444-%dseg" % n, from_pixels(g[:, :8 * n], "444", restart=1)))
    # markers on chunk edges, fill runs across one, scans shorter than 128 bytes
    big = content("photo", 48, 160, 7)
    for sub, r in (("gray", 4), ("420", 1), ("444", 3)):
        for k in (0, 5):
            for residue in (-1, 0, 1):
                mk = lambda fill, info, sub=sub, r=r: from_pixels(big, sub, restart=r, rst_fill=fill, info=info)  # noqa
                b, _, n = place_marker(mk, k, residue)
                out.append(("rst-%s-marker%d-at-chunk%+d-fill%d" % (sub, k, residue, n), b))
        info = {}
        from_pixels(big, sub, restart=r, info=info)
        c = chunk(info["scan_len"])
        n = c + 3                                                 # a fill run longer than a chunk
        out.append(("rst-%s-fill-across-chunks" % sub, from_pixels(big, sub, restart=r, rst_fill={2: n, 3: 1})))
    flat = np.full((8, 64, 3), 90, np.uint8)
    for sub in ("gray", "444"):
        out.append(("rst-short-scan-%s" % sub, from_pixels(flat, sub, restart=1)))
        out.append(("rst-short-scan-%s-fill" % sub, from_pixels(flat, sub, restart=1, rst_fill={1: 3, 4: 1, 6: 9})))
    return out


TILE_W_RES = (0, 1, 2, 8, 15, 16, 17, 31, 32, 33, 48, 63)     # w mod 64: tile edges, chroma blocks and their halo
TILE_H_RES = (0, 1, 2, 8, 15, 16, 17, 31)                      # h mod 32


def _tile_edges():
    out = []
    k = 0
    for sub in SAMPLINGS:
        for i, rw in enumerate(TILE_W_RES):
            for tx, ty in ((0, 0), (1, 1), (2, 2), (2, 1)):
                rh = TILE_H_RES[(i + tx + 3 * ty) % len(TILE_H_RES)]
                w, h = 64 * tx + rw, 32 * ty + rh
                if w == 0 or h == 0:
                    w, h = w or 64, h or 32
                a = content("photo" if k % 2 else "noise", h, w, 300 + k)
                out.append(("tile-%s-%dx%d" % (sub, h, w), from_pixels(a, sub, restart=[0, 0, 3, 1][k % 4])))
                k += 1
    return out


def _segment_counts():
    out = []
    g = content("noise", 16, 16 * 260, 8)
    out.append(("seg1-interval-past-mcus", from_pixels(g[:, :96], "gray", restart=1000)))
    for n in (2, 127, 128, 129, 255, 256, 257):
        out.append(("seg%d-gray" % n, from_pixels(g[:8, :8 * n], "gray", restart=1)))
        out.append(("seg%d-420" % n, from_pixels(g[:, :16 * n], "420", restart=1)))
    huge = content("photo", 8 * 80, 8 * 128, 9)                  # 10 240 segments of one MCU
    out.append(("seg10240", from_pixels(huge, "gray", restart=1)))
    return out


def _refusals():
    rng = np.random.default_rng(303)
    quant = {0: np.full(64, 5)}
    blocks = [jw.random_blocks(rng, (2, 3), quant[0])]
    W = lambda **kw: jw.write(16, 24, blocks, quant, **kw)  # noqa: E731
    return [
        ("all-ones-dc-code", W(huff={("dc", 0): ([0, 0, 0, 16] + [0] * 12, list(range(16)))}), False),
        ("all-ones-ac-code", W(huff={("ac", 0): jw.all_ones}), False),
        ("one-short-of-all-ones", W(huff={("dc", 0): ([0, 0, 0, 15] + [0] * 12, list(range(15)))}), True),
        ("stray-bytes-after-app0", W(before={1: b"\x00\x01", 2: b"\x7f"}), True),
        ("no-dht", W(huff=dict(jw.STANDARD), segments=["app0", "dqt", "sof"]), True),
        ("no-dqt", W(segments=["app0", "sof", "dht"]), False),
        ("no-dht-table-2", W(huff={("dc", 2): jw.STANDARD[("dc", 0)], ("ac", 2): jw.STANDARD[("ac", 0)]},
                             tsel=[(2, 2)], segments=["app0", "dqt", "sof"]), False),
    ]


RANDOM = _random()
EDGE = _edge()
LAYOUTS = _layouts() + _gray_sampling()
NARROW = _narrow()
RESTARTS = _restarts()
TILE_EDGES = _tile_edges()
SEGMENT_COUNTS = _segment_counts()
REFUSALS = _refusals()
