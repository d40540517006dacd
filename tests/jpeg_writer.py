"""A small baseline JPEG writer for the decoder tests, TEST INFRASTRUCTURE ONLY.

It writes given quantised coefficient blocks, so a test controls what no encoder it could call lets it choose: the
quantisation tables and their precision (8-bit DQT with SOF0, or 16-bit with SOF1), which tables each component uses,
the Huffman tables themselves (including ones whose most frequent symbols have codes of 10 to 16 bits), the restart
interval, fill bytes before any marker (enough to put a chosen restart marker's 0xFF at a chosen scan offset), stray
bytes between segments, the segment layout (tables merged into one segment or split, APPn and COM segments), the
component ids and the declared sampling factors.  It does not try to match libjpeg's encoder: the oracle is Pillow
decoding the bytes written.

Coefficients come from pixels (``coefs_from_plane``: a float DCT and a chosen table) or are given directly.  Keep every
dequantised coefficient within what a forward DCT of 8-bit samples can produce (``in_range``): beyond it Pillow's SIMD
IDCT wraps 16-bit lanes, which the decoder does not model."""
import heapq
import math

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])      # natural index of the k-th coefficient in zigzag order
AC_LIMIT, DC_LIMIT = 1023, 1024                                  # |coef * q| a forward DCT of 8-bit samples reaches


def limits(q):
    """largest |coefficient| per natural position that stays in range under quantisation table q (64, natural order)"""
    q = np.asarray(q, np.int64).reshape(64)
    lim = AC_LIMIT // q
    lim[0] = DC_LIMIT // q[0]
    return lim


def in_range(blocks, q):
    return bool((np.abs(np.asarray(blocks, np.int64)) <= limits(q)).all())


def _dct_matrix():
    k = np.arange(8)
    m = np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16) * 0.5
    m[0] /= math.sqrt(2)
    return m


def coefs_from_plane(plane, q, grid):
    """int16 [gy, gx, 64] quantised coefficients (natural order) of a uint8 sample plane: the plane is edge-replicated
    to the block grid (gy, gx), level-shifted, float-DCT'd and divided by q with rounding, then clipped into range"""
    gy, gx = grid
    p = np.asarray(plane, np.float64)
    p = np.pad(p, ((0, max(0, 8 * gy - p.shape[0])), (0, max(0, 8 * gx - p.shape[1]))), mode="edge")[:8 * gy, :8 * gx]
    m = _dct_matrix()
    blocks = p.reshape(gy, 8, gx, 8).transpose(0, 2, 1, 3) - 128.0
    f = np.einsum("ux,abxy,vy->abuv", m, blocks, m).reshape(gy, gx, 64)
    qq = np.asarray(q, np.float64).reshape(64)
    c = np.round(f / qq)
    lim = limits(q)
    return np.clip(c, -lim, lim).astype(np.int16)


def random_blocks(rng, shape, q, density=0.3):
    """random in-range blocks [*shape, 64]: sparse AC of every magnitude up to the limit, DC anywhere in range"""
    lim = limits(q)
    n = int(np.prod(shape))
    mag = np.rint(lim[None, :] * rng.random((n, 64)) ** rng.uniform(1, 4, (n, 1)))
    sign = rng.choice([-1, 1], (n, 64))
    keep = rng.random((n, 64)) < density
    keep[:, 0] = True
    return (mag * sign * keep).astype(np.int16).reshape(*shape, 64)


# ------------------------------------------------------------------------------------------------ Huffman tables --
def canonical(lengths):
    """(bits[16], vals) of a canonical table from {symbol: code length}, symbols of a length in increasing order"""
    bits = [0] * 16
    vals = []
    for l in range(1, 17):
        syms = sorted(s for s, n in lengths.items() if n == l)
        bits[l - 1] = len(syms)
        vals += syms
    return bits, vals


def optimal(freq):
    """(bits, vals) of a Huffman table for {symbol: count}, lengths limited to 16 and the all-ones code left unused
    (T.81 K.2: a reserved pseudo-symbol takes it)"""
    freq = {s: max(int(n), 1) for s, n in freq.items()}
    items = [(n, i, [s]) for i, (s, n) in enumerate(sorted(freq.items()))] + [(1, -1, [None])]
    heapq.heapify(items)
    depth = {s: 0 for s in list(freq) + [None]}
    k = len(items)
    while len(items) > 1:
        n1, _, a = heapq.heappop(items)
        n2, _, b = heapq.heappop(items)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(items, (n1 + n2, k, a + b))
        k += 1
    count = [0] * 64
    for d in depth.values():
        count[d] += 1
    for l in range(63, 16, -1):                       # K.2 Figure K.3 (Adjust_BITS)
        while count[l] > 0:
            j = l - 2
            while count[j] == 0:
                j -= 1
            count[l] -= 2
            count[l - 1] += 1
            count[j + 1] += 2
            count[j] -= 1
    l = 16
    while count[l] == 0:
        l -= 1
    count[l] -= 1                                     # the pseudo-symbol: the longest, last code
    order = sorted(freq, key=lambda s: (-freq[s], s))
    lengths, at = {}, 0
    for l in range(1, 17):
        for _ in range(count[l]):
            lengths[order[at]] = l
            at += 1
    return canonical(lengths)


def long_codes(freq, shortest=10):
    """(bits, vals): every symbol of {symbol: count} gets a code of `shortest` to 16 bits, the most frequent ones the
    longest, so a decoder with a 9-bit lookup takes its slow path for them"""
    order = sorted(freq, key=lambda s: (-freq[s], s))
    span = 16 - shortest + 1
    lengths = {s: 16 - (i * span // max(len(order), 1)) for i, s in enumerate(order)}
    return canonical(lengths)


# the tables of ITU T.81 K.3, which a decoder uses for a scan whose table 0 or 1 no DHT defines
_AC0 = bytes.fromhex("01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a"
                     "3435363738393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a9293"
                     "9495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7"
                     "e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC1 = bytes.fromhex("000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728"
                     "292a35363738393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a"
                     "92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5"
                     "e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STANDARD = {("dc", 0): ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
            ("dc", 1): ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
            ("ac", 0): ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125], list(_AC0)),
            ("ac", 1): ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119], list(_AC1))}


def all_ones(freq):
    """(bits, vals) that give the symbols of {symbol: count} codes from a table using every code of its longest
    length, the all-ones one included (which T.81 forbids): one 1-bit code and 128 8-bit ones, spare symbols added"""
    syms = sorted(freq)
    assert len(syms) <= 129
    spare = [s for s in range(256) if s not in freq][:129 - len(syms)]
    lengths = {s: 8 for s in syms[1:] + spare}
    lengths[syms[0]] = 1
    return canonical(lengths)


def codes(table):
    """{symbol: (code, length)} of a (bits, vals) table"""
    bits, vals = table
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


# ------------------------------------------------------------------------------------------------ scan --
def _category(v):
    return int(abs(int(v))).bit_length()


def _block_symbols(zz, pred):
    """[(is_ac, symbol, extra bits, n extra)] of one block in zigzag order, DC as a difference from pred"""
    out = []
    zz = zz.tolist()
    d = zz[0] - pred
    s = _category(d)
    out.append((0, s, d if d >= 0 else d + (1 << s) - 1, s))
    last = 63
    while last > 0 and zz[last] == 0:
        last -= 1
    run = 0
    for k in range(1, last + 1):
        v = zz[k]
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append((1, 0xF0, 0, 0))
            run -= 16
        s = _category(v)
        out.append((1, (run << 4) | s, v if v >= 0 else v + (1 << s) - 1, s))
        run = 0
    if last < 63:
        out.append((1, 0x00, 0, 0))
    return out


class _Bits:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, v, n):
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 255
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def block_grid(h, w, sampling, c):
    """(rows, cols) of component c's block grid in a scan: one block per MCU for a single component, else
    mcu_y * v x mcu_x * h"""
    if len(sampling) == 1:
        return -(-h // 8), -(-w // 8)
    hm, vm = max(s[0] for s in sampling), max(s[1] for s in sampling)
    mx, my = -(-w // (8 * hm)), -(-h // (8 * vm))
    return my * sampling[c][1], mx * sampling[c][0]


def _u16(v):
    return bytes([(v >> 8) & 255, v & 255])


def _seg(marker, payload):
    return bytes([0xFF, marker]) + _u16(len(payload) + 2) + bytes(payload)


def write(h, w, blocks, quant, *, sampling=None, qsel=None, ids=None, qbits=8, sof=None, huff=None, tsel=None,
          restart=0, merge_dqt=False, merge_dht=False, jfif=True, segments=None, before=None, rst_fill=None,
          trailing=b"", eoi=True, info=None):
    """JPEG bytes of one interleaved baseline scan.

    blocks      component c's int [rows, cols, 64] quantised coefficients, natural order, on ``block_grid``
    quant       {table id: 64 entries, natural order}; written 8-bit (qbits=8, SOF0) or 16-bit (qbits=16, SOF1)
    sampling    per component (h, v); default 1x1.  qsel: per component table id (default 0 for component 0, 1 else)
    ids         component ids (default 1, 2, 3).  sof: frame marker (default 0xC0, or 0xC1 for 16-bit tables)
    huff        {("dc" | "ac", id): (bits, vals)}; a missing table is built from the scan's statistics (``optimal``),
                a callable value is called with those statistics ({symbol: count}).  tsel: per component (dc, ac) ids
    restart     MCUs per restart interval (0: none).  rst_fill: {k: n} n extra 0xFF before the k-th RST marker
    merge_dqt / merge_dht   all tables in one segment each, else one segment per table
    segments    header layout after SOI: a list of "app0", "dqt", "dht", "sof", "dri", or (marker, payload) for
                any other segment (APPn, COM); default app0 (if jfif), dqt, sof, dht, dri
    before      {segment index in that list, or "sos" / "eoi": bytes} written before that marker (fill or stray bytes)
    info        a dict that gets scan_off (file offset of the scan) and rst_ff (scan offset of the 0xFF just
                before each RST marker code)"""
    nc = len(blocks)
    sampling = [tuple(s) for s in (sampling or [(1, 1)] * nc)]
    qsel = list(qsel if qsel is not None else [0] + [1] * (nc - 1))
    ids = list(ids if ids is not None else range(1, nc + 1))
    tsel = list(tsel if tsel is not None else [(0, 0)] + [(1, 1)] * (nc - 1))
    sof = sof if sof is not None else (0xC1 if qbits == 16 else 0xC0)
    for c in range(nc):
        assert tuple(np.shape(blocks[c])[:2]) == block_grid(h, w, sampling, c), (c, np.shape(blocks[c]))
    zz = [np.asarray(b, np.int64).reshape(-1, 64)[:, ZIGZAG].reshape(*np.shape(b)[:2], 64) for b in blocks]
    # MCU order of (component, block) and the symbols of each restart segment
    if nc == 1:
        rows, cols = block_grid(h, w, sampling, 0)
        mcus = [[(0, y, x)] for y in range(rows) for x in range(cols)]
    else:
        hm, vm = max(s[0] for s in sampling), max(s[1] for s in sampling)
        mx, my = -(-w // (8 * hm)), -(-h // (8 * vm))
        mcus = [[(c, y * sampling[c][1] + v, x * sampling[c][0] + u) for c in range(nc) for v in range(sampling[c][1])
                 for u in range(sampling[c][0])] for y in range(my) for x in range(mx)]
    per = restart if restart > 0 else len(mcus)
    segs = []
    for m0 in range(0, len(mcus), per):
        pred = [0] * nc
        syms = []
        for mcu in mcus[m0:m0 + per]:
            for c, y, x in mcu:
                for is_ac, s, v, n in _block_symbols(zz[c][y, x], pred[c]):
                    syms.append((c, is_ac, s, v, n))
                pred[c] = int(zz[c][y, x, 0])
        segs.append(syms)
    freq = {}
    for syms in segs:
        for c, is_ac, s, _, _ in syms:
            key = ("ac" if is_ac else "dc", tsel[c][is_ac])
            freq.setdefault(key, {}).setdefault(s, 0)
            freq[key][s] += 1
    tables = {}
    for key, f in sorted(freq.items()):
        t = (huff or {}).get(key)
        tables[key] = t(f) if callable(t) else (t if t is not None else optimal(f))
    for key, t in (huff or {}).items():
        if key not in tables and not callable(t):
            tables[key] = t
    cmap = {key: codes(t) for key, t in tables.items()}
    # entropy-coded data
    scan = bytearray()
    rst_ff = []
    for k, syms in enumerate(segs):
        if k:
            scan += b"\xff" * (rst_fill or {}).get(k - 1, 0)
            rst_ff.append(len(scan))
            scan += bytes([0xFF, 0xD0 + (k - 1) % 8])
        bw = _Bits()
        for c, is_ac, s, v, n in syms:
            code, l = cmap[("ac" if is_ac else "dc", tsel[c][is_ac])][s]
            bw.put((code << n) | v, l + n)
        bw.flush()
        scan += bw.out
    # header segments
    prec = 1 if qbits == 16 else 0

    def dqt_payload(tid):
        q = np.asarray(quant[tid], np.int64).reshape(64)[ZIGZAG]
        return bytes([(prec << 4) | tid]) + (b"".join(_u16(int(v)) for v in q) if prec else bytes(int(v) for v in q))

    def dht_payload(key):
        bits, vals = tables[key]
        return bytes([(0 if key[0] == "dc" else 1) << 4 | key[1]]) + bytes(bits) + bytes(vals)

    dqt = [_seg(0xDB, b"".join(dqt_payload(t) for t in sorted(quant)))] if merge_dqt else \
        [_seg(0xDB, dqt_payload(t)) for t in sorted(quant)]
    keys = sorted(tables)
    dht = [_seg(0xC4, b"".join(dht_payload(k) for k in keys))] if merge_dht else [_seg(0xC4, dht_payload(k)) for k in keys]
    sof_seg = _seg(sof, bytes([8]) + _u16(h) + _u16(w) + bytes([nc]) +
                   b"".join(bytes([ids[c], sampling[c][0] << 4 | sampling[c][1], qsel[c]]) for c in range(nc)))
    app0 = _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    dri = _seg(0xDD, _u16(restart)) if restart else b""
    parts = {"app0": app0, "dqt": b"".join(dqt), "dht": b"".join(dht), "sof": sof_seg, "dri": dri}
    layout = segments if segments is not None else (["app0"] if jfif else []) + ["dqt", "sof", "dht", "dri"]
    before = before or {}
    out = bytearray(b"\xff\xd8")
    for i, s in enumerate(layout):
        out += before.get(i, b"")
        out += parts[s] if isinstance(s, str) else _seg(s[0], s[1])
    out += before.get("sos", b"")
    out += _seg(0xDA, bytes([nc]) + b"".join(bytes([ids[c], tsel[c][0] << 4 | tsel[c][1]]) for c in range(nc)) +
                b"\x00\x3f\x00")
    if info is not None:
        info["scan_off"] = len(out)
        info["rst_ff"] = rst_ff
        info["scan_len"] = len(scan)
    out += scan
    out += before.get("eoi", b"")
    if eoi:
        out += b"\xff\xd9"
    out += trailing
    return bytes(out)
