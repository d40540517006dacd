"""A small progressive JPEG writer for the progressive decoder tests, TEST INFRASTRUCTURE ONLY.

It writes given quantised coefficient blocks under a given scan script, so a test reaches what Pillow's one script
never does: non-interleaved and partially interleaved DC scans, single-coefficient bands, several refinement levels,
long EOB runs (up to 32767) across block rows and restart intervals, a restart interval, Huffman table or quantisation
table redefined between scans.  The entropy coding follows libjpeg's progressive encoder (jcphuff.c: EOB runs, ZRL, the
correction bits of a refinement buffered behind the EOB run they belong to); the Huffman tables are optimal for each
scan and written in a DHT before it.  Blocks use ``jpeg_writer``'s layout (component c's natural-order
coefficients on ``block_grid``); the oracle is Pillow decoding the bytes written."""
import numpy as np

from jpeg_writer import ZIGZAG, _Bits, _seg, _u16, block_grid, codes, optimal


def extent(h, w, sampling, c):
    """(rows, cols) of the blocks a scan of component c alone walks: ceil(comp_h / 8) x ceil(comp_w / 8)"""
    hm, vm = max(s[0] for s in sampling), max(s[1] for s in sampling)
    cw, ch = -(-w * sampling[c][0] // hm), -(-h * sampling[c][1] // vm)
    return -(-ch // 8), -(-cw // 8)


def _units(h, w, sampling, comps):
    """[[(c, y, x) of each block of the unit]] in scan order"""
    if len(comps) == 1:
        c = comps[0]
        rows, cols = extent(h, w, sampling, c)
        return [[(c, y, x)] for y in range(rows) for x in range(cols)]
    hm, vm = max(s[0] for s in sampling), max(s[1] for s in sampling)
    mx, my = -(-w // (8 * hm)), -(-h // (8 * vm))
    if len(sampling) == 1:
        mx, my = -(-w // 8), -(-h // 8)
    return [[(c, y * sampling[c][1] + v, x * sampling[c][0] + u) for c in comps for v in range(sampling[c][1])
             for u in range(sampling[c][0])] for y in range(my) for x in range(mx)]


class _Ops:
    """the symbols and raw bits of one scan, in order, and its restart boundaries"""

    def __init__(self):
        self.ops = []
        self.eobrun = 0
        self.be = []                     # correction bits buffered behind the EOB run (refinement)

    def sym(self, key, s):
        self.ops.append(("sym", key, s))

    def bits(self, v, n):
        if n:
            self.ops.append(("bits", v, n))

    def emit_eobrun(self):
        if self.eobrun > 0:
            r = self.eobrun.bit_length() - 1
            self.sym(("ac", 0), r << 4)
            self.bits(self.eobrun - (1 << r), r)
            self.eobrun = 0
            for b in self.be:
                self.bits(b, 1)
            self.be = []


def _scan_ops(blocks, units, scan, restart):
    ss, se, ah, al = scan["ss"], scan["se"], scan["ah"], scan["al"]
    zz = {c: np.asarray(b, np.int64).reshape(-1, 64)[:, ZIGZAG].reshape(*np.shape(b)[:2], 64)
          for c, b in enumerate(blocks)}
    o = _Ops()
    comps = scan["comps"]
    pred = {c: 0 for c in comps}
    for u, unit in enumerate(units):
        if restart and u and u % restart == 0:
            o.emit_eobrun()
            o.ops.append(("rst",))
            pred = {c: 0 for c in comps}
        for c, y, x in unit:
            blk = zz[c][y, x]
            if ss == 0:
                if ah == 0:
                    t = int(blk[0]) >> al
                    d = t - pred[c]
                    pred[c] = t
                    n = abs(d).bit_length()
                    o.sym(("dc", min(c, 1)), n)
                    o.bits(d if d >= 0 else d + (1 << n) - 1, n)
                else:
                    o.bits((int(blk[0]) >> al) & 1, 1)
            elif ah == 0:                                 # AC first (encode_mcu_AC_first)
                r = 0
                for k in range(ss, se + 1):
                    v = int(blk[k])
                    m = abs(v) >> al
                    if m == 0:
                        r += 1
                        continue
                    o.emit_eobrun()
                    while r > 15:
                        o.sym(("ac", 0), 0xF0)
                        r -= 16
                    n = m.bit_length()
                    o.sym(("ac", 0), (r << 4) | n)
                    o.bits(m if v >= 0 else ~m, n)
                    r = 0
                if r > 0:
                    o.eobrun += 1
                    if o.eobrun == 0x7FFF:
                        o.emit_eobrun()
            else:                                         # AC refinement (encode_mcu_AC_refine)
                absv = [abs(int(blk[k])) >> al for k in range(64)]
                eob = max([k for k in range(ss, se + 1) if absv[k] == 1], default=0)
                r, br = 0, []
                for k in range(ss, se + 1):
                    t = absv[k]
                    if t == 0:
                        r += 1
                        continue
                    while r > 15 and k <= eob:
                        o.emit_eobrun()
                        o.sym(("ac", 0), 0xF0)
                        r -= 16
                        for b in br:
                            o.bits(b, 1)
                        br = []
                    if t > 1:
                        br.append(t & 1)
                        continue
                    o.emit_eobrun()
                    o.sym(("ac", 0), (r << 4) | 1)
                    o.bits(0 if int(blk[k]) < 0 else 1, 1)
                    for b in br:
                        o.bits(b, 1)
                    br, r = [], 0
                if r > 0 or br:
                    o.eobrun += 1
                    o.be += br
                    if o.eobrun == 0x7FFF or len(o.be) > 1000 - 64 + 1:
                        o.emit_eobrun()
    o.emit_eobrun()
    return o.ops


def write(h, w, blocks, quant, scans, *, sampling=None, qsel=None, info=None):
    """JPEG bytes of a progressive file (SOF2).

    blocks   component c's int [rows, cols, 64] quantised coefficients, natural order, on ``jpeg_writer.block_grid``
             (the AC of blocks outside the component's own ``extent`` are never written)
    quant    {table id: 64 entries, natural order}, 8-bit.  qsel: per component table id (default 0, then 1)
    scans    dicts (pass them through ``script``): comps (frame indices), ss, se, ah, al; optional restart (units
             per interval: a DRI before the scan, in force from there on) and dqt ({table id: table} written before
             the scan)
    info     a dict that gets the scan ranges [(offset, length)]"""
    nc = len(blocks)
    sampling = [tuple(s) for s in (sampling or [(1, 1)] * nc)]
    qsel = list(qsel if qsel is not None else [0] + [1] * (nc - 1))
    for c in range(nc):
        assert tuple(np.shape(blocks[c])[:2]) == block_grid(h, w, sampling, c)

    def dqt(tid, q):
        q = np.asarray(q, np.int64).reshape(64)[ZIGZAG]
        return _seg(0xDB, bytes([tid]) + bytes(int(v) for v in q))

    out = bytearray(b"\xff\xd8") + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in sorted(quant):
        out += dqt(t, quant[t])
    out += _seg(0xC2, bytes([8]) + _u16(h) + _u16(w) + bytes([nc]) +
                b"".join(bytes([c + 1, sampling[c][0] << 4 | sampling[c][1], qsel[c]]) for c in range(nc)))
    ranges = []
    for sc in scans:
        for t, q in (sc.get("dqt") or {}).items():
            out += dqt(t, q)
        restart = sc.get("restart")
        if restart is not None:
            out += _seg(0xDD, _u16(restart))
        units = _units(h, w, sampling, sc["comps"])
        ops = _scan_ops(blocks, units, sc, sc.get("_restart_in_force", 0))
        freq = {}
        for op in ops:
            if op[0] == "sym":
                freq.setdefault(op[1], {}).setdefault(op[2], 0)
                freq[op[1]][op[2]] += 1
        tables = {k: optimal(f) for k, f in sorted(freq.items())}
        for (cls, tid), (bits, vals) in sorted(tables.items()):
            out += _seg(0xC4, bytes([(0 if cls == "dc" else 1) << 4 | tid]) + bytes(bits) + bytes(vals))
        cm = {k: codes(t) for k, t in tables.items()}
        out += _seg(0xDA, bytes([len(sc["comps"])]) +
                    b"".join(bytes([c + 1, min(c, 1) << 4]) for c in sc["comps"]) +
                    bytes([sc["ss"], sc["se"], sc["ah"] << 4 | sc["al"]]))
        start = len(out)
        bw, k = _Bits(), 0
        for op in ops:
            if op[0] == "sym":
                code, n = cm[op[1]][op[2]]
                bw.put(code, n)
            elif op[0] == "bits":
                bw.put(op[1], op[2])
            else:
                bw.flush()
                out += bw.out + bytes([0xFF, 0xD0 + k % 8])
                bw, k = _Bits(), k + 1
        bw.flush()
        out += bw.out
        ranges.append((start, len(out) - start))
    out += b"\xff\xd9"
    if info is not None:
        info["scans"] = ranges
    return bytes(out)


def script(scans, restart=0):
    """the scans with the restart interval in force at each (a scan with ``restart`` changes it from there on)"""
    out, cur = [], restart
    for sc in scans:
        sc = dict(sc)
        if "restart" in sc:
            cur = sc["restart"]
        sc["_restart_in_force"] = cur
        out.append(sc)
    return out
