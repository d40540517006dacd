// faa_jpeg.cuh - arithmetic of the baseline JPEG decoder, shared by the sm_90a kernels (faa_jpeg.cu) and by the host
// build of the CPU tests (tests/emu).
//
// What it reproduces: the reference reads every ImageNet file with torchvision's default_loader (imagenet.py:80,
// `Image.open(f).convert('RGB')`), i.e. Pillow on libjpeg-turbo with libjpeg's default decompression parameters:
//   * Huffman decoding of a sequential scan (ITU T.81 F.2.2), DC prediction, de-zigzag;
//   * JDCT_ISLOW: the integer separable IDCT of Loeffler, Ligtenberg and Moschytz with 13-bit constants, two extra
//     bits of precision between the column and the row pass, descaling with round-half-up, and the range-limit
//     table that adds +128 and clamps (indexed modulo 1024, as libjpeg's table is);
//   * fancy upsampling (triangle filter) of 2x1 and 2x2 subsampled chroma, with its alternating rounding biases
//     (+1/+2 horizontally, +8/+7 in 2-D) and the replication of the edge column / row of the downsampled plane;
//     planes no more than two samples wide are replicated instead, as libjpeg does;
//   * YCbCr -> RGB in 16-bit fixed point (R = Y + 1.402 Cr', G = Y - 0.34414 Cb' - 0.71414 Cr', B = Y + 1.772 Cb').
// Every shift and bias below is part of that specification; tests/test_jpeg_host.py compares the result with Pillow
// byte for byte.
//
// Streams: SOF0 / SOF1, 8-bit, one interleaved scan, 1 component or 3 components in YCbCr with luma sampling 1x1,
// 2x1 or 2x2 and chroma 1x1, any restart interval.  Everything else is refused by parse_jpeg with a reason.
// The decoder reads no byte outside the scan, writes no coefficient outside the image's block grid and reports a
// corrupt or truncated scan in a status word instead of faulting.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define FAA_JHD __host__ __device__ __forceinline__
#else
#define FAA_JHD inline
#endif

namespace faa {

// layout of faa_jpeg_header_t (include/faa_b200.h)
struct JpegHeader {
    int64_t offset, len;              // the file is bytes [offset, offset + len) of the decode call's source buffer
    int64_t scan_off, scan_len;       // entropy-coded data, relative to the file
    int32_t h, w, ncomp, hs, vs, restart, mcu_x, mcu_y;
    int32_t table_at[9];              // file offsets of the table payloads: quant c0..c2, DC c0..c2, AC c0..c2
    int32_t pool[9];                  // the same tables as indices into a JpegTable pool
    int32_t qprec;                    // bit c: component c's quantisation table has 16-bit entries
    int32_t reserved;
};
// layout of faa_jpeg_table_t: a quantisation table (q, natural order) or a Huffman table (bits, vals)
struct JpegTable {
    uint16_t q[64];
    uint8_t bits[16];
    uint8_t vals[256];
};

enum JpegStatus : int32_t {
    JPEG_OK = 0,
    JPEG_TRUNCATED = 1,       // the scan ended (or met a marker) before its last MCU
    JPEG_BAD_CODE = 2,        // a bit pattern that is no code of the Huffman table
    JPEG_BAD_COEF = 4,        // a run that goes past coefficient 63
    JPEG_BAD_RESTART = 8,     // the scan does not hold one restart marker per interval boundary
};

enum JpegParse { JPARSE_OK = 0, JPARSE_UNSUPPORTED = 1, JPARSE_MALFORMED = 2 };

// natural (row-major) index of the k-th coefficient in zigzag order
#define FAA_JPEG_ZIGZAG                                                                                                   \
    {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, \
     21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, \
     47, 55, 62, 63}
static const uint8_t kJpegZigzag[64] = FAA_JPEG_ZIGZAG;
#if defined(__CUDACC__)
static __device__ __constant__ uint8_t kJpegZigzagDev[64] = FAA_JPEG_ZIGZAG;
#endif

FAA_JHD int jpeg_zigzag(int k) {
#if defined(__CUDA_ARCH__)
    return kJpegZigzagDev[k];
#else
    return kJpegZigzag[k];
#endif
}

// ------------------------------------------------------------------------------------------------ header parsing --
FAA_JHD int jpeg_u16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Parses the markers of a whole file (host only; done once per file when a dataset is built).  Returns JPARSE_*;
// *why names the reason of a refusal.  h.offset = 0, h.len = len, pool[] = -1.
inline int parse_jpeg(const uint8_t* b, size_t len, JpegHeader& h, const char** why) {
    memset(&h, 0, sizeof h);
    for (int k = 0; k < 9; ++k) { h.table_at[k] = -1; h.pool[k] = -1; }
    h.len = (int64_t)len;
    *why = "";
#define FAA_BAD(msg) do { *why = msg; return JPARSE_MALFORMED; } while (0)
#define FAA_NO(msg) do { *why = msg; return JPARSE_UNSUPPORTED; } while (0)
    if (len < 4 || b[0] != 0xFF || b[1] != 0xD8) FAA_BAD("no SOI marker: not a JPEG file");
    if (len > 0x7FFFFFFF) FAA_NO("file larger than 2 GiB");
    int32_t dqt_at[4] = {-1, -1, -1, -1}, dqt_prec[4] = {0, 0, 0, 0}, dht_at[2][4];
    for (int c = 0; c < 2; ++c) for (int k = 0; k < 4; ++k) dht_at[c][k] = -1;
    bool jfif = false, adobe = false, have_sof = false, have_scan = false;
    int adobe_transform = -1, sof = 0;
    int comp_id[3] = {0, 0, 0}, comp_h[3] = {0, 0, 0}, comp_v[3] = {0, 0, 0}, comp_q[3] = {0, 0, 0};
    size_t i = 2;
    while (true) {
        if (i >= len) {
            if (have_scan) break;                        // a file cut after its scan: decoded, status reports it
            FAA_BAD("file ends before its scan");
        }
        if (b[i] != 0xFF) FAA_BAD("expected a marker");
        while (i < len && b[i] == 0xFF) ++i;             // fill bytes
        if (i >= len) { if (have_scan) break; FAA_BAD("file ends before its scan"); }
        const int m = b[i++];
        if (m == 0xD9) {                                 // EOI
            if (!have_scan) FAA_BAD("EOI before a scan");
            break;
        }
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;      // TEM, stray RSTn: no payload
        if (m == 0xD8) FAA_BAD("second SOI marker");
        if (i + 2 > len) FAA_BAD("marker segment cut off");
        const int L = jpeg_u16(b + i);
        if (L < 2 || i + (size_t)L > len) FAA_BAD("marker segment length out of range");
        const uint8_t* p = b + i + 2;
        const int n = L - 2;
        const size_t seg_end = i + (size_t)L;
        if (m == 0xC0 || m == 0xC1) {
            if (have_sof) FAA_BAD("second frame header");
            if (n < 6) FAA_BAD("frame header too short");
            if (p[0] != 8) FAA_NO("12-bit (or other non-8-bit) samples");
            h.h = jpeg_u16(p + 1); h.w = jpeg_u16(p + 3);
            const int nf = p[5];
            if (h.h == 0) FAA_NO("height defined by a DNL marker");
            if (h.w == 0) FAA_BAD("zero width");
            if (h.h > 8192 || h.w > 8192) FAA_NO("image larger than 8192 pixels on a side");
            if (nf == 4) FAA_NO("4 components (CMYK or YCCK)");
            if (nf != 1 && nf != 3) FAA_NO("component count other than 1 or 3");
            if (n != 6 + 3 * nf) FAA_BAD("frame header length does not match its components");
            for (int c = 0; c < nf; ++c) {
                comp_id[c] = p[6 + 3 * c]; comp_h[c] = p[7 + 3 * c] >> 4; comp_v[c] = p[7 + 3 * c] & 15;
                comp_q[c] = p[8 + 3 * c];
                if (comp_h[c] < 1 || comp_h[c] > 4 || comp_v[c] < 1 || comp_v[c] > 4) FAA_BAD("sampling factor out of range");
                if (comp_q[c] > 3) FAA_BAD("quantisation table index out of range");
            }
            h.ncomp = nf; sof = m; have_sof = true;
        } else if (m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE) {
            FAA_NO(m == 0xC2 ? "progressive coding" : m == 0xCA ? "progressive arithmetic coding" : "hierarchical coding");
        } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
            FAA_NO("lossless coding");
        } else if (m == 0xC5 || m == 0xCD) {
            FAA_NO("hierarchical coding");
        } else if (m == 0xC9 || m == 0xCC) {
            FAA_NO("arithmetic coding");
        } else if (m == 0xC8) {
            FAA_NO("JPG extension frame");
        } else if (m == 0xDC) {
            FAA_NO("DNL marker");
        } else if (m == 0xC4) {                          // DHT
            int k = 0;
            while (k < n) {
                if (k + 17 > n) FAA_BAD("Huffman table cut off");
                const int tc = p[k] >> 4, th = p[k] & 15;
                if (tc > 1 || th > 3) FAA_BAD("Huffman table class or index out of range");
                int total = 0;
                unsigned code = 0;
                for (int l = 0; l < 16; ++l) {
                    total += p[k + 1 + l];
                    code = (code + p[k + 1 + l]);
                    if (code > (1u << (l + 1))) FAA_BAD("Huffman table with more codes than its lengths allow");
                    code <<= 1;
                }
                if (total > 256 || k + 17 + total > n) FAA_BAD("Huffman table symbol count out of range");
                if (tc == 0)
                    for (int s = 0; s < total; ++s)
                        if (p[k + 17 + s] > 15) FAA_BAD("DC Huffman symbol above 15");
                dht_at[tc][th] = (int32_t)(p + k + 1 - b);
                k += 17 + total;
            }
        } else if (m == 0xDB) {                          // DQT
            int k = 0;
            while (k < n) {
                const int pq = p[k] >> 4, tq = p[k] & 15;
                if (pq > 1 || tq > 3) FAA_BAD("quantisation table precision or index out of range");
                if (k + 1 + 64 * (pq + 1) > n) FAA_BAD("quantisation table cut off");
                dqt_at[tq] = (int32_t)(p + k + 1 - b); dqt_prec[tq] = pq;
                k += 1 + 64 * (pq + 1);
            }
        } else if (m == 0xDD) {                          // DRI
            if (n < 2) FAA_BAD("restart interval segment too short");
            h.restart = jpeg_u16(p);
        } else if (m == 0xE0) {
            if (n >= 14 && p[0] == 'J' && p[1] == 'F' && p[2] == 'I' && p[3] == 'F' && p[4] == 0) jfif = true;
        } else if (m == 0xEE) {
            if (n >= 12 && p[0] == 'A' && p[1] == 'd' && p[2] == 'o' && p[3] == 'b' && p[4] == 'e') {
                adobe = true; adobe_transform = p[11];
            }
        } else if (m == 0xDA) {                          // SOS
            if (have_scan) FAA_NO("more than one scan (multi-scan sequential)");
            if (!have_sof) FAA_BAD("scan before the frame header");
            if (n < 1) FAA_BAD("scan header too short");
            const int ns = p[0];
            if (n != 4 + 2 * ns) FAA_BAD("scan header length does not match its components");
            if (ns != h.ncomp) FAA_NO("a scan without every component (multi-scan sequential)");
            const int max_tab = sof == 0xC0 ? 1 : 3;
            for (int c = 0; c < ns; ++c) {
                if (p[1 + 2 * c] != comp_id[c]) FAA_NO("scan components out of frame order (multi-scan sequential)");
                const int td = p[2 + 2 * c] >> 4, ta = p[2 + 2 * c] & 15;
                if (td > max_tab || ta > max_tab) FAA_BAD("Huffman table index out of range for the frame type");
                if (dht_at[0][td] < 0 || dht_at[1][ta] < 0) FAA_BAD("scan uses an undefined Huffman table");
                if (dqt_at[comp_q[c]] < 0) FAA_BAD("component uses an undefined quantisation table");
                h.table_at[c] = dqt_at[comp_q[c]];
                h.table_at[3 + c] = dht_at[0][td];
                h.table_at[6 + c] = dht_at[1][ta];
                if (dqt_prec[comp_q[c]]) h.qprec |= 1 << c;
            }
            const uint8_t* q = p + 1 + 2 * ns;
            if (q[0] != 0 || q[1] != 63 || q[2] != 0) FAA_BAD("spectral selection / approximation of a sequential scan");
            // entropy-coded data: up to the first marker that is not RSTn (0xFF 0x00 is a stuffed 0xFF)
            size_t s = seg_end, e = s;
            while (e < len) {
                if (b[e] != 0xFF) { ++e; continue; }
                size_t f = e + 1;
                while (f < len && b[f] == 0xFF) ++f;
                if (f >= len) break;
                if (b[f] == 0x00 || (b[f] >= 0xD0 && b[f] <= 0xD7)) { e = f + 1; continue; }
                break;
            }
            if (e > len) e = len;
            h.scan_off = (int64_t)s; h.scan_len = (int64_t)(e - s);
            have_scan = true;
            i = e;
            continue;
        }
        i = seg_end;
    }
    if (h.ncomp == 3) {
        if (!jfif && adobe && adobe_transform == 0) FAA_NO("Adobe-transformed RGB (APP14 transform 0)");
        if (!jfif && !adobe && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B') FAA_NO("RGB components");
        const bool ok = comp_h[1] == 1 && comp_v[1] == 1 && comp_h[2] == 1 && comp_v[2] == 1 &&
                        ((comp_h[0] == 1 && comp_v[0] == 1) || (comp_h[0] == 2 && comp_v[0] == 1) ||
                         (comp_h[0] == 2 && comp_v[0] == 2));
        if (!ok) FAA_NO("sampling factors other than 4:4:4, 4:2:2 (2x1) or 4:2:0 (2x2)");
        h.hs = comp_h[0]; h.vs = comp_v[0];
    } else {
        h.hs = h.vs = 1;                                 // one component: one block per MCU whatever it declares
    }
    h.mcu_x = (h.w + 8 * h.hs - 1) / (8 * h.hs);
    h.mcu_y = (h.h + 8 * h.vs - 1) / (8 * h.vs);
    return JPARSE_OK;
#undef FAA_BAD
#undef FAA_NO
}

// the tables a parsed header refers to, in pool form (unused slots zeroed)
inline void jpeg_tables(const uint8_t* b, const JpegHeader& h, JpegTable out[9]) {
    memset(out, 0, 9 * sizeof(JpegTable));
    for (int c = 0; c < h.ncomp; ++c) {
        const uint8_t* q = b + h.table_at[c];
        for (int k = 0; k < 64; ++k)
            out[c].q[kJpegZigzag[k]] = (h.qprec >> c & 1) ? (uint16_t)jpeg_u16(q + 2 * k) : q[k];
        for (int t = 1; t < 3; ++t) {
            const uint8_t* d = b + h.table_at[3 * t + c];
            int total = 0;
            for (int l = 0; l < 16; ++l) { out[3 * t + c].bits[l] = d[l]; total += d[l]; }
            memcpy(out[3 * t + c].vals, d + 16, (size_t)total);
        }
    }
}

// ------------------------------------------------------------------------------------------------ Huffman tables --
constexpr int kJpegLookBits = 9;
struct JpegHuff {
    uint16_t look[1 << kJpegLookBits];   // (length << 8) | symbol of the code the next 9 bits start with; 0: longer code
    int32_t maxcode[18];                 // [l]: largest code of length l (-1: none); [17] catches every pattern
    int32_t valoff[17];                  // symbol of code c of length l = vals[c + valoff[l]]
    uint8_t vals[256];
};

// maxcode / valoff / vals of a canonical table (ITU T.81 C.2, F.2.2.3)
FAA_JHD void jpeg_huff_codes(const JpegTable& t, JpegHuff& d) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        const int n = t.bits[l - 1];
        d.valoff[l] = k - code;
        code += n; k += n;
        d.maxcode[l] = n ? code - 1 : -1;
        code <<= 1;
    }
    d.maxcode[17] = 0x7FFFFFFF;
    d.valoff[0] = 0;
    d.maxcode[0] = -1;
    for (int s = 0; s < 256; ++s) d.vals[s] = t.vals[s];
}

// lookup entry e of a table whose codes are set
FAA_JHD uint16_t jpeg_huff_look(const JpegHuff& d, int e) {
    for (int l = 1; l <= kJpegLookBits; ++l) {
        const int c = e >> (kJpegLookBits - l);
        if (c <= d.maxcode[l]) return (uint16_t)((l << 8) | d.vals[(c + d.valoff[l]) & 255]);
    }
    return 0;
}

FAA_JHD void jpeg_huff_build(const JpegTable& t, JpegHuff& d) {
    jpeg_huff_codes(t, d);
    for (int e = 0; e < (1 << kJpegLookBits); ++e) d.look[e] = jpeg_huff_look(d, e);
}

// ------------------------------------------------------------------------------------------------ bit reader --
// Bytes of [lo, end) come in through aligned 32-bit loads (byte loads for the words that straddle either bound);
// a stuffed 0xFF 0x00 yields 0xFF; any other marker, or the end, yields zero bits and counts them in `fake`.
struct JpegBits {
    const uint8_t* p;
    const uint8_t* lo;
    const uint8_t* end;
    uintptr_t wa;          // address of the cached word
    uint32_t w;
    uint64_t acc;          // bits, most significant first
    int32_t n;             // bits in acc
    int32_t fake;          // of which the last `fake` were made up past the data
    bool stop;             // met a marker or the end
};

FAA_JHD void jpeg_bits_init(JpegBits& r, const uint8_t* lo, const uint8_t* p, const uint8_t* end) {
    r.p = p; r.lo = lo; r.end = end; r.wa = ~(uintptr_t)0; r.w = 0; r.acc = 0; r.n = 0; r.fake = 0;
    r.stop = p >= end;
}

FAA_JHD uint32_t jpeg_byte_at(JpegBits& r, const uint8_t* q) {
    const uintptr_t a = (uintptr_t)q & ~(uintptr_t)3;
    if (a != r.wa) {
        r.wa = a;
        if (a >= (uintptr_t)r.lo && a + 4 <= (uintptr_t)r.end) {
#if defined(__CUDA_ARCH__)
            r.w = __ldg(reinterpret_cast<const unsigned int*>(a));
#else
            memcpy(&r.w, reinterpret_cast<const void*>(a), 4);
#endif
        } else {
            r.w = 0;
            for (int k = 0; k < 4; ++k)
                if (a + k >= (uintptr_t)r.lo && a + k < (uintptr_t)r.end)
                    r.w |= (uint32_t)(*reinterpret_cast<const uint8_t*>(a + k)) << (8 * k);
        }
    }
    return (r.w >> (8 * ((uintptr_t)q & 3))) & 255u;
}

FAA_JHD void jpeg_fill(JpegBits& r) {
    while (r.n <= 56) {
        uint32_t c = 0;
        if (!r.stop && r.p < r.end) {
            c = jpeg_byte_at(r, r.p);
            if (c != 0xFF) ++r.p;
            else if (r.p + 1 < r.end && jpeg_byte_at(r, r.p + 1) == 0) r.p += 2;
            else { r.stop = true; c = 0; }
        } else {
            r.stop = true;
        }
        if (r.stop) r.fake += 8;
        r.acc |= (uint64_t)c << (56 - r.n);
        r.n += 8;
    }
}

FAA_JHD uint32_t jpeg_get(JpegBits& r, int s) {       // s in 1..16, at least s bits in acc
    const uint32_t v = (uint32_t)(r.acc >> (64 - s));
    r.acc <<= s; r.n -= s;
    return v;
}

FAA_JHD int jpeg_extend(uint32_t v, int s) {           // T.81 F.2.2.1 EXTEND
    return s == 0 ? 0 : (v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v);
}

// next symbol of table d, or -1 for a pattern that is no code; needs at least 16 bits in acc
FAA_JHD int jpeg_decode(JpegBits& r, const JpegHuff& d) {
    const uint32_t e = (uint32_t)(r.acc >> (64 - kJpegLookBits));
    const uint32_t v = d.look[e];
    if (v) { r.acc <<= (v >> 8); r.n -= (int)(v >> 8); return (int)(v & 255); }
    const uint32_t p = (uint32_t)(r.acc >> 48);
    for (int l = kJpegLookBits + 1; l <= 16; ++l) {
        const int c = (int)(p >> (16 - l));
        if (c <= d.maxcode[l]) { r.acc <<= l; r.n -= l; return d.vals[(c + d.valoff[l]) & 255]; }
    }
    return -1;
}

// ------------------------------------------------------------------------------------------------ coefficients --
// Coefficient planes of one image: component c's blocks form a grid of (mcu_x * hc) x (mcu_y * vc) blocks of 64 int16
// (natural order, not dequantised), plane after plane starting at `coef`.
FAA_JHD int64_t jpeg_plane_blocks(const JpegHeader& h, int c) {
    const int hc = c == 0 ? h.hs : 1, vc = c == 0 ? h.vs : 1;
    return (int64_t)h.mcu_x * hc * h.mcu_y * vc;
}
FAA_JHD int64_t jpeg_image_blocks(const JpegHeader& h) {
    int64_t n = 0;
    for (int c = 0; c < h.ncomp; ++c) n += jpeg_plane_blocks(h, c);
    return n;
}
FAA_JHD int jpeg_blocks_per_mcu(const JpegHeader& h) { return h.ncomp == 1 ? 1 : h.hs * h.vs + 2; }
FAA_JHD int64_t jpeg_mcus(const JpegHeader& h) { return (int64_t)h.mcu_x * h.mcu_y; }
FAA_JHD int64_t jpeg_segments(const JpegHeader& h) {
    return h.restart > 0 ? (jpeg_mcus(h) + h.restart - 1) / h.restart : 1;
}

// block index (within the image's coefficient buffer) of block b of MCU m
FAA_JHD int64_t jpeg_block_of(const JpegHeader& h, int64_t m, int b) {
    const int64_t mx = m % h.mcu_x, my = m / h.mcu_x;
    if (h.ncomp == 1) return my * h.mcu_x + mx;
    const int ny = h.hs * h.vs;
    if (b < ny) {
        const int by = b / h.hs, bx = b % h.hs;
        return (my * h.vs + by) * ((int64_t)h.mcu_x * h.hs) + mx * h.hs + bx;
    }
    return jpeg_plane_blocks(h, 0) + (int64_t)(b - ny) * jpeg_mcus(h) + my * h.mcu_x + mx;
}

// Block sink: `scratch` holds the block being decoded (64 int16), `store` moves it to its place in the buffer.
FAA_JHD void jpeg_store_block(int16_t* dst, const int16_t* scratch) {
#if defined(__CUDA_ARCH__)
    const uint4* s = reinterpret_cast<const uint4*>(scratch);
    uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = s[k];
#else
    memcpy(dst, scratch, 128);
#endif
}
FAA_JHD void jpeg_zero_block(int16_t* s) {
#if defined(__CUDA_ARCH__)
    uint4* d = reinterpret_cast<uint4*>(s);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = make_uint4(0, 0, 0, 0);
#else
    memset(s, 0, 128);
#endif
}

// Decodes MCUs [m0, m1) from `data` (the segment's first byte) into coef.  huff[c] / huff[3 + c]: DC / AC tables of
// component c.  On an error the blocks from the failing one to the end of the segment are zeroed.  Returns JpegStatus.
FAA_JHD int jpeg_decode_segment(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* lo, const uint8_t* data,
                                const uint8_t* end, int64_t m0, int64_t m1, int16_t* coef, int16_t* scratch) {
    JpegBits r;
    jpeg_bits_init(r, lo, data, end);
    int pred[3] = {0, 0, 0};
    const int nb = jpeg_blocks_per_mcu(h);
    const int ny = h.ncomp == 1 ? 1 : h.hs * h.vs;
    int status = JPEG_OK;
    int64_t m = m0;
    int b = 0;
    for (; m < m1; ++m) {
        for (b = 0; b < nb; ++b) {
            const int c = b < ny ? 0 : b - ny + 1;
            const JpegHuff& dc = *huff[c];
            const JpegHuff& ac = *huff[3 + c];
            jpeg_zero_block(scratch);
            jpeg_fill(r);
            int s = jpeg_decode(r, dc);
            if (s < 0) { status = JPEG_BAD_CODE; break; }
            if (s) s = jpeg_extend(jpeg_get(r, s), s);
            pred[c] += s;
            scratch[0] = (int16_t)pred[c];
            for (int k = 1; k < 64;) {
                jpeg_fill(r);
                const int rs = jpeg_decode(r, ac);
                if (rs < 0) { status = JPEG_BAD_CODE; break; }
                const int run = rs >> 4, sz = rs & 15;
                if (sz) {
                    k += run;
                    if (k > 63) { status = JPEG_BAD_COEF; break; }
                    scratch[jpeg_zigzag(k)] = (int16_t)jpeg_extend(jpeg_get(r, sz), sz);
                    ++k;
                } else {
                    if (run != 15) break;
                    k += 16;
                    if (k > 64) { status = JPEG_BAD_COEF; break; }
                }
            }
            if (status) break;
            jpeg_store_block(coef + 64 * jpeg_block_of(h, m, b), scratch);
        }
        if (status) break;
        if (r.n < r.fake) { status = JPEG_TRUNCATED; ++m; b = 0; break; }     // this MCU used bits past the data
    }
    if (status) {
        jpeg_zero_block(scratch);
        for (; m < m1; ++m, b = 0)
            for (; b < nb; ++b) jpeg_store_block(coef + 64 * jpeg_block_of(h, m, b), scratch);
    }
    return status;
}

// Restart markers of the scan bytes [from, to) (a marker is 0xFF 0xD0..0xD7; its 0xFF may be the last of the range):
// count them, or with `at` record start (byte after the marker, relative to the scan) of segment first + k for the
// k-th marker, up to segment n_seg - 1.
FAA_JHD int jpeg_markers(JpegBits& r, const uint8_t* scan, int64_t from, int64_t to, int64_t scan_len, int32_t* at,
                         int64_t first, int64_t n_seg) {
    int cnt = 0;
    for (int64_t i = from; i < to; ++i) {
        if (jpeg_byte_at(r, scan + i) != 0xFF || i + 1 >= scan_len) continue;
        const uint32_t c = jpeg_byte_at(r, scan + i + 1);
        if (c >= 0xD0 && c <= 0xD7) {
            if (at && first + cnt < n_seg) at[first + cnt] = (int32_t)(i + 2);
            ++cnt;
        }
    }
    return cnt;
}

// ------------------------------------------------------------------------------------------------ IDCT (islow) --
constexpr int kIdctConstBits = 13, kIdctPass1Bits = 2;
constexpr int32_t FIX_0_298631336 = 2446, FIX_0_390180644 = 3196, FIX_0_541196100 = 4433, FIX_0_765366865 = 6270,
                  FIX_0_899976223 = 7373, FIX_1_175875602 = 9633, FIX_1_501321110 = 12299, FIX_1_847759065 = 15137,
                  FIX_1_961570560 = 16069, FIX_2_053119869 = 16819, FIX_2_562915447 = 20995, FIX_3_072711026 = 25172;

FAA_JHD int32_t jpeg_descale(int32_t x, int n) { return (x + (1 << (n - 1))) >> n; }

// one 1-D pass on 8 values v[0..7] -> o[0..7], descaled by `shift`
FAA_JHD void jpeg_idct_1d(const int32_t v[8], int32_t o[8], int shift) {
    int32_t z2 = v[2], z3 = v[6];
    int32_t z1 = (z2 + z3) * FIX_0_541196100;
    int32_t tmp2 = z1 + z3 * (-FIX_1_847759065);
    int32_t tmp3 = z1 + z2 * FIX_0_765366865;
    int32_t tmp0 = (v[0] + v[4]) * (1 << kIdctConstBits);
    int32_t tmp1 = (v[0] - v[4]) * (1 << kIdctConstBits);
    const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = v[7]; tmp1 = v[5]; tmp2 = v[3]; tmp3 = v[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    int32_t z4 = tmp1 + tmp3;
    const int32_t z5 = (z3 + z4) * FIX_1_175875602;
    tmp0 *= FIX_0_298631336; tmp1 *= FIX_2_053119869; tmp2 *= FIX_3_072711026; tmp3 *= FIX_1_501321110;
    z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    o[0] = jpeg_descale(tmp10 + tmp3, shift); o[7] = jpeg_descale(tmp10 - tmp3, shift);
    o[1] = jpeg_descale(tmp11 + tmp2, shift); o[6] = jpeg_descale(tmp11 - tmp2, shift);
    o[2] = jpeg_descale(tmp12 + tmp1, shift); o[5] = jpeg_descale(tmp12 - tmp1, shift);
    o[3] = jpeg_descale(tmp13 + tmp0, shift); o[4] = jpeg_descale(tmp13 - tmp0, shift);
}

// libjpeg's post-IDCT range limit: +128, clamp to 0..255, the index taken modulo 1024
FAA_JHD uint8_t jpeg_range_limit(int32_t x) {
    const int32_t i = x & 1023;
    return (uint8_t)(i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896);
}

// column pass: column `col` of block `in` (natural order, stride 8) dequantised by q -> workspace column (stride 8)
FAA_JHD void jpeg_idct_col(const int16_t* in, const uint16_t* q, int col, int32_t* ws) {
    int32_t v[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (int32_t)in[8 * k + col] * (int32_t)q[8 * k + col];
    jpeg_idct_1d(v, o, kIdctConstBits - kIdctPass1Bits);
#pragma unroll
    for (int k = 0; k < 8; ++k) ws[8 * k + col] = o[k];
}

// row pass: workspace row `row` -> 8 samples
FAA_JHD void jpeg_idct_row(const int32_t* ws, int row, uint8_t* out) {
    int32_t v[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = ws[8 * row + k];
    jpeg_idct_1d(v, o, kIdctConstBits + kIdctPass1Bits + 3);
#pragma unroll
    for (int k = 0; k < 8; ++k) out[k] = jpeg_range_limit(o[k]);
}

// ------------------------------------------------------------------------------------------------ upsampling + colour --
// a window of a component's sample plane: sample (cx, cy) of the plane is p[(cy - y0) * stride + cx - x0]
struct JpegPlane {
    const uint8_t* p;
    int32_t stride, x0, y0;
    FAA_JHD int operator()(int cx, int cy) const { return p[(cy - y0) * stride + (cx - x0)]; }
};

// Chroma value of output pixel (x, y) from a plane; cw x ch is the plane's downsampled size.
FAA_JHD int jpeg_upsample(const JpegPlane& get, int x, int y, int hs, int vs, int cw, int ch) {
    if (hs == 1) return get(x, y);
    const int i = x >> 1;
    if (cw <= 2) return get(i, vs == 2 ? y >> 1 : y);                 // plain replication
    const int in = (x & 1) ? (i + 1 < cw ? i + 1 : cw - 1) : (i > 0 ? i - 1 : 0);
    if (vs == 1) {
        const int t = 3 * get(i, y) + get(in, y);
        return (x & 1) ? (t + 2) >> 2 : (t + 1) >> 2;
    }
    const int r = y >> 1;
    const int rf = (y & 1) ? (r + 1 < ch ? r + 1 : ch - 1) : (r > 0 ? r - 1 : 0);
    const int s0 = 3 * get(i, r) + get(i, rf), s1 = 3 * get(in, r) + get(in, rf);
    return (x & 1) ? (3 * s0 + s1 + 7) >> 4 : (3 * s0 + s1 + 8) >> 4;
}

FAA_JHD uint8_t jpeg_clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

FAA_JHD void jpeg_ycc_rgb(int y, int cb, int cr, uint8_t* o) {
    const int32_t b = cb - 128, r = cr - 128;
    o[0] = jpeg_clamp255(y + ((91881 * r + 32768) >> 16));
    o[1] = jpeg_clamp255(y + ((-22554 * b + 32768 - 46802 * r) >> 16));
    o[2] = jpeg_clamp255(y + ((116130 * b + 32768) >> 16));
}

// downsampled chroma size
FAA_JHD int jpeg_chroma_w(const JpegHeader& h) { return (h.w + h.hs - 1) / h.hs; }
FAA_JHD int jpeg_chroma_h(const JpegHeader& h) { return (h.h + h.vs - 1) / h.vs; }

// ------------------------------------------------------------------------------------------------ host decode --
// The whole decode of one file on the host, serially, with the functions above: the CPU tests' model of the two
// kernels.  out: h.h * h.w * 3 bytes.  Returns the JpegStatus bits.
inline int jpeg_decode_host(const uint8_t* file, const JpegHeader& h, const JpegTable* tabs, uint8_t* out) {
    static_assert(sizeof(JpegTable) == 400, "table layout");
    JpegHuff huffs[6];
    const JpegHuff* hp[6];
    for (int c = 0; c < h.ncomp; ++c)
        for (int t = 0; t < 2; ++t) { jpeg_huff_build(tabs[3 * (t + 1) + c], huffs[3 * t + c]); hp[3 * t + c] = &huffs[3 * t + c]; }
    for (int c = h.ncomp; c < 3; ++c) { hp[c] = hp[0]; hp[3 + c] = hp[3]; }
    const int64_t nblk = jpeg_image_blocks(h);
    int16_t* coef = new int16_t[(size_t)nblk * 64];
    alignas(16) int16_t scratch[64];
    const uint8_t* scan = file + h.scan_off;
    const uint8_t* end = scan + h.scan_len;
    const int64_t n_seg = jpeg_segments(h), mcus = jpeg_mcus(h);
    int32_t* at = new int32_t[(size_t)n_seg];
    for (int64_t k = 0; k < n_seg; ++k) at[k] = -1;
    at[0] = 0;
    int status = 0;
    if (n_seg > 1) {
        JpegBits r; jpeg_bits_init(r, scan, scan, end);
        if (jpeg_markers(r, scan, 0, h.scan_len, h.scan_len, at, 1, n_seg) != n_seg - 1) status |= JPEG_BAD_RESTART;
    }
    for (int64_t k = 0; k < n_seg; ++k) {
        const int64_t m0 = k * (h.restart > 0 ? h.restart : mcus), m1 = n_seg == 1 ? mcus : (m0 + h.restart < mcus ? m0 + h.restart : mcus);
        const uint8_t* p = at[k] < 0 ? end : scan + at[k];
        status |= jpeg_decode_segment(h, hp, scan, p, end, m0, m1, coef, scratch);
    }
    // planes of samples
    uint8_t* planes[3] = {nullptr, nullptr, nullptr};
    int pw[3], ph[3];
    int64_t base = 0;
    for (int c = 0; c < h.ncomp; ++c) {
        const int bw = h.mcu_x * (c == 0 ? h.hs : 1), bh = h.mcu_y * (c == 0 ? h.vs : 1);
        pw[c] = bw * 8; ph[c] = bh * 8;
        planes[c] = new uint8_t[(size_t)pw[c] * ph[c]];
        for (int by = 0; by < bh; ++by)
            for (int bx = 0; bx < bw; ++bx) {
                int32_t ws[64];
                const int16_t* blk = coef + 64 * (base + (int64_t)by * bw + bx);
                for (int col = 0; col < 8; ++col) jpeg_idct_col(blk, tabs[c].q, col, ws);
                for (int row = 0; row < 8; ++row) jpeg_idct_row(ws, row, planes[c] + (size_t)(by * 8 + row) * pw[c] + bx * 8);
            }
        base += (int64_t)bw * bh;
    }
    const int cw = jpeg_chroma_w(h), ch = jpeg_chroma_h(h);
    for (int y = 0; y < h.h; ++y)
        for (int x = 0; x < h.w; ++x) {
            uint8_t* o = out + ((size_t)y * h.w + x) * 3;
            const int Y = planes[0][(size_t)y * pw[0] + x];
            if (h.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; continue; }
            const int cb = jpeg_upsample(JpegPlane{planes[1], pw[1], 0, 0}, x, y, h.hs, h.vs, cw, ch);
            const int cr = jpeg_upsample(JpegPlane{planes[2], pw[1], 0, 0}, x, y, h.hs, h.vs, cw, ch);
            jpeg_ycc_rgb(Y, cb, cr, o);
        }
    for (int c = 0; c < 3; ++c) delete[] planes[c];
    delete[] at;
    delete[] coef;
    return status;
}

}  // namespace faa
