// faa_jpeg.cuh - arithmetic of the baseline JPEG decoder, shared by the sm_90a kernels (faa_jpeg.cu) and by the host
// build of the CPU tests (tests/emu).
//
// What it reproduces: the reference reads every ImageNet file with torchvision's default_loader (imagenet.py:80,
// `Image.open(f).convert('RGB')`), i.e. Pillow on libjpeg-turbo with libjpeg's default decompression parameters:
//   * Huffman decoding of a sequential scan (ITU T.81 F.2.2), DC prediction, de-zigzag;
//   * JDCT_ISLOW: the integer separable IDCT of Loeffler, Ligtenberg and Moschytz with 13-bit constants, two extra
//     bits of precision between the column and the row pass, descaling with round-half-up, and the range limit
//     that adds +128 and saturates to 0..255, as libjpeg-turbo's SIMD islow IDCT on x86-64 does (libjpeg's C table
//     wraps modulo 1024 instead; the two differ only on IDCT outputs outside [-512, 511]);
//   * fancy upsampling (triangle filter) of 2x1 and 2x2 subsampled chroma, with its alternating rounding biases
//     (+1/+2 horizontally, +8/+7 in 2-D) and the replication of the edge column / row of the downsampled plane;
//     planes no more than two samples wide are replicated instead, as libjpeg does;
//   * YCbCr -> RGB in 16-bit fixed point (R = Y + 1.402 Cr', G = Y - 0.34414 Cb' - 0.71414 Cr', B = Y + 1.772 Cb').
// Every shift and bias below is part of that specification; tests/test_jpeg_host.py and
// tests/test_jpeg_streams_host.py compare the result with Pillow byte for byte.  It is exact for every stream whose
// dequantised coefficients stay within what a forward DCT of 8-bit samples can produce (|coef * q| <= 1023 for AC,
// <= 1024 for DC); beyond that libjpeg-turbo's SIMD IDCT wraps and saturates 16-bit lanes, which is not modelled.
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
                                      // (a Huffman table no DHT defines: kJpegStdAt - k, standard table k)
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

// The Huffman tables of ITU T.81 K.3 (BITS, then HUFFVAL): DC 0, DC 1, AC 0, AC 1.  A scan whose table 0 or 1 no DHT
// defines uses these, as libjpeg-turbo does (Motion-JPEG frames leave them out); its header's table_at then holds
// kJpegStdAt - k for table k instead of a file offset.
constexpr int32_t kJpegStdAt = -2;
static const uint8_t kJpegStdHuff[4][16 + 162] = {
    {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11},
    {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11},
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125,
     0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119,
     0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// the standard table a Huffman table_at entry names, or nullptr when it is a file offset (or unset)
inline const uint8_t* jpeg_std_huff(int32_t at) {
    return at <= kJpegStdAt && at > kJpegStdAt - 4 ? kJpegStdHuff[kJpegStdAt - at] : nullptr;
}

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
    int adobe_transform = -1;
    int comp_id[3] = {0, 0, 0}, comp_h[3] = {0, 0, 0}, comp_v[3] = {0, 0, 0}, comp_q[3] = {0, 0, 0};
    size_t i = 2;
    while (true) {
        if (i >= len) {
            if (have_scan) break;                        // a file cut after its scan: decoded, status reports it
            FAA_BAD("file ends before its scan");
        }
        while (i < len && b[i] != 0xFF) ++i;             // stray bytes before a marker: skipped, as libjpeg does
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
            h.ncomp = nf; have_sof = true;
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
                    // (>=: a table may not use the all-ones code of a length, T.81 C.2; libjpeg refuses it too)
                    if (code >= (1u << (l + 1))) FAA_BAD("Huffman table with more codes than its lengths allow");
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
            for (int c = 0; c < ns; ++c) {
                if (p[1 + 2 * c] != comp_id[c]) FAA_NO("scan components out of frame order (multi-scan sequential)");
                const int td = p[2 + 2 * c] >> 4, ta = p[2 + 2 * c] & 15;
                // (tables 2 and 3 in a baseline frame too: libjpeg decodes them whatever the SOF says)
                if (td > 3 || ta > 3) FAA_BAD("Huffman table index out of range");
                const int32_t dc_at = dht_at[0][td] >= 0 ? dht_at[0][td] : td < 2 ? kJpegStdAt - td : -1;
                const int32_t ac_at = dht_at[1][ta] >= 0 ? dht_at[1][ta] : ta < 2 ? kJpegStdAt - 2 - ta : -1;
                if (dc_at == -1 || ac_at == -1) FAA_BAD("scan uses an undefined Huffman table");
                if (dqt_at[comp_q[c]] < 0) FAA_BAD("component uses an undefined quantisation table");
                h.table_at[c] = dqt_at[comp_q[c]];
                h.table_at[3 + c] = dc_at;
                h.table_at[6 + c] = ac_at;
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
            const uint8_t* std_table = jpeg_std_huff(h.table_at[3 * t + c]);
            const uint8_t* d = std_table ? std_table : b + h.table_at[3 * t + c];
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

// ------------------------------------------------------------------------------------------------ sync points --
// The decoder's state at an MCU boundary (layout of faa_jpeg_sync_t): MCU `mcu` is the next to decode, its first bit is
// bit `bit` (0 = most significant) of the data byte at scan offset `byte` (a stuffed 0xFF 0x00 is one data byte, at the
// 0xFF's offset), and pred[] are the DC predictors.  A scan index is a list of such points; a segment started at one
// decodes as the serial decoder does from that MCU on.
struct JpegSync {
    int32_t mcu;
    int32_t byte;
    int16_t bit;
    int16_t pred[3];
};

constexpr int kJpegIndexMaxParts = 128;        // segments of an indexed scan: the entropy kernel's threads
constexpr int kJpegIndexBytesPerPart = 1024;

// The placement rule of a scan index, the one place it is stated.  A scan of scan_len bytes without restart markers is
// cut into P = min(128, scan_len / 1024) segments of about equal bytes (bytes are the work, not MCUs); point k (1 <= k
// < P) is the first MCU boundary whose start byte is >= k * scan_len / P, and points that coincide are dropped.  Below
// two segments, and for files with a restart interval, there is no index: jpeg_index_parts returns 0.
FAA_JHD int jpeg_index_parts(const JpegHeader& h) {
    if (h.restart > 0) return 0;
    const int64_t p = h.scan_len / kJpegIndexBytesPerPart;
    return p < 2 ? 0 : p > kJpegIndexMaxParts ? kJpegIndexMaxParts : (int)p;
}
// most points an index of this file holds
FAA_JHD int jpeg_index_capacity(const JpegHeader& h) { const int p = jpeg_index_parts(h); return p ? p - 1 : 0; }
FAA_JHD int64_t jpeg_index_threshold(const JpegHeader& h, int parts, int k) { return (int64_t)k * h.scan_len / parts; }

// Whether an index can be used as it stands: a file the rule gives points to, at most 127 points, MCUs strictly
// increasing inside (0, mcus), bytes inside the scan, bits 0..7.  Anything else decodes serially.
FAA_JHD bool jpeg_index_point_ok(const JpegHeader& h, const JpegSync& s, int32_t prev_mcu) {
    return s.mcu > prev_mcu && s.mcu > 0 && (int64_t)s.mcu < (int64_t)h.mcu_x * h.mcu_y && s.byte >= 0 &&
           (int64_t)s.byte < h.scan_len && s.bit >= 0 && s.bit <= 7;
}
FAA_JHD bool jpeg_index_count_ok(const JpegHeader& h, int64_t n) {
    return n > 0 && n < kJpegIndexMaxParts && jpeg_index_parts(h) > 0;
}

// the end state of one segment equals the point the next one starts at (its MCU is implied)
FAA_JHD bool jpeg_sync_same(const JpegSync& a, const JpegSync& b) {
    return a.byte == b.byte && a.bit == b.bit && a.pred[0] == b.pred[0] && a.pred[1] == b.pred[1] && a.pred[2] == b.pred[2];
}

// The bit reader's consumed position in canonical form, at an MCU boundary: walk back from the next unread byte over
// the data bytes whose bits are still buffered (a 0x00 after a 0xFF is the stuffing of that 0xFF: one data byte).
// Bits made up past the data (`fake`) were never in a byte.
FAA_JHD void jpeg_bits_pos(JpegBits& r, int32_t* byte, int16_t* bit) {
    const int u = r.n > r.fake ? r.n - r.fake : 0;        // real bits buffered, not consumed
    const uint8_t* q = r.p;
    for (int k = (u + 7) >> 3; k > 0; --k) {
        --q;
        if (q > r.lo && jpeg_byte_at(r, q) == 0 && jpeg_byte_at(r, q - 1) == 0xFF) --q;
    }
    *byte = (int32_t)(q - r.lo);
    *bit = (int16_t)((8 - (u & 7)) & 7);
}

// Starts the bit reader of the scan [lo, end) at a sync point: at its data byte (`data`, lo + s.byte), with the first
// s.bit bits of it dropped.
FAA_JHD void jpeg_bits_start(JpegBits& r, const uint8_t* lo, const uint8_t* data, const uint8_t* end, const JpegSync& s) {
    jpeg_bits_init(r, lo, data, end);
    if (s.bit > 0) { jpeg_fill(r); jpeg_get(r, s.bit); }
}

// Where a recording decode puts the points of the placement rule: at most `cap`, `n` written so far.
struct JpegIndexSink {
    JpegSync* at;
    int32_t cap, n;
    int32_t parts, next;     // segments of the rule; the next point k to place
};

// Where a decode that finds a scan index stops (jpeg_find_candidate, jpeg_find_link): at the first MCU boundary, its
// start state included, whose canonical start byte (jpeg_bits_pos) is >= `at`.  `hit`: it got there before its last MCU.
struct JpegStop {
    int64_t at;
    bool hit;
};

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

// Decodes MCUs [from.mcu, m1) of the scan [lo, end), starting in the state `from` (a restart segment: its first byte,
// bit 0, zero predictors), into coef.  huff[c] / huff[3 + c]: DC / AC tables of component c.  On an error the blocks
// from the failing one to the end of the segment are zeroed.  With `to`, a segment that decodes cleanly reports the
// state it ends in (MCU m1).  With `rec` (a recording decode of a whole restart-free scan) it places the points of the
// rule (jpeg_index_parts) at the MCU boundaries it passes; a recording decode stores the coefficients (and zeroes the
// blocks after an error) only when it has a `coef` (written `!rec || coef`: a decode without a sink always has one, and
// compiles without the test).
// `data`: the start byte as a pointer, instead of lo + from.byte (a restart segment whose marker is missing starts at
// `end`).  With `stop` it stores nothing and ends at the stop's boundary (unless it has a `coef`); `to` then reports that
// boundary, with to->mcu the MCUs decoded.  Returns JpegStatus.
FAA_JHD int jpeg_decode_segment(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* lo, const uint8_t* end,
                                const JpegSync& from, int64_t m1, int16_t* coef, int16_t* scratch, JpegSync* to = nullptr,
                                JpegIndexSink* rec = nullptr, const uint8_t* data = nullptr, JpegStop* stop = nullptr) {
    JpegBits r;
    jpeg_bits_start(r, lo, data ? data : lo + from.byte, end, from);
    int pred[3] = {from.pred[0], from.pred[1], from.pred[2]};
    const int nb = jpeg_blocks_per_mcu(h);
    const int ny = h.ncomp == 1 ? 1 : h.hs * h.vs;
    int status = JPEG_OK;
    int64_t m = from.mcu;
    int b = 0;
    for (; m < m1; ++m) {
        if (stop) {                                      // an MCU boundary (the start included): far enough?
            int32_t byte;
            int16_t bit;
            jpeg_bits_pos(r, &byte, &bit);
            if ((int64_t)byte >= stop->at) { stop->hit = true; break; }
        }
        if (rec && m > from.mcu) {                       // an MCU boundary: the points whose threshold it reaches
            JpegSync s;
            jpeg_bits_pos(r, &s.byte, &s.bit);
            bool placed = false;
            while (rec->next < rec->parts && (int64_t)s.byte >= jpeg_index_threshold(h, rec->parts, rec->next)) {
                if (!placed && rec->n < rec->cap) {
                    s.mcu = (int32_t)m;
                    for (int c = 0; c < 3; ++c) s.pred[c] = (int16_t)pred[c];
                    rec->at[rec->n++] = s;
                    placed = true;                       // (the later thresholds it reaches coincide: dropped)
                }
                ++rec->next;
            }
        }
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
            if ((!rec && !stop) || coef) jpeg_store_block(coef + 64 * jpeg_block_of(h, m, b), scratch);
        }
        if (status) break;
        if (r.n < r.fake) { status = JPEG_TRUNCATED; ++m; b = 0; break; }     // this MCU used bits past the data
    }
    if (status && ((!rec && !stop) || coef)) {
        jpeg_zero_block(scratch);
        for (; m < m1; ++m, b = 0)
            for (; b < nb; ++b) jpeg_store_block(coef + 64 * jpeg_block_of(h, m, b), scratch);
    }
    if (to && !status) {
        to->mcu = (int32_t)(stop && stop->hit ? m - from.mcu : m1);
        jpeg_bits_pos(r, &to->byte, &to->bit);
        for (int c = 0; c < 3; ++c) to->pred[c] = (int16_t)pred[c];
    }
    return status;
}

// a restart segment: MCUs [m0, m1) from `data` (its first byte), zero predictors
FAA_JHD int jpeg_decode_segment(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* lo, const uint8_t* data,
                                const uint8_t* end, int64_t m0, int64_t m1, int16_t* coef, int16_t* scratch) {
    const JpegSync from = {(int32_t)m0, 0, 0, {0, 0, 0}};
    return jpeg_decode_segment(h, huff, lo, end, from, m1, coef, scratch, nullptr, nullptr, data);
}

// The recording decode of a scan index: the whole scan, serially, placing the points of the rule into at[0, cap).
// Returns the number of points, 0 when the scan does not decode cleanly (or the file gets no index); *status gets the
// decode's status.
FAA_JHD int jpeg_index_record(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* scan, JpegSync* at,
                              int cap, int16_t* scratch, int* status) {
    *status = 0;
    const int parts = jpeg_index_parts(h);
    if (!parts || cap <= 0) return 0;
    JpegIndexSink rec = {at, cap < parts - 1 ? cap : parts - 1, 0, parts, 1};
    const JpegSync zero = {0, 0, 0, {0, 0, 0}};
    *status = jpeg_decode_segment(h, huff, scan, scan + h.scan_len, zero, jpeg_mcus(h), nullptr, scratch, nullptr, &rec);
    return *status ? 0 : rec.n;
}

// The sink of a recording entropy decode (a recording faa_jpeg_decode) of a restart-free scan decoded whole and serially:
// the file's points go to at[0, cap), cap being the room the caller planned for it (faa_jpeg_index_capacity).  False,
// and no sink, when the rule gives the file no points or it has no room.
FAA_JHD bool jpeg_record_sink(const JpegHeader& h, JpegSync* at, int64_t cap, JpegIndexSink& s) {
    const int parts = jpeg_index_parts(h);
    if (!parts || cap <= 0) return false;
    s = {at, cap < parts - 1 ? (int32_t)cap : parts - 1, 0, parts, 1};
    return true;
}

// Segment k of an indexed scan with n points: MCUs [pts[k - 1].mcu, pts[k].mcu), the first from the scan's start and
// the last to its end.  Its status, and whether it ended where the next segment starts (the last one always does).
FAA_JHD int jpeg_index_segment(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* scan, const JpegSync* pts,
                               int n, int k, int16_t* coef, int16_t* scratch, bool* linked) {
    const JpegSync zero = {0, 0, 0, {0, 0, 0}};
    const JpegSync& from = k == 0 ? zero : pts[k - 1];
    const int64_t m1 = k < n ? (int64_t)pts[k].mcu : jpeg_mcus(h);
    JpegSync to;
    const int st = jpeg_decode_segment(h, huff, scan, scan + h.scan_len, from, m1, coef, scratch, &to);
    *linked = k == n || (st == 0 && jpeg_sync_same(to, pts[k]));
    return st;
}

// ------------------------------------------------------------------------------------------------ finding an index --
// The points of the placement rule found in parallel, without a serial decode, for a restart-free scan of P =
// jpeg_index_parts parts with thresholds T_k = jpeg_index_threshold(k).  Huffman streams self-synchronise: a parse
// started at an arbitrary bit soon falls onto the true code boundaries, and onto the true block of its MCU.
//   pass 1  part k (1 <= k < P) starts W bytes before T_k (bit 0, past the 0x00 of a stuffed pair), assumes block 0 of
//           an MCU, and decodes to the first MCU boundary of its own parse at or past T_k: candidate c_k.  c_0 is the
//           scan's start.
//   pass 2  link k (0 <= k < P - 1) decodes from c_k, with MCU count and DC predictors 0, to the first MCU boundary at
//           or past T_{k + 1} (c_k itself when it is there already: the points coincide).  It holds when it ends at
//           c_{k + 1}; when it does not, its end becomes c_{k + 1} and link k + 1 runs again in the next round.
//   prefix  from the scan's start, each link that holds gives the next point its MCU and predictors (the start's plus
//           the link's); the walk stops at the first link that does not hold or is stale.
// By induction every point of the prefix is the rule's, with the serial decoder's MCU and predictors: found points are
// always a prefix of jpeg_index_record's, and all of them once every link holds.  Each round extends the verified
// prefix by at least one link.  The window W and the round cap R are measured (DESIGN §4.8).
constexpr int kJpegFindWindow = 512;           // W, bytes
constexpr int kJpegFindRounds = 8;             // R, rounds of pass 2

// pass 1 for part k: candidate c_k (byte -1 when the parse fails before T_k)
FAA_JHD void jpeg_find_candidate(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* scan, int parts, int k,
                                 int window, int16_t* scratch, JpegSync* c) {
    const int64_t t = jpeg_index_threshold(h, parts, k);
    int64_t s = t > window ? t - window : 0;
    if (s > 0 && scan[s] == 0 && scan[s - 1] == 0xFF) ++s;        // the stuffing of a 0xFF is no data byte
    const JpegSync from = {0, (int32_t)s, 0, {0, 0, 0}};
    JpegStop stop = {t, false};
    JpegSync to;
    const int st = jpeg_decode_segment(h, huff, scan, scan + h.scan_len, from, jpeg_mcus(h), nullptr, scratch, &to,
                                       nullptr, nullptr, &stop);
    *c = to;
    if (st || !stop.hit) c->byte = -1;
}

// pass 2, link k from c: the end it reaches, with mcu = the MCUs it decoded and pred = the DC differences (mcu -1 when
// it fails: a bad start, a decode error, or no boundary at or past T_{k + 1})
FAA_JHD void jpeg_find_link(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* scan, int parts, int k,
                            const JpegSync& c, int16_t* scratch, JpegSync* e) {
    e->mcu = -1;
    if (c.byte < 0) return;
    const JpegSync from = {0, c.byte, c.bit, {0, 0, 0}};
    JpegStop stop = {jpeg_index_threshold(h, parts, k + 1), false};
    JpegSync to;
    const int st = jpeg_decode_segment(h, huff, scan, scan + h.scan_len, from, jpeg_mcus(h), nullptr, scratch, &to,
                                       nullptr, nullptr, &stop);
    if (!st && stop.hit) *e = to;
}

FAA_JHD bool jpeg_find_holds(const JpegSync& e, const JpegSync& c) { return e.mcu >= 0 && e.byte == c.byte && e.bit == c.bit; }

// the repair after a round, for link k: a link that ended cleanly elsewhere than c_{k + 1} moves it there.  Returns
// whether link k + 1 is now stale (and runs again next round).
FAA_JHD bool jpeg_find_repair(const JpegSync* link, JpegSync* cand, int parts, int k) {
    const JpegSync& e = link[k];
    if (e.mcu < 0 || jpeg_find_holds(e, cand[k + 1])) return false;
    cand[k + 1] = e;
    return k + 2 < parts;
}

// The verified prefix into at[0, cap): walk the links from the scan's start while each is fresh (stale[k] == 0) and
// holds.  Returns the number of points; *full: every point of the rule was found (the walk passed the last link, or a
// link went past the scan's last MCU, after which the rule places nothing).
FAA_JHD int jpeg_find_prefix(const JpegHeader& h, int parts, const JpegSync* cand, const JpegSync* link,
                             const uint8_t* stale, JpegSync* at, int cap, bool* full) {
    JpegSync p = {0, 0, 0, {0, 0, 0}};
    int n = 0;
    *full = false;
    for (int k = 0; k + 1 < parts; ++k) {
        const JpegSync& e = link[k];
        if (stale[k] || !jpeg_find_holds(e, cand[k + 1])) return n;
        if (e.mcu == 0) continue;                                  // point k + 1 coincides with point k: dropped
        if ((int64_t)p.mcu + e.mcu >= jpeg_mcus(h)) { *full = true; return n; }
        if (n == cap) return n;
        p.mcu += e.mcu;
        p.byte = e.byte;
        p.bit = e.bit;
        for (int c = 0; c < 3; ++c) p.pred[c] = (int16_t)(p.pred[c] + e.pred[c]);
        at[n++] = p;
    }
    *full = true;
    return n;
}

// what one find did, for the measurement of W and R
struct JpegFindStats {
    int32_t links, held_first, rounds;       // links of the chain, links that held in round 1, rounds run
    int32_t full;                            // every point of the rule was found
};

// The whole find on one thread, as the find kernel runs it on one thread per part (host build and measurement): at
// most `rounds` rounds of pass 2, window W = `window` bytes.  Returns the number of points written to at[0, cap).
inline int jpeg_index_find(const JpegHeader& h, const JpegHuff* const* huff, const uint8_t* scan, int window, int rounds,
                           JpegSync* at, int cap, int16_t* scratch, JpegFindStats* stats) {
    JpegFindStats st = {0, 0, 0, 0};
    const int parts = jpeg_index_parts(h);
    int n = 0;
    if (parts) {
        JpegSync cand[kJpegIndexMaxParts], link[kJpegIndexMaxParts];
        uint8_t stale[kJpegIndexMaxParts];
        cand[0] = {0, 0, 0, {0, 0, 0}};
        for (int k = 1; k < parts; ++k) jpeg_find_candidate(h, huff, scan, parts, k, window, scratch, &cand[k]);
        for (int k = 0; k < parts; ++k) stale[k] = k + 1 < parts;
        st.links = parts - 1;
        for (int r = 0; r < rounds; ++r) {
            for (int k = 0; k + 1 < parts; ++k)
                if (stale[k]) jpeg_find_link(h, huff, scan, parts, k, cand[k], scratch, &link[k]);
            if (r == 0)
                for (int k = 0; k + 1 < parts; ++k) st.held_first += jpeg_find_holds(link[k], cand[k + 1]);
            bool any = false;
            stale[0] = 0;
            for (int k = 0; k + 1 < parts; ++k) any |= stale[k + 1] = jpeg_find_repair(link, cand, parts, k);
            st.rounds = r + 1;
            if (!any) break;
        }
        bool full = false;
        n = jpeg_find_prefix(h, parts, cand, link, stale, at, cap, &full);
        st.full = full;
    }
    if (stats) *stats = st;
    return n;
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

// post-IDCT range limit: +128, saturated to 0..255 (libjpeg-turbo's x86-64 SIMD islow IDCT, which Pillow runs;
// libjpeg's C table would wrap outputs outside [-512, 511] modulo 1024)
FAA_JHD uint8_t jpeg_range_limit(int32_t x) {
    const int32_t v = x + 128;
    return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
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

// ------------------------------------------------------------------------------------------------ output tiles --
constexpr int kJpegTileW = 64, kJpegTileH = 32;    // output pixels of one reconstruct CTA

// component c's blocks [bx0, bx0 + nbx) x [by0, by0 + nby) cover what a tile reads of its plane; they are blocks
// [first, first + nbx * nby) of the tile's blocks, row-major
struct JpegTileWindow { int32_t bx0, by0, nbx, nby, first; };

// Windows of the tile of output pixels [x0, x1) x [y0, y1): its luma blocks, and its chroma blocks with the one-sample
// halo fancy upsampling reads (clamped to the plane).  Components past h.ncomp get empty windows.  Returns the number
// of blocks of the tile.
FAA_JHD int jpeg_tile_windows(const JpegHeader& h, int x0, int y0, int x1, int y1, JpegTileWindow pl[3]) {
    const int cw = jpeg_chroma_w(h), ch = jpeg_chroma_h(h);
    int n_blocks = 0;
    for (int c = 0; c < 3; ++c) {
        if (c >= h.ncomp) { pl[c] = {0, 0, 0, 0, n_blocks}; continue; }
        int px0 = x0, px1 = x1 - 1, py0 = y0, py1 = y1 - 1;
        if (c > 0) {
            const int fx = h.hs == 2 ? 1 : 0, fy = h.vs == 2 ? 1 : 0;
            px0 = x0 / h.hs - fx; px1 = (x1 - 1) / h.hs + fx;
            py0 = y0 / h.vs - fy; py1 = (y1 - 1) / h.vs + fy;
            px0 = px0 < 0 ? 0 : px0; px1 = px1 > cw - 1 ? cw - 1 : px1;
            py0 = py0 < 0 ? 0 : py0; py1 = py1 > ch - 1 ? ch - 1 : py1;
        }
        pl[c] = {px0 >> 3, py0 >> 3, (px1 >> 3) - (px0 >> 3) + 1, (py1 >> 3) - (py0 >> 3) + 1, n_blocks};
        n_blocks += pl[c].nbx * pl[c].nby;
    }
    return n_blocks;
}

// ------------------------------------------------------------------------------------------------ host decode --
// The whole decode of one file on the host, serially, with the functions above: the CPU tests' model of the two
// kernels.  out: h.h * h.w * 3 bytes.  With a scan index (npts points) the entropy decode runs as the entropy kernel's
// indexed path does: validate, one segment per point, end states checked, a serial decode when anything disagrees.
// With rec_count, as the recording kernel does: a restart-free scan decoded whole and serially places its points into
// rec_at[0, rec_cap) (jpeg_record_sink), and *rec_count gets their number, or 0 when the scan was not decoded that way,
// gets no points or did not decode cleanly.  coef_out: the coefficients (jpeg_image_blocks(h) blocks).  Returns the
// JpegStatus bits.
inline void jpeg_reconstruct_host(const JpegHeader& h, const JpegTable* tabs, const int16_t* coef, uint8_t* out);
inline int jpeg_decode_host(const uint8_t* file, const JpegHeader& h, const JpegTable* tabs, uint8_t* out,
                            const JpegSync* pts = nullptr, int64_t npts = 0, JpegSync* rec_at = nullptr,
                            int64_t rec_cap = 0, int32_t* rec_count = nullptr, int16_t* coef_out = nullptr) {
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
    int64_t n_seg = jpeg_segments(h);
    const int64_t mcus = jpeg_mcus(h);
    int32_t* at = new int32_t[(size_t)n_seg];
    for (int64_t k = 0; k < n_seg; ++k) at[k] = -1;
    at[0] = 0;
    int status = 0;
    if (n_seg > 1) {
        JpegBits r; jpeg_bits_init(r, scan, scan, end);
        if (jpeg_markers(r, scan, 0, h.scan_len, h.scan_len, at, 1, n_seg) != n_seg - 1) status |= JPEG_BAD_RESTART;
    }
    bool indexed = pts && jpeg_index_count_ok(h, npts);
    for (int64_t k = 0; indexed && k < npts; ++k) indexed = jpeg_index_point_ok(h, pts[k], k ? pts[k - 1].mcu : 0);
    if (indexed) {
        bool linked = true;
        for (int k = 0; k <= (int)npts; ++k) {
            bool ok = true;
            const int st = jpeg_index_segment(h, hp, scan, pts, (int)npts, k, coef, scratch, &ok);
            linked = linked && ok;
            if (k == (int)npts) status = st;
        }
        if (linked) n_seg = 0;                           // done; otherwise the serial decode below overwrites it all
        else status = 0;
    }
    JpegIndexSink sink;
    JpegIndexSink* rec = rec_count && n_seg == 1 && jpeg_record_sink(h, rec_at, rec_cap, sink) ? &sink : nullptr;
    for (int64_t k = 0; k < n_seg; ++k) {
        const int64_t m0 = k * (h.restart > 0 ? h.restart : mcus), m1 = n_seg == 1 ? mcus : (m0 + h.restart < mcus ? m0 + h.restart : mcus);
        const uint8_t* p = at[k] < 0 ? end : scan + at[k];
        const JpegSync from = {(int32_t)m0, 0, 0, {0, 0, 0}};
        status |= jpeg_decode_segment(h, hp, scan, end, from, m1, coef, scratch, nullptr, rec, p);
    }
    if (rec_count) *rec_count = rec && !status ? rec->n : 0;
    if (coef_out) memcpy(coef_out, coef, (size_t)nblk * 128);
    jpeg_reconstruct_host(h, tabs, coef, out);
    delete[] at;
    delete[] coef;
    return status;
}

// The reconstruct kernel's work on the host: coefficient planes -> islow IDCT -> fancy upsampling -> RGB (h.h * h.w * 3)
inline void jpeg_reconstruct_host(const JpegHeader& h, const JpegTable* tabs, const int16_t* coef, uint8_t* out) {
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
}

// ------------------------------------------------------------------------------------------------ progressive --
// Progressive Huffman files (SOF2), ITU T.81 G.1.2, decoded as libjpeg does, into the same coefficient planes the
// reconstruct stage reads.  parse_jpeg_progressive takes what parse_jpeg takes (8-bit, 1 or 3 components, 4:4:4 / 4:2:2 /
// 4:2:0) when it is coded progressively and every coefficient of every component ends at bit 0; libjpeg smooths the
// blocks of an incomplete progression, which is not modelled, so those files are refused.  Its header has
// reserved = kJpegProgressive, restart = 0 and no scan_off / scan_len; the scans are a separate list.
constexpr int32_t kJpegProgressive = 1;      // JpegHeader::reserved of a progressive file (0 for every other)
constexpr int kJpegMaxScans = 64;

// layout of faa_jpeg_scan_t
struct JpegScan {
    int64_t off, len;            // entropy-coded data, relative to the file
    int32_t restart;             // restart interval in force at its SOS (0: none)
    int32_t ns;                  // components in the scan, comp[0, ns) their frame indices in frame order
    int32_t comp[3];
    int32_t ss, se, ah, al;      // spectral band [ss, se], successive approximation bits
    int32_t wave;                // 1 + the largest wave of an earlier scan sharing a (component, coefficient)
    int32_t dc_at[3], ac_at[3];  // file offsets of the DC tables of comp[k] (DC first scans) / the AC table (k = 0; AC
                                 // scans) as defined at its SOS, kJpegStdAt - k for standard table k, -1 when unused
    int32_t pool[6];             // the same tables as pool indices: DC of comp[k] at k, AC at 3 (-1 when unused)
    int32_t reserved[2];
};

FAA_JHD bool jpeg_is_progressive(const JpegHeader& h) { return h.reserved == kJpegProgressive; }

// Huffman tables a scan uses: DC first: one per component; DC refinement: none; AC: one
FAA_JHD int jpeg_scan_tables(const JpegScan& s) { return s.ss == 0 ? (s.ah == 0 ? s.ns : 0) : 1; }

// Wave numbers of scans [0, n) (the dependency rule of JpegScan::wave).  Scans of one wave share no (component,
// coefficient), so they can be decoded in any order.
inline void jpeg_scan_waves(JpegScan* s, int n) {
    int8_t last[3][64];
    memset(last, -1, sizeof last);
    for (int i = 0; i < n; ++i) {
        int w = 0;
        for (int k = 0; k < s[i].ns; ++k)
            for (int q = s[i].ss; q <= s[i].se; ++q) w = last[s[i].comp[k]][q] + 1 > w ? last[s[i].comp[k]][q] + 1 : w;
        s[i].wave = w;
        for (int k = 0; k < s[i].ns; ++k)
            for (int q = s[i].ss; q <= s[i].se; ++q) last[s[i].comp[k]][q] = (int8_t)w;
    }
}

// Parses a progressive file (host only): its header and at most max_scans scans (*n_scans of them).  Returns JPARSE_*
// with the reason of a refusal in *why, as parse_jpeg does; a file that is not progressive is refused too.
inline int parse_jpeg_progressive(const uint8_t* b, size_t len, JpegHeader& h, JpegScan* scans, int max_scans,
                                  int* n_scans, const char** why) {
    memset(&h, 0, sizeof h);
    for (int k = 0; k < 9; ++k) { h.table_at[k] = -1; h.pool[k] = -1; }
    h.len = (int64_t)len;
    h.reserved = kJpegProgressive;
    *n_scans = 0;
    *why = "";
#define FAA_BAD(msg) do { *why = msg; return JPARSE_MALFORMED; } while (0)
#define FAA_NO(msg) do { *why = msg; return JPARSE_UNSUPPORTED; } while (0)
    if (len < 4 || b[0] != 0xFF || b[1] != 0xD8) FAA_BAD("no SOI marker: not a JPEG file");
    if (len > 0x7FFFFFFF) FAA_NO("file larger than 2 GiB");
    int32_t dqt_at[4] = {-1, -1, -1, -1}, dqt_prec[4] = {0, 0, 0, 0}, dht_at[2][4];
    for (int c = 0; c < 2; ++c) for (int k = 0; k < 4; ++k) dht_at[c][k] = -1;
    bool jfif = false, adobe = false, have_sof = false;
    int adobe_transform = -1, restart = 0;
    int comp_id[3] = {0, 0, 0}, comp_h[3] = {0, 0, 0}, comp_v[3] = {0, 0, 0}, comp_q[3] = {0, 0, 0};
    int bitpos[3][64];                                   // current bit position of each coefficient, -1: not yet sent
    for (int c = 0; c < 3; ++c) for (int k = 0; k < 64; ++k) bitpos[c][k] = -1;
    size_t i = 2;
    while (true) {
        while (i < len && b[i] != 0xFF) ++i;
        while (i < len && b[i] == 0xFF) ++i;
        if (i >= len) break;                             // a file cut short: the progression check below judges it
        const int m = b[i++];
        if (m == 0xD9) break;                            // EOI
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
        if (m == 0xD8) FAA_BAD("second SOI marker");
        if (i + 2 > len) FAA_BAD("marker segment cut off");
        const int L = jpeg_u16(b + i);
        if (L < 2 || i + (size_t)L > len) FAA_BAD("marker segment length out of range");
        const uint8_t* p = b + i + 2;
        const int n = L - 2;
        const size_t seg_end = i + (size_t)L;
        if (m == 0xC2) {
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
            h.ncomp = nf; have_sof = true;
        } else if (m == 0xC0 || m == 0xC1) {
            FAA_NO("not a progressive frame (parse_jpeg takes it)");
        } else if (m == 0xCA) {
            FAA_NO("progressive arithmetic coding");
        } else if (m == 0xC6 || m == 0xCE || m == 0xC5 || m == 0xCD) {
            FAA_NO("hierarchical coding");
        } else if (m == 0xC3 || m == 0xC7 || m == 0xCB || m == 0xCF) {
            FAA_NO("lossless coding");
        } else if (m == 0xC9 || m == 0xCC) {
            FAA_NO("arithmetic coding");
        } else if (m == 0xC8) {
            FAA_NO("JPG extension frame");
        } else if (m == 0xDC) {
            FAA_NO("DNL marker");
        } else if (m == 0xC4) {                          // DHT (the checks of parse_jpeg)
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
                    if (code >= (1u << (l + 1))) FAA_BAD("Huffman table with more codes than its lengths allow");
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
        } else if (m == 0xDD) {                          // DRI: in force from the next SOS on
            if (n < 2) FAA_BAD("restart interval segment too short");
            restart = jpeg_u16(p);
        } else if (m == 0xE0) {
            if (n >= 14 && p[0] == 'J' && p[1] == 'F' && p[2] == 'I' && p[3] == 'F' && p[4] == 0) jfif = true;
        } else if (m == 0xEE) {
            if (n >= 12 && p[0] == 'A' && p[1] == 'd' && p[2] == 'o' && p[3] == 'b' && p[4] == 'e') {
                adobe = true; adobe_transform = p[11];
            }
        } else if (m == 0xDA) {                          // SOS
            if (!have_sof) FAA_BAD("scan before the frame header");
            if (n < 1) FAA_BAD("scan header too short");
            const int ns = p[0];
            if (ns < 1 || ns > h.ncomp || n != 4 + 2 * ns) FAA_BAD("scan header length does not match its components");
            if (*n_scans >= max_scans) FAA_NO("more scans than the decoder takes (64)");
            JpegScan& sc = scans[*n_scans];
            memset(&sc, 0, sizeof sc);
            for (int k = 0; k < 3; ++k) { sc.comp[k] = -1; sc.dc_at[k] = sc.ac_at[k] = -1; }
            for (int k = 0; k < 6; ++k) sc.pool[k] = -1;
            sc.ns = ns;
            const uint8_t* q = p + 1 + 2 * ns;
            sc.ss = q[0]; sc.se = q[1]; sc.ah = q[2] >> 4; sc.al = q[2] & 15;
            // the parameter checks of libjpeg's progressive decoder (it refuses these files too)
            if (sc.ss == 0 ? sc.se != 0 : ns != 1) FAA_BAD("bad progression: a DC scan with AC coefficients or an AC scan of several components");
            if (sc.se > 63 || sc.ss > sc.se) FAA_BAD("bad progression: spectral band out of range");
            if (sc.al > 13) FAA_BAD("bad progression: Al above 13");
            if (sc.ah != 0 && sc.ah != sc.al + 1) FAA_BAD("bad progression: Ah is neither 0 nor Al + 1");
            int prev = -1;
            for (int k = 0; k < ns; ++k) {
                int c = 0;
                while (c < h.ncomp && comp_id[c] != p[1 + 2 * k]) ++c;
                if (c == h.ncomp) FAA_BAD("scan names a component the frame does not have");
                if (c <= prev) FAA_NO("scan components out of frame order");
                prev = c;
                sc.comp[k] = c;
                const int td = p[2 + 2 * k] >> 4, ta = p[2 + 2 * k] & 15;
                if (td > 3 || ta > 3) FAA_BAD("Huffman table index out of range");
                if (sc.ss == 0 && sc.ah == 0) {
                    sc.dc_at[k] = dht_at[0][td] >= 0 ? dht_at[0][td] : td < 2 ? kJpegStdAt - td : -1;
                    if (sc.dc_at[k] == -1) FAA_BAD("scan uses an undefined Huffman table");
                } else if (sc.ss > 0) {
                    sc.ac_at[k] = dht_at[1][ta] >= 0 ? dht_at[1][ta] : ta < 2 ? kJpegStdAt - 2 - ta : -1;
                    if (sc.ac_at[k] == -1) FAA_BAD("scan uses an undefined Huffman table");
                }
                if (h.table_at[c] < 0) {                 // the quantisation table is latched at the first scan
                    if (dqt_at[comp_q[c]] < 0) FAA_BAD("component uses an undefined quantisation table");
                    h.table_at[c] = dqt_at[comp_q[c]];
                    if (dqt_prec[comp_q[c]]) h.qprec |= 1 << c;
                }
                // the progression: libjpeg decodes these with a warning; refused here
                if (sc.ss > 0 && bitpos[c][0] < 0) FAA_NO("bad progression: AC before the component's first DC scan");
                for (int z = sc.ss; z <= sc.se; ++z) {
                    if (sc.ah == 0 && bitpos[c][z] >= 0) FAA_NO("bad progression: a second first pass over a coefficient");
                    if (sc.ah != 0 && bitpos[c][z] != sc.ah) FAA_NO("bad progression: a refinement whose Ah is not the coefficient's bit position");
                    bitpos[c][z] = sc.al;
                }
            }
            sc.restart = restart;
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
            sc.off = (int64_t)s; sc.len = (int64_t)(e - s);
            ++*n_scans;
            i = e;
            continue;
        }
        i = seg_end;
    }
    if (!have_sof) FAA_BAD("no progressive frame header");
    if (*n_scans == 0) FAA_BAD("no scan");
    for (int c = 0; c < h.ncomp; ++c)
        for (int z = 0; z < 64; ++z)
            if (bitpos[c][z] != 0) FAA_NO("incomplete progression (a coefficient does not end at bit 0)");
    if (h.ncomp == 3) {
        if (!jfif && adobe && adobe_transform == 0) FAA_NO("Adobe-transformed RGB (APP14 transform 0)");
        if (!jfif && !adobe && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B') FAA_NO("RGB components");
        const bool ok = comp_h[1] == 1 && comp_v[1] == 1 && comp_h[2] == 1 && comp_v[2] == 1 &&
                        ((comp_h[0] == 1 && comp_v[0] == 1) || (comp_h[0] == 2 && comp_v[0] == 1) ||
                         (comp_h[0] == 2 && comp_v[0] == 2));
        if (!ok) FAA_NO("sampling factors other than 4:4:4, 4:2:2 (2x1) or 4:2:0 (2x2)");
        h.hs = comp_h[0]; h.vs = comp_v[0];
    } else {
        h.hs = h.vs = 1;
    }
    h.mcu_x = (h.w + 8 * h.hs - 1) / (8 * h.hs);
    h.mcu_y = (h.h + 8 * h.vs - 1) / (8 * h.vs);
    jpeg_scan_waves(scans, *n_scans);
    return JPARSE_OK;
#undef FAA_BAD
#undef FAA_NO
}

// the quantisation tables of a progressive header (out[0, 3)) and the Huffman tables of its scans (out[3 + 6 s + k]:
// DC of comp[k] at k, AC at 3), in pool form, unused slots zeroed
inline void jpeg_progressive_tables(const uint8_t* b, const JpegHeader& h, const JpegScan* scans, int n, JpegTable* out) {
    memset(out, 0, (size_t)(3 + 6 * n) * sizeof(JpegTable));
    for (int c = 0; c < h.ncomp; ++c) {
        const uint8_t* q = b + h.table_at[c];
        for (int k = 0; k < 64; ++k) out[c].q[kJpegZigzag[k]] = (h.qprec >> c & 1) ? (uint16_t)jpeg_u16(q + 2 * k) : q[k];
    }
    for (int s = 0; s < n; ++s)
        for (int k = 0; k < 6; ++k) {
            const int32_t at = k < 3 ? scans[s].dc_at[k] : scans[s].ac_at[k - 3];
            if (at == -1) continue;
            const uint8_t* std_table = jpeg_std_huff(at);
            const uint8_t* d = std_table ? std_table : b + at;
            JpegTable& t = out[3 + 6 * s + k];
            int total = 0;
            for (int l = 0; l < 16; ++l) { t.bits[l] = d[l]; total += d[l]; }
            memcpy(t.vals, d + 16, (size_t)total);
        }
}

// Block extent of component c in a scan of that component alone (T.81 A.2): ceil(comp_w / 8) x ceil(comp_h / 8)
FAA_JHD int jpeg_comp_bw(const JpegHeader& h, int c) { return ((c == 0 ? h.w : jpeg_chroma_w(h)) + 7) / 8; }
FAA_JHD int jpeg_comp_bh(const JpegHeader& h, int c) { return ((c == 0 ? h.h : jpeg_chroma_h(h)) + 7) / 8; }
// units of a scan: the frame's MCUs (interleaved) or the component's blocks (one component)
FAA_JHD int64_t jpeg_scan_units(const JpegHeader& h, const JpegScan& s) {
    return s.ns > 1 ? jpeg_mcus(h) : (int64_t)jpeg_comp_bw(h, s.comp[0]) * jpeg_comp_bh(h, s.comp[0]);
}
FAA_JHD int64_t jpeg_scan_segments(const JpegHeader& h, const JpegScan& s) {
    return s.restart > 0 ? (jpeg_scan_units(h, s) + s.restart - 1) / s.restart : 1;
}
// block index (within the image's coefficient buffer) of block (bx, by) of component c's padded grid
FAA_JHD int64_t jpeg_comp_block(const JpegHeader& h, int c, int64_t bx, int64_t by) {
    if (c == 0) return by * ((int64_t)h.mcu_x * h.hs) + bx;
    return jpeg_plane_blocks(h, 0) + (int64_t)(c - 1) * jpeg_mcus(h) + by * h.mcu_x + bx;
}

FAA_JHD uint32_t jpeg_bit(JpegBits& r) {
    if (r.n < 1) jpeg_fill(r);
    return jpeg_get(r, 1);
}

// Decodes units [u0, u1) of scan s (a restart segment: its data from `data`, EOBRUN and predictors zero) of the scan
// bytes [lo, end) into coef, accumulating into what earlier waves wrote.  huff[k]: the table of slot k
// (jpeg_scan_tables).  Stops at the first error; returns JpegStatus.
FAA_JHD int jpeg_prog_segment(const JpegHeader& h, const JpegScan& s, const JpegHuff* const* huff, const uint8_t* lo,
                              const uint8_t* data, const uint8_t* end, int64_t u0, int64_t u1, int16_t* coef) {
    JpegBits r;
    jpeg_bits_init(r, lo, data, end);
    int pred[3] = {0, 0, 0};
    int eobrun = 0;
    const int p1 = 1 << s.al, m1 = -p1;
    const int bw = s.ns == 1 ? jpeg_comp_bw(h, s.comp[0]) : 1;
    for (int64_t u = u0; u < u1; ++u) {
        if (s.ss == 0) {                                 // DC: every block of the MCU (one block without interleaving)
            for (int k = 0; k < s.ns; ++k) {
                const int c = s.comp[k];
                const int hc = s.ns == 1 || c > 0 ? 1 : h.hs, vc = s.ns == 1 || c > 0 ? 1 : h.vs;
                const int64_t ux = s.ns == 1 ? u % bw : (u % h.mcu_x) * hc, uy = s.ns == 1 ? u / bw : (u / h.mcu_x) * vc;
                for (int b = 0; b < hc * vc; ++b) {
                    int16_t* blk = coef + 64 * jpeg_comp_block(h, c, ux + b % hc, uy + b / hc);
                    jpeg_fill(r);
                    if (s.ah == 0) {
                        int t = jpeg_decode(r, *huff[k]);
                        if (t < 0) return JPEG_BAD_CODE;
                        if (t) t = jpeg_extend(jpeg_get(r, t), t);
                        pred[k] += t;
                        blk[0] = (int16_t)(int32_t)((uint32_t)pred[k] << s.al);
                    } else if (jpeg_get(r, 1)) {
                        blk[0] = (int16_t)(blk[0] | p1);
                    }
                }
            }
        } else {
            int16_t* blk = coef + 64 * jpeg_comp_block(h, s.comp[0], u % bw, u / bw);
            int k = s.ss;
            if (s.ah == 0) {                             // AC first pass
                if (eobrun > 0) {
                    --eobrun;
                } else {
                    for (; k <= s.se; ++k) {
                        jpeg_fill(r);
                        const int rs = jpeg_decode(r, *huff[0]);
                        if (rs < 0) return JPEG_BAD_CODE;
                        const int run = rs >> 4, sz = rs & 15;
                        if (sz) {
                            k += run;
                            if (k > s.se) return JPEG_BAD_COEF;
                            blk[jpeg_zigzag(k)] = (int16_t)(int32_t)((uint32_t)jpeg_extend(jpeg_get(r, sz), sz) << s.al);
                        } else if (run == 15) {
                            // (libjpeg lets a ZRL run past Se end the band; no encoder writes one, so it is reported
                            // as BAD_COEF here, as the baseline decoder reports one past coefficient 63)
                            k += 15;
                            if (k > s.se) return JPEG_BAD_COEF;
                        } else {
                            eobrun = 1 << run;
                            if (run) eobrun += (int)jpeg_get(r, run);
                            --eobrun;
                            break;
                        }
                    }
                }
            } else {                                     // AC refinement (libjpeg's decode_mcu_AC_refine)
                if (eobrun == 0) {
                    for (; k <= s.se; ++k) {
                        jpeg_fill(r);
                        const int rs = jpeg_decode(r, *huff[0]);
                        if (rs < 0) return JPEG_BAD_CODE;
                        int run = rs >> 4, val = 0;
                        if (rs & 15) {                   // (a size other than 1 is decoded as 1, as libjpeg does)
                            val = jpeg_get(r, 1) ? p1 : m1;
                        } else if (run != 15) {
                            eobrun = 1 << run;
                            if (run) eobrun += (int)jpeg_get(r, run);
                            break;
                        }
                        // correction bits of the nonzero coefficients passed; stop at the run's last zero
                        for (; k <= s.se; ++k) {
                            int16_t& v = blk[jpeg_zigzag(k)];
                            if (v != 0) {
                                if (jpeg_bit(r) && (v & p1) == 0) v = (int16_t)(v >= 0 ? v + p1 : v + m1);
                            } else if (--run < 0) {
                                break;
                            }
                        }
                        // (a run past Se: libjpeg ends the band, or writes the new coefficient at natural index 63;
                        // no encoder writes either, so it is reported as BAD_COEF)
                        if (k > s.se) return JPEG_BAD_COEF;
                        if (val) blk[jpeg_zigzag(k)] = (int16_t)val;
                    }
                }
                if (eobrun > 0) {                        // in an EOB run: correction bits of the band's rest
                    for (; k <= s.se; ++k) {
                        int16_t& v = blk[jpeg_zigzag(k)];
                        if (v != 0 && jpeg_bit(r) && (v & p1) == 0) v = (int16_t)(v >= 0 ? v + p1 : v + m1);
                    }
                    --eobrun;
                }
            }
        }
        if (r.n < r.fake) return JPEG_TRUNCATED;        // this unit used bits past the data
    }
    return JPEG_OK;
}

// The progressive kernel's entropy work on the host, one scan after another in file order (waves are an order the
// kernel may use instead: they give the same coefficients).  coef: jpeg_image_blocks(h) blocks, zeroed here.  tabs: the
// scans' tables in jpeg_progressive_tables' layout.  Returns JpegStatus bits.
inline int jpeg_progressive_entropy_host(const uint8_t* file, const JpegHeader& h, const JpegScan* scans, int n,
                                         const JpegTable* tabs, int16_t* coef) {
    memset(coef, 0, (size_t)jpeg_image_blocks(h) * 128);
    int status = 0;
    JpegHuff* huffs = new JpegHuff[3];
    for (int i = 0; i < n; ++i) {
        const JpegScan& s = scans[i];
        const JpegHuff* hp[3] = {&huffs[0], &huffs[1], &huffs[2]};
        for (int k = 0; k < jpeg_scan_tables(s); ++k) jpeg_huff_build(tabs[3 + 6 * i + (s.ss == 0 ? k : 3)], huffs[k]);
        const uint8_t* scan = file + s.off;
        const uint8_t* end = scan + s.len;
        const int64_t n_seg = jpeg_scan_segments(h, s), units = jpeg_scan_units(h, s);
        int32_t* at = new int32_t[(size_t)n_seg];
        for (int64_t k = 0; k < n_seg; ++k) at[k] = k ? -1 : 0;
        if (n_seg > 1) {
            JpegBits r; jpeg_bits_init(r, scan, scan, end);
            if (jpeg_markers(r, scan, 0, s.len, s.len, at, 1, n_seg) != n_seg - 1) status |= JPEG_BAD_RESTART;
        }
        for (int64_t k = 0; k < n_seg; ++k) {
            const int64_t u0 = k * (n_seg > 1 ? s.restart : 0), u1 = n_seg == 1 ? units : (u0 + s.restart < units ? u0 + s.restart : units);
            status |= jpeg_prog_segment(h, s, hp, scan, at[k] < 0 ? end : scan + at[k], end, u0, u1, coef);
        }
        delete[] at;
    }
    delete[] huffs;
    return status;
}

// The whole decode of one progressive file on the host (the progressive entropy kernel, then the reconstruct kernel).
// out: h.h * h.w * 3 bytes; coef_out: the coefficients, when given.  Returns JpegStatus bits.
inline int jpeg_decode_progressive_host(const uint8_t* file, const JpegHeader& h, const JpegScan* scans, int n,
                                        const JpegTable* tabs, uint8_t* out, int16_t* coef_out = nullptr) {
    const int64_t nblk = jpeg_image_blocks(h);
    int16_t* coef = new int16_t[(size_t)nblk * 64];
    const int status = jpeg_progressive_entropy_host(file, h, scans, n, tabs, coef);
    if (coef_out) memcpy(coef_out, coef, (size_t)nblk * 128);
    jpeg_reconstruct_host(h, tabs, coef, out);
    delete[] coef;
    return status;
}

}  // namespace faa
