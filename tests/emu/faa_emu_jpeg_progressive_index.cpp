// faa_emu_jpeg_progressive_index.cpp - HOST build of the progressive JPEG scan index, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host: the progressive decode with a scan index and with
// recording (jpeg_decode_progressive_host, which runs the progressive kernel's split into waves, items and whole-image
// redo on one thread), and the placement rule computed a second way, by chaining one-unit segments.  The package never
// loads it.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

namespace {

// parse, mark the header scan-indexed (or not) as the Python parse does, and build the tables
int parse(const uint8_t* bytes, int64_t len, int indexed, JpegHeader& h, JpegScan* scans, int* n,
          std::vector<JpegTable>& tabs) {
    const char* why = "";
    const int e = parse_jpeg_progressive(bytes, (size_t)len, h, scans, kJpegMaxScans, n, &why);
    if (e != JPARSE_OK) return e;
    if (indexed) {
        h.reserved = kJpegProgressive | kJpegScanIndexed;
        h.scan_len = jpeg_prog_axis(scans, *n);
    }
    tabs.resize((size_t)(3 + 6 * *n));
    jpeg_progressive_tables(bytes, h, scans, *n, tabs.data());
    return JPARSE_OK;
}

}  // namespace

extern "C" {

// The header of a file (scan-indexed when `indexed`): JPARSE_*.
int faa_emu_jpi_header(const uint8_t* bytes, int64_t len, int indexed, JpegHeader* hdr, int32_t* n_scans) {
    JpegScan scans[kJpegMaxScans];
    std::vector<JpegTable> tabs;
    int n = 0;
    const int e = parse(bytes, len, indexed, *hdr, scans, &n, tabs);
    *n_scans = n;
    return e;
}

// Decodes a progressive file as the progressive kernel does: with points pts[0, npts) (pts may be null), recording
// into rec_at[0, rec_cap) when rec_count is given.  out: h * w * 3 bytes (out_cap at most); coef: the coefficients when
// given (coef_cap int16 at most).  Returns the parse result; the decode runs when the file parses and the buffers have
// room.
int faa_emu_jpi_decode(const uint8_t* bytes, int64_t len, int indexed, const JpegSync* pts, int64_t npts,
                       JpegSync* rec_at, int64_t rec_cap, int32_t* rec_count, uint8_t* out, int64_t out_cap,
                       int16_t* coef, int64_t coef_cap, int32_t* status) {
    JpegHeader h;
    JpegScan scans[kJpegMaxScans];
    std::vector<JpegTable> tabs;
    int n = 0;
    *status = 0;
    const int e = parse(bytes, len, indexed, h, scans, &n, tabs);
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap || (coef && jpeg_image_blocks(h) * 64 > coef_cap)) return -1;
    *status = jpeg_decode_progressive_host(bytes, h, scans, n, tabs.data(), out, coef, pts, npts, rec_at, rec_cap,
                                           rec_count);
    return JPARSE_OK;
}

// The points of the placement rule, computed without the recording sink: every scan is decoded serially in file order,
// a restart-free one unit by unit (a one-unit segment from each unit's start state to the next), which gives the state
// at every unit boundary; then threshold k takes the first boundary u >= 1 of its scan whose byte is >= T_k and inside
// the scan, unless the previous point is that boundary.  Returns the number of points written to at[0, cap), or -1
// when the file does not parse or decode cleanly.  (With want_scan >= 0: stops at that boundary, see faa_emu_jpi_state.)
int faa_emu_jpi_rule_or_state(const uint8_t* bytes, int64_t len, JpegSync* at, int64_t cap, int want_scan,
                              int64_t want_unit) {
    JpegHeader h;
    JpegScan scans[kJpegMaxScans];
    std::vector<JpegTable> tabs;
    int n = 0;
    if (parse(bytes, len, 1, h, scans, &n, tabs) != JPARSE_OK) return -1;
    std::vector<int16_t> coef((size_t)jpeg_image_blocks(h) * 64, 0);
    JpegHuff huffs[3];
    const JpegHuff* hp[3] = {&huffs[0], &huffs[1], &huffs[2]};
    const int parts = jpeg_index_parts(h);
    std::vector<std::vector<JpegSync>> bounds((size_t)n);      // boundary states (axis bytes) of restart-free scans
    int64_t a = 0;
    for (int i = 0; i < n; ++i) {
        const JpegScan& s = scans[i];
        for (int k = 0; k < jpeg_scan_tables(s); ++k) jpeg_huff_build(tabs[(size_t)(3 + 6 * i + (s.ss == 0 ? k : 3))], huffs[k]);
        const uint8_t* scan = bytes + s.off;
        const uint8_t* end = scan + s.len;
        const int64_t units = jpeg_scan_units(h, s), n_seg = jpeg_scan_segments(h, s);
        if (n_seg == 1) {
            JpegSync st = {0, 0, 0, {0, 0, 0}};
            for (int64_t u = 0; u < units; ++u) {
                JpegSync to;
                if (jpeg_prog_segment(h, s, hp, scan, scan + st.byte, end, u, u + 1, coef.data(), &st, &to)) return -1;
                st = to;
                if (u + 1 < units) { JpegSync p = to; p.byte = (int32_t)(p.byte + a); bounds[(size_t)i].push_back(p); }
                if (i == want_scan && u + 1 == want_unit) { *at = bounds[(size_t)i].back(); return 1; }
            }
        } else {
            std::vector<int32_t> seg((size_t)n_seg, -1);
            seg[0] = 0;
            JpegBits r; jpeg_bits_init(r, scan, scan, end);
            if (jpeg_markers(r, scan, 0, s.len, s.len, seg.data(), 1, n_seg) != n_seg - 1) return -1;
            for (int64_t k = 0; k < n_seg; ++k) {
                const int64_t u0 = k * s.restart, u1 = u0 + s.restart < units ? u0 + s.restart : units;
                if (jpeg_prog_segment(h, s, hp, scan, scan + seg[(size_t)k], end, u0, u1, coef.data())) return -1;
            }
        }
        a += s.len;
    }
    int cnt = 0;
    const JpegSync* prev = nullptr;
    for (int k = 1; k < parts; ++k) {
        const int64_t t = jpeg_index_threshold(h, parts, k);
        const int i = jpeg_prog_scan_of(scans, n, t);
        if (i == n || scans[i].restart > 0) continue;
        const int64_t e = jpeg_prog_axis(scans, i) + scans[i].len;
        for (const JpegSync& p : bounds[(size_t)i]) {
            if (p.byte < t) continue;
            if (p.byte < e && &p != prev && cnt < cap) { at[cnt++] = p; prev = &p; }
            break;
        }
    }
    return cnt;
}

int faa_emu_jpi_rule(const uint8_t* bytes, int64_t len, JpegSync* at, int64_t cap) {
    return faa_emu_jpi_rule_or_state(bytes, len, at, cap, -1, 0);
}

// The state at unit boundary `unit` (1 <= unit < units) of restart-free scan `scan`, as a point: 1, or -1.
int faa_emu_jpi_state(const uint8_t* bytes, int64_t len, int scan, int64_t unit, JpegSync* at) {
    return faa_emu_jpi_rule_or_state(bytes, len, at, 1, scan, unit) == 1 ? 1 : -1;
}

}  // extern "C"
