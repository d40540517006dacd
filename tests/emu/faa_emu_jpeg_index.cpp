// faa_emu_jpeg_index.cpp - HOST build of the JPEG scan index, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host: the recording decode faa_jpeg_index_kernel runs
// (jpeg_index_record), the indexed decode of the entropy kernel (jpeg_decode_host with points: validation, one segment
// per point, end states checked, serial decode when any disagrees), and the serial decoder's state at every MCU
// boundary, found by chaining one-MCU segments through their reported end states rather than by the recording code.
// The package never loads it.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

namespace {

struct Parsed {
    JpegHeader h;
    JpegTable tabs[9];
    JpegHuff huffs[6];
    const JpegHuff* hp[6];
};

bool parse(const uint8_t* bytes, int64_t len, Parsed& p) {
    const char* why = "";
    if (parse_jpeg(bytes, (size_t)len, p.h, &why) != JPARSE_OK) return false;
    jpeg_tables(bytes, p.h, p.tabs);
    for (int t = 0; t < 6; ++t)
        if (t % 3 < p.h.ncomp) jpeg_huff_build(p.tabs[3 + t], p.huffs[t]);
    for (int t = 0; t < 6; ++t) p.hp[t] = &p.huffs[t % 3 < p.h.ncomp ? t : (t / 3) * 3];
    return true;
}

}  // namespace

extern "C" {

// The scan index of a file, at most cap points into out.  Returns the number of points, -1 when the file does not
// parse; *status gets the recording decode's status, scan[0] / scan[1] the scan's offset and length.
int faa_emu_jpeg_index(const uint8_t* bytes, int64_t len, JpegSync* out, int32_t cap, int32_t* status, int64_t* scan) {
    Parsed p;
    *status = 0;
    if (!parse(bytes, len, p)) return -1;
    scan[0] = p.h.scan_off; scan[1] = p.h.scan_len;
    alignas(16) int16_t scratch[64];
    int st = 0;
    const int n = jpeg_index_record(p.h, p.hp, bytes + p.h.scan_off, out, cap, scratch, &st);
    *status = st;
    return n;
}

// The serial decoder's state at MCU boundaries 0, 1, ... into out (up to cap of them): each one-MCU segment starts in
// the state the previous one reported.  Returns the number of states, which stops short of the MCU count at the first
// MCU that does not decode cleanly; -1 when the file does not parse.
int64_t faa_emu_jpeg_states(const uint8_t* bytes, int64_t len, JpegSync* out, int64_t cap) {
    Parsed p;
    if (!parse(bytes, len, p)) return -1;
    const uint8_t* scan = bytes + p.h.scan_off;
    std::vector<int16_t> coef((size_t)jpeg_image_blocks(p.h) * 64);
    alignas(16) int16_t scratch[64];
    const int64_t mcus = jpeg_mcus(p.h);
    JpegSync s = {0, 0, 0, {0, 0, 0}};
    int64_t n = 0;
    for (int64_t m = 0; m < mcus && n < cap; ++m) {
        out[n++] = s;
        JpegSync to;
        if (jpeg_decode_segment(p.h, p.hp, scan, scan + p.h.scan_len, s, m + 1, coef.data(), scratch, &to)) break;
        s = to;
    }
    return n;
}

// Decodes a file with npts points of a scan index (jpeg_decode_host), as faa_emu_jpeg_decode does without one.
int faa_emu_jpeg_decode_indexed(const uint8_t* bytes, int64_t len, const JpegSync* pts, int64_t npts, uint8_t* out,
                                int64_t out_cap, int32_t* status, int32_t* hw) {
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg(bytes, (size_t)len, h, &why);
    *status = 0;
    hw[0] = h.h; hw[1] = h.w;
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap) return JPARSE_OK;
    JpegTable tabs[9];
    jpeg_tables(bytes, h, tabs);
    *status = jpeg_decode_host(bytes, h, tabs, out, pts, npts);
    return JPARSE_OK;
}

// Whether npts points are used as they stand: they pass the device checks and every segment ends in the state the
// next one starts in (1), or the decode falls back to the serial one (0); -1 when the file does not parse.
int faa_emu_jpeg_index_linked(const uint8_t* bytes, int64_t len, const JpegSync* pts, int64_t npts) {
    Parsed p;
    if (!parse(bytes, len, p)) return -1;
    bool ok = pts && jpeg_index_count_ok(p.h, npts);
    for (int64_t k = 0; ok && k < npts; ++k) ok = jpeg_index_point_ok(p.h, pts[k], k ? pts[k - 1].mcu : 0);
    if (!ok) return 0;
    std::vector<int16_t> coef((size_t)jpeg_image_blocks(p.h) * 64);
    alignas(16) int16_t scratch[64];
    for (int k = 0; k <= (int)npts; ++k) {
        bool linked = true;
        jpeg_index_segment(p.h, p.hp, bytes + p.h.scan_off, pts, (int)npts, k, coef.data(), scratch, &linked);
        if (!linked) return 0;
    }
    return 1;
}

}  // extern "C"
