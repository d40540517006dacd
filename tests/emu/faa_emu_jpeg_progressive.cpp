// faa_emu_jpeg_progressive.cpp - HOST build of the progressive JPEG decoder, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host: parse_jpeg_progressive and the progressive entropy
// decode (jpeg_prog_segment, the function the progressive kernel runs) followed by the reconstruct arithmetic.  The
// package never loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

extern "C" {

// Parses a file: header into hdr, scans into scans[0, max_scans), their number into *n.  Returns JPARSE_*; *why the
// reason of a refusal.
int faa_emu_jpeg_progressive_parse(const uint8_t* bytes, int64_t len, JpegHeader* hdr, JpegScan* scans, int max_scans,
                                   int32_t* n, const char** why) {
    int ns = 0;
    const int e = parse_jpeg_progressive(bytes, (size_t)len, *hdr, scans, max_scans, &ns, why);
    *n = ns;
    return e;
}

// Waves of scans[0, n) by the dependency rule (overwrites their wave fields).
void faa_emu_jpeg_scan_waves(JpegScan* scans, int n) { jpeg_scan_waves(scans, n); }

// Parses and decodes a progressive file into out (h * w * 3 bytes, out_cap at most) and, with coef, its coefficients
// (coef_cap int16 at most).  hw gets the size.  Returns the parse result; the decode runs only when the file parses
// and out and coef have room.
int faa_emu_jpeg_progressive_decode(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t out_cap, int32_t* status,
                                    int32_t* hw, int16_t* coef, int64_t coef_cap) {
    JpegHeader h;
    JpegScan scans[kJpegMaxScans];
    int n = 0;
    const char* why = "";
    const int e = parse_jpeg_progressive(bytes, (size_t)len, h, scans, kJpegMaxScans, &n, &why);
    *status = 0;
    hw[0] = h.h; hw[1] = h.w;
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap || (coef && jpeg_image_blocks(h) * 64 > coef_cap)) return JPARSE_OK;
    JpegTable* tabs = new JpegTable[3 + 6 * n];
    jpeg_progressive_tables(bytes, h, scans, n, tabs);
    *status = jpeg_decode_progressive_host(bytes, h, scans, n, tabs, out, coef);
    delete[] tabs;
    return JPARSE_OK;
}

}  // extern "C"
