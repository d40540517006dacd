// faa_emu_jpeg_record.cpp - HOST build of the recording JPEG decode, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host: jpeg_decode_host with and without recording, as the
// entropy kernel's recording and plain / indexed instantiations run it, with its coefficients.  The package never
// loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

extern "C" {

// Decodes a file with npts points (none: pts null) into out (h * w * 3 bytes, out_cap at most) and, with coef, its
// coefficients (coef_cap int16 at most).  With rec_count it records as a recording faa_jpeg_decode does: points into
// rec_at[0, rec_cap), their number in *rec_count.  hw gets the size.  Returns the parse result (JPARSE_*); the decode
// runs only when the file parses and out and coef have room.
int faa_emu_jpeg_decode_recording(const uint8_t* bytes, int64_t len, const JpegSync* pts, int64_t npts, uint8_t* out,
                                  int64_t out_cap, int32_t* status, int32_t* hw, JpegSync* rec_at, int64_t rec_cap,
                                  int32_t* rec_count, int16_t* coef, int64_t coef_cap) {
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg(bytes, (size_t)len, h, &why);
    *status = 0;
    hw[0] = h.h; hw[1] = h.w;
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap || (coef && jpeg_image_blocks(h) * 64 > coef_cap)) return JPARSE_OK;
    JpegTable tabs[9];
    jpeg_tables(bytes, h, tabs);
    *status = jpeg_decode_host(bytes, h, tabs, out, pts, npts, rec_at, rec_cap, rec_count, coef);
    return JPARSE_OK;
}

}  // extern "C"
