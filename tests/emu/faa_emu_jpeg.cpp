// faa_emu_jpeg.cpp - HOST build of the JPEG decoder arithmetic, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host and decodes one file serially with it: the same
// Huffman, IDCT, upsampling and colour functions the entropy and reconstruct kernels run, so the CPU tests can hold
// them against Pillow.  The package never loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

extern "C" {

// Parses `bytes` and, when it is supported and out_cap >= h * w * 3, decodes it into out (uint8 HWC).
// Returns the parse result (0 ok, 1 unsupported, 2 malformed); *status gets the decode status bits, *hw the size.
int faa_emu_jpeg_decode(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t out_cap, int32_t* status, int32_t* hw) {
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg(bytes, (size_t)len, h, &why);
    *status = 0;
    hw[0] = h.h; hw[1] = h.w;
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap) return JPARSE_OK;
    JpegTable tabs[9];
    jpeg_tables(bytes, h, tabs);
    *status = jpeg_decode_host(bytes, h, tabs, out);
    return JPARSE_OK;
}

}  // extern "C"
