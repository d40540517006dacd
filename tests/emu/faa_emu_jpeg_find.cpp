// faa_emu_jpeg_find.cpp - HOST build of the scan index find, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host: jpeg_index_find, the steps faa_jpeg_find_kernel runs
// on one thread per part (candidates, rounds of links and repairs, the verified prefix), with the window W and the
// round cap R as parameters.  tools/jpeg_find_sweep.py measures W and R with it.  The package never loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

extern "C" {

// The points the find gives a file, at most cap into out; stats[4]: links, links that held in round 1, rounds run,
// whether every point of the rule was found.  Returns the number of points, -1 when the file does not parse.
int faa_emu_jpeg_find(const uint8_t* bytes, int64_t len, int32_t window, int32_t rounds, JpegSync* out, int32_t cap,
                      int32_t* stats) {
    JpegHeader h;
    const char* why = "";
    if (parse_jpeg(bytes, (size_t)len, h, &why) != JPARSE_OK) return -1;
    JpegTable tabs[9];
    jpeg_tables(bytes, h, tabs);
    JpegHuff huffs[6];
    const JpegHuff* hp[6];
    for (int t = 0; t < 6; ++t)
        if (t % 3 < h.ncomp) jpeg_huff_build(tabs[3 + t], huffs[t]);
    for (int t = 0; t < 6; ++t) hp[t] = &huffs[t % 3 < h.ncomp ? t : (t / 3) * 3];
    alignas(16) int16_t scratch[64];
    JpegFindStats st;
    const int n = jpeg_index_find(h, hp, bytes + h.scan_off, window, rounds, out, cap, scratch, &st);
    stats[0] = st.links; stats[1] = st.held_first; stats[2] = st.rounds; stats[3] = st.full;
    return n;
}

}  // extern "C"
