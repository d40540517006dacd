// faa_emu_jpeg.cpp - HOST build of the JPEG decoder arithmetic, TEST INFRASTRUCTURE ONLY.
//
// Compiles fast_autoaugment_b200/csrc/faa_jpeg.cuh for the host and decodes one file with it: the same Huffman, IDCT,
// upsampling and colour functions the entropy and reconstruct kernels run, so the CPU tests can hold them against
// Pillow.  Two decodes: jpeg_decode_host, serially over the whole image, and a model of the kernels' split of the work
// (restart markers found over 128 chunks, a count, a prefix sum and a record pass, as the entropy kernel's threads do;
// then every 64 x 32 output tile built only from the blocks of its jpeg_tile_windows, as a reconstruct CTA is).  The
// package never loads it.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../fast_autoaugment_b200/csrc/faa_jpeg.cuh"

using namespace faa;

namespace {

constexpr int kChunks = 128;              // faa_jpeg_entropy_kernel's threads

// Decode with the kernels' split of the work.  trim > 0 drops the last block column of every chroma window wider than
// one block: a window too small, which must show in the output (what the sample poisoning is for).
int decode_tiled(const uint8_t* file, const JpegHeader& h, const JpegTable* tabs, uint8_t* out, int trim) {
    JpegHuff huffs[6];
    const JpegHuff* hp[6];
    for (int t = 0; t < 6; ++t)
        if (t % 3 < h.ncomp) { jpeg_huff_build(tabs[3 + t], huffs[t]); }
    for (int t = 0; t < 6; ++t) hp[t] = &huffs[t % 3 < h.ncomp ? t : (t / 3) * 3];
    const int64_t nblk = jpeg_image_blocks(h);
    std::vector<int16_t> coef((size_t)nblk * 64, (int16_t)0x7B7B);       // every block must be written
    alignas(16) int16_t scratch[64];
    const uint8_t* scan = file + h.scan_off;
    const uint8_t* end = scan + h.scan_len;
    const int64_t n_seg = jpeg_segments(h), mcus = jpeg_mcus(h);
    std::vector<int32_t> segs((size_t)n_seg, -1);
    segs[0] = 0;
    int status = 0;
    if (n_seg > 1) {                       // restart markers: count per chunk, prefix, record
        const int64_t chunk = (h.scan_len + kChunks - 1) / kChunks;
        int32_t count[kChunks];
        for (int t = 0; t < kChunks; ++t) {
            const int64_t a = std::min((int64_t)t * chunk, (int64_t)h.scan_len), b = std::min(a + chunk, (int64_t)h.scan_len);
            JpegBits r;
            jpeg_bits_init(r, scan, scan, end);
            count[t] = jpeg_markers(r, scan, a, b, h.scan_len, nullptr, 0, 0);
        }
        int32_t run = 0;
        for (int t = 0; t < kChunks; ++t) { const int32_t c = count[t]; count[t] = run; run += c; }
        if (run != n_seg - 1) status |= JPEG_BAD_RESTART;
        for (int t = 0; t < kChunks; ++t) {
            const int64_t a = std::min((int64_t)t * chunk, (int64_t)h.scan_len), b = std::min(a + chunk, (int64_t)h.scan_len);
            JpegBits r;
            jpeg_bits_init(r, scan, scan, end);
            jpeg_markers(r, scan, a, b, h.scan_len, segs.data(), 1 + count[t], n_seg);
        }
    }
    for (int64_t k = 0; k < n_seg; ++k) {
        const int64_t m0 = n_seg == 1 ? 0 : k * h.restart;
        const int64_t m1 = n_seg == 1 ? mcus : std::min(m0 + h.restart, mcus);
        status |= jpeg_decode_segment(h, hp, scan, segs[k] < 0 ? end : scan + segs[k], end, m0, m1, coef.data(), scratch);
    }
    // full sample planes, as a serial decode makes them; a tile's planes start as these with every sample flipped by
    // 128, and only the blocks of the tile's windows are decoded into them
    int64_t plane_base[3] = {0, 0, 0};
    int grid_w[3] = {1, 1, 1}, grid_h[3] = {1, 1, 1};
    std::vector<uint8_t> full[3], tile[3];
    int64_t base = 0;
    auto idct_block = [&](int c, int bx, int by, uint8_t* plane) {
        int32_t ws[64];
        const int16_t* blk = coef.data() + 64 * (plane_base[c] + (int64_t)by * grid_w[c] + bx);
        for (int col = 0; col < 8; ++col) jpeg_idct_col(blk, tabs[c].q, col, ws);
        for (int row = 0; row < 8; ++row) jpeg_idct_row(ws, row, plane + (size_t)(by * 8 + row) * grid_w[c] * 8 + bx * 8);
    };
    for (int c = 0; c < h.ncomp; ++c) {
        plane_base[c] = base;
        grid_w[c] = h.mcu_x * (c == 0 ? h.hs : 1);
        grid_h[c] = h.mcu_y * (c == 0 ? h.vs : 1);
        base += jpeg_plane_blocks(h, c);
        full[c].resize((size_t)grid_w[c] * grid_h[c] * 64);
        for (int by = 0; by < grid_h[c]; ++by)
            for (int bx = 0; bx < grid_w[c]; ++bx) idct_block(c, bx, by, full[c].data());
        tile[c].resize(full[c].size());
    }
    const int cw = jpeg_chroma_w(h), ch = jpeg_chroma_h(h);
    const int tiles_x = (h.w + kJpegTileW - 1) / kJpegTileW, tiles_y = (h.h + kJpegTileH - 1) / kJpegTileH;
    for (int t = 0; t < tiles_x * tiles_y; ++t) {
        const int x0 = (t % tiles_x) * kJpegTileW, y0 = (t / tiles_x) * kJpegTileH;
        const int x1 = std::min(x0 + kJpegTileW, h.w), y1 = std::min(y0 + kJpegTileH, h.h);
        JpegTileWindow pl[3];
        jpeg_tile_windows(h, x0, y0, x1, y1, pl);
        for (int c = 1; c < h.ncomp && trim > 0; ++c)
            if (pl[c].nbx > 1) --pl[c].nbx;
        for (int c = 0; c < h.ncomp; ++c) {
            for (size_t k = 0; k < full[c].size(); ++k) tile[c][k] = (uint8_t)(full[c][k] ^ 0x80);
            for (int by = pl[c].by0; by < pl[c].by0 + pl[c].nby; ++by)
                for (int bx = pl[c].bx0; bx < pl[c].bx0 + pl[c].nbx; ++bx) idct_block(c, bx, by, tile[c].data());
        }
        for (int y = y0; y < y1; ++y)
            for (int x = x0; x < x1; ++x) {
                uint8_t* o = out + ((size_t)y * h.w + x) * 3;
                const int Y = tile[0][(size_t)y * grid_w[0] * 8 + x];
                if (h.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; continue; }
                const int cb = jpeg_upsample(JpegPlane{tile[1].data(), grid_w[1] * 8, 0, 0}, x, y, h.hs, h.vs, cw, ch);
                const int cr = jpeg_upsample(JpegPlane{tile[2].data(), grid_w[2] * 8, 0, 0}, x, y, h.hs, h.vs, cw, ch);
                jpeg_ycc_rgb(Y, cb, cr, o);
            }
    }
    return status;
}

}  // namespace

extern "C" {

// Parses `bytes` and, when it is supported and out_cap >= h * w * 3, decodes it into out (uint8 HWC): mode 0 serially
// (jpeg_decode_host), mode 1 with the kernels' split of the work, mode 2 as 1 with chroma windows one block too narrow.
// Returns the parse result (0 ok, 1 unsupported, 2 malformed); *status gets the decode status bits, *hw the size.
int faa_emu_jpeg_decode_mode(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t out_cap, int32_t* status, int32_t* hw,
                             int mode) {
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg(bytes, (size_t)len, h, &why);
    *status = 0;
    hw[0] = h.h; hw[1] = h.w;
    if (e != JPARSE_OK) return e;
    if ((int64_t)h.h * h.w * 3 > out_cap) return JPARSE_OK;
    JpegTable tabs[9];
    jpeg_tables(bytes, h, tabs);
    *status = mode == 0 ? jpeg_decode_host(bytes, h, tabs, out) : decode_tiled(bytes, h, tabs, out, mode - 1);
    return JPARSE_OK;
}

int faa_emu_jpeg_decode(const uint8_t* bytes, int64_t len, uint8_t* out, int64_t out_cap, int32_t* status, int32_t* hw) {
    return faa_emu_jpeg_decode_mode(bytes, len, out, out_cap, status, hw, 0);
}

}  // extern "C"
