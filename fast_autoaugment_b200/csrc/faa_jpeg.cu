// faa_jpeg.cu - sm_90a kernels of the baseline JPEG decoder (faa_jpeg_decode), arithmetic in faa_jpeg.cuh.
//
// Two launches per call, no host wait between them:
//   faa_jpeg_entropy_kernel      one CTA per image.  The CTA builds the image's Huffman lookup tables in shared
//                                memory; when the image has restart markers its threads find them in parallel (a
//                                count, a prefix sum, then the positions); then one thread per restart segment turns
//                                the scan into int16 coefficients.  An image without restart markers is one segment,
//                                decoded serially by one thread: the known limit of this design.
//   faa_jpeg_reconstruct_kernel  one CTA per 64 x 32 output tile of one image.  It runs the islow IDCT of the tile's
//                                blocks, with the one-block chroma halo fancy upsampling reads, into shared memory,
//                                upsamples and converts to RGB, and writes uint8 HWC rows with 32-bit stores where the
//                                destination address allows.
#include <cuda_runtime.h>
#include <stdint.h>

#include "faa_kernels.cuh"

namespace faa {

constexpr int kEntropyThreads = 128;
constexpr int kReconThreads = 256;
constexpr int kReconMaxBlocks = 96;        // 4:4:4: 8 x 4 blocks of each of the three components

__global__ void __launch_bounds__(kEntropyThreads) faa_jpeg_entropy_kernel(const __grid_constant__ JpegDecodeParams P) {
    __shared__ JpegHuff s_huff[6];
    __shared__ __align__(16) int16_t s_scratch[kEntropyThreads][64];
    __shared__ int32_t s_count[kEntropyThreads];
    __shared__ int32_t s_status;
    const int img = blockIdx.x, tid = threadIdx.x;
    const JpegHeader h = P.hdrs[img];
    const JpegJob job = P.jobs[img];
    const uint8_t* scan = P.src + h.offset + h.scan_off;
    const uint8_t* end = scan + h.scan_len;
    int32_t* segs = P.segs + job.seg;
    const int64_t n_seg = jpeg_segments(h), mcus = jpeg_mcus(h);
    if (tid == 0) s_status = 0;
    if (tid < 6 && tid % 3 < h.ncomp) jpeg_huff_codes(P.pool[h.pool[3 + tid]], s_huff[tid]);
    for (int64_t k = tid; k < n_seg; k += kEntropyThreads) segs[k] = k == 0 ? 0 : -1;
    __syncthreads();
    for (int e = tid; e < 6 << kJpegLookBits; e += kEntropyThreads) {
        const int t = e >> kJpegLookBits;
        if (t % 3 < h.ncomp) s_huff[t].look[e & ((1 << kJpegLookBits) - 1)] = jpeg_huff_look(s_huff[t], e & ((1 << kJpegLookBits) - 1));
    }
    if (n_seg > 1) {                                       // restart markers: count, prefix, record
        const int64_t chunk = (h.scan_len + kEntropyThreads - 1) / kEntropyThreads;
        const int64_t a = min((int64_t)tid * chunk, h.scan_len), b = min(a + chunk, h.scan_len);
        JpegBits r;
        jpeg_bits_init(r, scan, scan, end);
        s_count[tid] = jpeg_markers(r, scan, a, b, h.scan_len, nullptr, 0, 0);
        __syncthreads();
        if (tid == 0) {
            int32_t run = 0;
            for (int t = 0; t < kEntropyThreads; ++t) { const int32_t c = s_count[t]; s_count[t] = run; run += c; }
            if (run != n_seg - 1) s_status = JPEG_BAD_RESTART;
        }
        __syncthreads();
        jpeg_markers(r, scan, a, b, h.scan_len, segs, 1 + s_count[tid], n_seg);
    }
    __syncthreads();
    const JpegHuff* hp[6];
    for (int t = 0; t < 6; ++t) hp[t] = &s_huff[t % 3 < h.ncomp ? t : (t / 3) * 3];
    int status = 0;
    for (int64_t k = tid; k < n_seg; k += kEntropyThreads) {
        const int64_t m0 = n_seg == 1 ? 0 : k * h.restart;
        const int64_t m1 = n_seg == 1 ? mcus : min(m0 + h.restart, mcus);
        const int32_t at = segs[k];
        status |= jpeg_decode_segment(h, hp, scan, at < 0 ? end : scan + at, end, m0, m1, P.coef + 64 * job.coef,
                                      s_scratch[tid]);
    }
    if (status) atomicOr(&s_status, status);
    __syncthreads();
    if (tid == 0) P.status[img] = s_status;
}

__global__ void __launch_bounds__(kReconThreads) faa_jpeg_reconstruct_kernel(const __grid_constant__ JpegDecodeParams P) {
    __shared__ uint16_t s_q[3][64];
    __shared__ int32_t s_ws[kReconMaxBlocks][64];
    __shared__ __align__(16) uint8_t s_pix[3][kJpegTileW * kJpegTileH];
    __shared__ __align__(16) uint8_t s_rgb[kJpegTileW * kJpegTileH * 3];
    const int tid = threadIdx.x;
    const int tile = blockIdx.x;
    int lo = 0, hi = P.batch - 1;                          // image whose tiles hold this one
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (P.jobs[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
    }
    const int img = lo;
    const JpegHeader h = P.hdrs[img];
    const int64_t coef0 = P.jobs[img].coef;
    const int tiles_x = (h.w + kJpegTileW - 1) / kJpegTileW;
    const int t = tile - P.jobs[img].tile0;
    const int x0 = (t % tiles_x) * kJpegTileW, y0 = (t / tiles_x) * kJpegTileH;
    const int x1 = min(x0 + kJpegTileW, h.w), y1 = min(y0 + kJpegTileH, h.h);
    const int cw = jpeg_chroma_w(h), ch = jpeg_chroma_h(h);
    JpegTileWindow pl[3];
    const int n_blocks = jpeg_tile_windows(h, x0, y0, x1, y1, pl);
    int64_t plane_base[3];
    int grid_w[3];
    int64_t base = 0;
    for (int c = 0; c < 3; ++c) {
        if (c >= h.ncomp) { plane_base[c] = 0; grid_w[c] = 1; continue; }
        plane_base[c] = base;
        grid_w[c] = h.mcu_x * (c == 0 ? h.hs : 1);
        base += jpeg_plane_blocks(h, c);
    }
    for (int k = tid; k < 64 * h.ncomp; k += kReconThreads) s_q[k >> 6][k & 63] = P.pool[h.pool[k >> 6]].q[k & 63];
    __syncthreads();
    // IDCT, column pass: one thread per (block, column)
    for (int item = tid; item < n_blocks * 8; item += kReconThreads) {
        const int k = item >> 3, col = item & 7;
        const int c = k < pl[1].first ? 0 : k < pl[2].first ? 1 : 2;
        const int local = k - pl[c].first;
        const int bx = pl[c].bx0 + local % pl[c].nbx, by = pl[c].by0 + local / pl[c].nbx;
        const int16_t* blk = P.coef + 64 * (coef0 + plane_base[c] + (int64_t)by * grid_w[c] + bx);
        jpeg_idct_col(blk, s_q[c], col, s_ws[k]);
    }
    __syncthreads();
    // row pass: one thread per (block, row) -> the component's sample plane of the tile
    for (int item = tid; item < n_blocks * 8; item += kReconThreads) {
        const int k = item >> 3, row = item & 7;
        const int c = k < pl[1].first ? 0 : k < pl[2].first ? 1 : 2;
        const int local = k - pl[c].first;
        const int lx = local % pl[c].nbx, ly = local / pl[c].nbx;
        jpeg_idct_row(s_ws[k], row, &s_pix[c][(ly * 8 + row) * (pl[c].nbx * 8) + lx * 8]);
    }
    __syncthreads();
    // upsampling + colour conversion into the tile's RGB rows
    const int ncols = x1 - x0, nrows = y1 - y0;
    for (int p = tid; p < ncols * nrows; p += kReconThreads) {
        const int x = x0 + p % ncols, y = y0 + p / ncols;
        uint8_t* o = &s_rgb[((y - y0) * kJpegTileW + (x - x0)) * 3];
        const int Y = s_pix[0][(y - pl[0].by0 * 8) * (pl[0].nbx * 8) + (x - pl[0].bx0 * 8)];
        if (h.ncomp == 1) { o[0] = o[1] = o[2] = (uint8_t)Y; continue; }
        const int cbx = pl[1].bx0 * 8, cby = pl[1].by0 * 8, cs = pl[1].nbx * 8;
        const int vcb = jpeg_upsample(JpegPlane{s_pix[1], cs, cbx, cby}, x, y, h.hs, h.vs, cw, ch);
        const int vcr = jpeg_upsample(JpegPlane{s_pix[2], cs, cbx, cby}, x, y, h.hs, h.vs, cw, ch);
        jpeg_ycc_rgb(Y, vcb, vcr, o);
    }
    __syncthreads();
    // rows out: leading bytes up to a 4-byte boundary, 32-bit words, trailing bytes
    uint8_t* dst0 = const_cast<uint8_t*>(P.out[img].data);
    const int nbytes = ncols * 3;
    constexpr int kUnits = kJpegTileW * 3 / 4 + 2;
    for (int item = tid; item < nrows * kUnits; item += kReconThreads) {
        const int r = item / kUnits, u = item % kUnits;
        uint8_t* g = dst0 + ((int64_t)(y0 + r) * h.w + x0) * 3;
        const uint8_t* s = &s_rgb[r * kJpegTileW * 3];
        const int head = min(nbytes, (int)((4 - ((uintptr_t)g & 3)) & 3));
        const int words = (nbytes - head) >> 2;
        if (u == 0) {
            for (int k = 0; k < head; ++k) g[k] = s[k];
        } else if (u == kUnits - 1) {
            for (int k = head + 4 * words; k < nbytes; ++k) g[k] = s[k];
        } else if (u - 1 < words) {
            const int k = head + 4 * (u - 1);
            *reinterpret_cast<uint32_t*>(g + k) =
                (uint32_t)s[k] | ((uint32_t)s[k + 1] << 8) | ((uint32_t)s[k + 2] << 16) | ((uint32_t)s[k + 3] << 24);
        }
    }
}

cudaError_t launch_jpeg_entropy(const JpegDecodeParams& p, cudaStream_t stream) {
    if (p.batch <= 0) return cudaSuccess;
    faa_jpeg_entropy_kernel<<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_jpeg_reconstruct(const JpegDecodeParams& p, int n_tiles, cudaStream_t stream) {
    if (p.batch <= 0 || n_tiles <= 0) return cudaSuccess;
    faa_jpeg_reconstruct_kernel<<<(unsigned)n_tiles, kReconThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace faa
