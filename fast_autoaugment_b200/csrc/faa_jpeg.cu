// faa_jpeg.cu - sm_90a kernels of the JPEG decoder (faa_jpeg_decode), arithmetic in faa_jpeg.cuh.
//
// A call launches, with no host wait between them, the find kernel (with find), the entropy kernel (when the batch has
// baseline images), the progressive kernel (when it has progressive images) and the reconstruct kernel over every
// image.  The two entropy kernels have one CTA per image of the batch; each returns at once on the other's images.
//   faa_jpeg_entropy_kernel      one CTA per baseline image.  The CTA builds the image's Huffman lookup tables in shared
//                                memory; when the image has restart markers its threads find them in parallel (a
//                                count, a prefix sum, then the positions); then one thread per restart segment turns
//                                the scan into int16 coefficients.  An image without restart markers is one segment,
//                                decoded serially by one thread, unless the call gives it a scan index: then thread k
//                                decodes from point k to point k + 1 and checks that it ended in that point's state;
//                                if any segment disagrees, thread 0 decodes the scan serially over it.  The recording
//                                instantiation (a recording faa_jpeg_decode) also places the scan index of every scan
//                                thread 0 decodes whole and serially, as faa_jpeg_index_kernel would.
//   faa_jpeg_index_kernel        (faa_jpeg_index_build) one CTA per image; one thread records the scan index.
//   faa_jpeg_find_kernel         (faa_jpeg_index_find, faa_jpeg_decode's find) one CTA per image; thread k finds point k
//                                of the scan index in parallel, and links checked against the next point verify a
//                                prefix of it.  The found decode's entropy instantiation reads the counts it leaves.
//   faa_jpeg_progressive_kernel  one CTA per progressive image: the entropy stage of progressive files, scans run wave
//                                by wave.  Its indexed instantiation splits a kJpegScanIndexed file's restart-free scans
//                                at their points and checks every split; its recording one places those points.
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

// the image's Huffman tables in shared memory, built by the whole CTA (the lookup entries are complete after the
// caller's next barrier); hp[t]: the table of slot t, slots of absent components pointing at component 0's
__device__ __forceinline__ void jpeg_cta_tables(const JpegHeader& h, const JpegTable* pool, JpegHuff* s_huff, int tid,
                                                const JpegHuff* hp[6]) {
    if (tid < 6 && tid % 3 < h.ncomp) jpeg_huff_codes(pool[h.pool[3 + tid]], s_huff[tid]);
    __syncthreads();
    for (int e = tid; e < 6 << kJpegLookBits; e += kEntropyThreads) {
        const int t = e >> kJpegLookBits;
        if (t % 3 < h.ncomp) s_huff[t].look[e & ((1 << kJpegLookBits) - 1)] = jpeg_huff_look(s_huff[t], e & ((1 << kJpegLookBits) - 1));
    }
    for (int t = 0; t < 6; ++t) hp[t] = &s_huff[t % 3 < h.ncomp ? t : (t / 3) * 3];
}

// kIndexed: the call gives scan indexes (P.first, P.points); the plain instantiation is the path without them.
// kRecord (with kIndexed, whose P.first may then be null): a restart-free scan that thread 0 decodes whole and serially
// (no points, or points that failed) records its points into P.rec_points[P.rec_first[i], P.rec_first[i + 1]), and
// P.count[i] gets their number; every other image gets count 0.
// kFound (with both, faa_jpeg_decode's find): an image without input points uses the points faa_jpeg_find_kernel left
// in its recording range, P.count[i] of them (~n: a prefix of n that did not converge); count[i] stays n when they were
// the whole index and were used.
template <bool kIndexed, bool kRecord, bool kFound = false>
__global__ void __launch_bounds__(kEntropyThreads) faa_jpeg_entropy_kernel(const __grid_constant__ JpegDecodeParams P) {
    __shared__ JpegHuff s_huff[6];
    __shared__ __align__(16) int16_t s_scratch[kEntropyThreads][64];
    __shared__ int32_t s_count[kEntropyThreads];
    __shared__ int32_t s_status;
    const int img = blockIdx.x, tid = threadIdx.x;
    if ((P.hdrs[img].reserved | kJpegScanIndexed) == (kJpegProgressive | kJpegScanIndexed))
        return;                                              // faa_jpeg_progressive_kernel's (before h: DESIGN §4.8)
    const JpegHeader h = P.hdrs[img];
    const JpegJob job = P.jobs[img];
    const uint8_t* scan = P.src + h.offset + h.scan_off;
    const uint8_t* end = scan + h.scan_len;
    int32_t* segs = P.segs + job.seg;
    const int64_t n_seg = jpeg_segments(h), mcus = jpeg_mcus(h);
    if (tid == 0) s_status = 0;
    for (int64_t k = tid; k < n_seg; k += kEntropyThreads) segs[k] = k == 0 ? 0 : -1;
    const JpegHuff* hp[6];
    jpeg_cta_tables(h, P.pool, s_huff, tid, hp);
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
    int status = 0;
    bool serial = true;
    int64_t n_pts = !kIndexed || (kRecord && !P.first) ? 0 : P.first[img + 1] - P.first[img];
    const JpegSync* pts = kIndexed && n_pts > 0 ? P.points + P.first[img] : nullptr;
    bool found_all = false;
    if constexpr (kFound) {
        if (n_pts == 0) {
            const int32_t c = P.count[img];
            found_all = c >= 0;
            n_pts = found_all ? c : ~c;
            pts = P.rec_points + P.rec_first[img];
        }
    }
    if (kIndexed && n_pts > 0) {                                       // a scan index: one segment per thread from its points
        bool ok = jpeg_index_count_ok(h, n_pts);
        if (ok && tid < n_pts) ok = jpeg_index_point_ok(h, pts[tid], tid ? pts[tid - 1].mcu : 0);
        if (__syncthreads_and(ok)) {
            bool linked = true;
            if (tid <= n_pts)
                status = jpeg_index_segment(h, hp, scan, pts, (int)n_pts, tid, P.coef + 64 * job.coef, s_scratch[tid], &linked);
            // every segment ended where the next one starts: by induction each started in the serial decode's state.
            // Otherwise thread 0 decodes the scan serially below, overwriting every block.
            serial = !__syncthreads_and(linked);
            if (serial) status = 0;
        }
    }
    JpegIndexSink sink;
    JpegIndexSink* rec = nullptr;
    if (kRecord && serial && n_seg == 1 && tid == 0 &&
        jpeg_record_sink(h, P.rec_points + P.rec_first[img], P.rec_first[img + 1] - P.rec_first[img], sink))
        rec = &sink;
    for (int64_t k = tid; serial && k < n_seg; k += kEntropyThreads) {
        const int64_t m0 = n_seg == 1 ? 0 : k * h.restart;
        const int64_t m1 = n_seg == 1 ? mcus : min(m0 + h.restart, mcus);
        const int32_t at = segs[k];
        if constexpr (kRecord) {
            const JpegSync from = {(int32_t)m0, 0, 0, {0, 0, 0}};
            status |= jpeg_decode_segment(h, hp, scan, end, from, m1, P.coef + 64 * job.coef, s_scratch[tid], nullptr,
                                          rec, at < 0 ? end : scan + at);
        } else {
            status |= jpeg_decode_segment(h, hp, scan, at < 0 ? end : scan + at, end, m0, m1, P.coef + 64 * job.coef,
                                          s_scratch[tid]);
        }
    }
    if (status) atomicOr(&s_status, status);
    __syncthreads();
    if (tid == 0) P.status[img] = s_status;
    if constexpr (kFound) {
        if (tid == 0) P.count[img] = s_status ? 0 : rec ? rec->n : found_all && !serial ? (int32_t)n_pts : 0;
    } else {
        if (kRecord && tid == 0) P.count[img] = rec && !s_status ? rec->n : 0;
    }
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

// One CTA per image: the CTA builds the Huffman tables, then one thread decodes the scan serially without storing a
// coefficient and records the points of the placement rule (jpeg_index_parts), at most the capacity planned for it.
__global__ void __launch_bounds__(kEntropyThreads) faa_jpeg_index_kernel(const __grid_constant__ JpegDecodeParams P) {
    __shared__ JpegHuff s_huff[6];
    __shared__ __align__(16) int16_t s_scratch[64];
    const int img = blockIdx.x, tid = threadIdx.x;
    const JpegHeader h = P.hdrs[img];
    const JpegHuff* hp[6];
    jpeg_cta_tables(h, P.pool, s_huff, tid, hp);
    __syncthreads();
    if (tid != 0) return;
    const int64_t cap = P.first[img + 1] - P.first[img];
    int status = 0;
    const int n = jpeg_index_record(h, hp, P.src + h.offset + h.scan_off, P.points + P.first[img],
                                    cap < kJpegIndexMaxParts ? (int)cap : kJpegIndexMaxParts, s_scratch, &status);
    P.count[img] = n;
    P.status[img] = status;
}

// Finds scan indexes in parallel (jpeg_index_find's steps, faa_jpeg.cuh), one CTA per image, thread k on part k.  The
// CTA builds the Huffman tables; threads 1 .. P - 1 find their candidates (pass 1); then up to kJpegFindRounds rounds of
// links (pass 2) and repairs, a barrier between each, stop early when every link holds; thread 0 walks the verified
// prefix in shared memory and writes it to P.rec_points[P.rec_first[i], P.rec_first[i + 1]), the count to P.count[i].
// Images with input points (P.first, may be null) and images the rule gives no points get count 0.  `mark`: a prefix
// that did not converge gets count ~n instead of n (the found decode's entropy kernel reads it so).
__global__ void __launch_bounds__(kEntropyThreads) faa_jpeg_find_kernel(const __grid_constant__ JpegDecodeParams P, int mark) {
    __shared__ JpegHuff s_huff[6];
    __shared__ __align__(16) int16_t s_scratch[kEntropyThreads][64];
    __shared__ JpegSync s_cand[kJpegIndexMaxParts], s_link[kJpegIndexMaxParts];
    __shared__ uint8_t s_stale[kJpegIndexMaxParts];
    static_assert(kJpegIndexMaxParts == kEntropyThreads, "one thread per part");
    const int img = blockIdx.x, tid = threadIdx.x;
    const JpegHeader h = P.hdrs[img];
    const bool given = P.first && P.first[img + 1] > P.first[img];
    const int parts = given || jpeg_is_progressive(h) ? 0 : jpeg_index_parts(h);     // (progressive: not found here)
    if (parts == 0) {
        if (tid == 0) P.count[img] = 0;
        return;
    }
    const JpegHuff* hp[6];
    jpeg_cta_tables(h, P.pool, s_huff, tid, hp);
    __syncthreads();
    const uint8_t* scan = P.src + h.offset + h.scan_off;
    if (tid == 0) s_cand[0] = {0, 0, 0, {0, 0, 0}};
    else if (tid < parts) jpeg_find_candidate(h, hp, scan, parts, tid, kJpegFindWindow, s_scratch[tid], &s_cand[tid]);
    s_stale[tid] = tid + 1 < parts;
    __syncthreads();
    for (int r = 0; r < kJpegFindRounds; ++r) {
        if (s_stale[tid]) jpeg_find_link(h, hp, scan, parts, tid, s_cand[tid], s_scratch[tid], &s_link[tid]);
        __syncthreads();
        // thread k alone writes c_{k + 1} and stale[k + 1]; nobody reads them until the barrier
        const bool again = tid + 1 < parts && jpeg_find_repair(s_link, s_cand, parts, tid);
        if (tid + 1 < parts) s_stale[tid + 1] = again;
        if (tid == 0) s_stale[0] = 0;
        if (!__syncthreads_or(again)) break;
    }
    if (tid != 0) return;
    const int64_t cap = P.rec_first[img + 1] - P.rec_first[img];
    bool full = false;
    const int n = jpeg_find_prefix(h, parts, s_cand, s_link, s_stale, P.rec_points + P.rec_first[img],
                                   cap < kJpegIndexMaxParts ? (int)cap : kJpegIndexMaxParts, &full);
    P.count[img] = mark && !full ? ~n : n;
}

cudaError_t launch_jpeg_find(const JpegDecodeParams& p, bool mark, cudaStream_t stream) {
    if (p.batch <= 0) return cudaSuccess;
    faa_jpeg_find_kernel<<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p, mark ? 1 : 0);
    return cudaGetLastError();
}

// Progressive entropy decode, one CTA per image.  The CTA zeroes the image's coefficient planes (progressive scans
// accumulate into them), finds every scan's restart markers as the baseline kernel does, then runs the scans wave by
// wave.  A wave's scans share no (component, coefficient), so its work items, one per (scan, restart segment), run on
// all threads at once; a barrier separates waves.  A wave whose scans need more Huffman tables than kProgSlots (or has
// more than kProgGroup scans) runs as several groups, one after the other.
// kIndexed: the call gives scan indexes (P.first, P.points).  A kJpegScanIndexed image whose points pass their check
// runs a restart-free scan with k points as k + 1 work items, each comparing its end state with the next point
// (jpeg_prog_item); any failure marks the image at the group's barrier, and a marked image zeroes its planes and runs
// again without its points.  kRecord (with kIndexed, whose P.first may then be null): a kJpegScanIndexed image decoded
// without usable points places the rule's points of each restart-free scan while decoding it whole, thread 0 compacts
// them into P.rec_points[P.rec_first[i], P.rec_first[i + 1]), and P.count[i] gets their number; every other image of
// this kernel gets count 0.
constexpr int kProgSlots = 8, kProgGroup = 16;

template <bool kIndexed, bool kRecord>
__global__ void __launch_bounds__(kEntropyThreads) faa_jpeg_progressive_kernel(const __grid_constant__ JpegDecodeParams P) {
    __shared__ JpegHuff s_huff[kProgSlots];
    __shared__ JpegScan s_scan[kJpegMaxScans];
    __shared__ int32_t s_seg[kJpegMaxScans];              // first segment-start entry of each scan
    __shared__ uint8_t s_order[kJpegMaxScans];            // scans by wave, file order within a wave
    __shared__ int32_t s_count[kEntropyThreads];
    __shared__ int32_t s_gscan[kProgGroup], s_gslot[kProgGroup], s_gitem[kProgGroup + 1], s_gtab[kProgSlots];
    __shared__ int32_t s_ng, s_nslot, s_pos, s_status;
    __shared__ int32_t s_pfirst[kJpegMaxScans + 1];       // (kIndexed) first point of each scan
    __shared__ JpegSync s_rec[kJpegIndexMaxParts];        // (kRecord) point k of the rule at [k], mcu -1 if none
    const int img = blockIdx.x, tid = threadIdx.x;
    if ((P.hdrs[img].reserved | kJpegScanIndexed) != (kJpegProgressive | kJpegScanIndexed)) return;  // the entropy kernel's
    const JpegHeader h = P.hdrs[img];
    const JpegJob job = P.jobs[img];
    const uint8_t* file = P.src + h.offset;
    const int n = (int)(P.scan_first[img + 1] - P.scan_first[img]);
    int16_t* coef = P.coef + 64 * job.coef;
    int32_t* segs = P.segs + job.seg;
    for (int k = tid; k < n; k += kEntropyThreads) s_scan[k] = P.scans[P.scan_first[img] + k];
    {
        uint4* z = reinterpret_cast<uint4*>(coef);
        const int64_t n16 = jpeg_image_blocks(h) * 8;
        for (int64_t k = tid; k < n16; k += kEntropyThreads) z[k] = make_uint4(0, 0, 0, 0);
    }
    if constexpr (kRecord) s_rec[tid].mcu = -1;
    __syncthreads();
    if (tid == 0) {
        s_status = 0;
        int32_t at = 0, o = 0;
        for (int k = 0; k < n; ++k) { s_seg[k] = at; at += (int32_t)jpeg_scan_segments(h, s_scan[k]); }
        for (int w = 0; o < n; ++w)
            for (int k = 0; k < n; ++k) if (s_scan[k].wave == w) s_order[o++] = (uint8_t)k;
    }
    __syncthreads();
    // restart-segment starts of every scan: count, prefix, record (as faa_jpeg_entropy_kernel)
    for (int k = 0; k < n; ++k) {
        const JpegScan& s = s_scan[k];
        const int64_t n_seg = jpeg_scan_segments(h, s);
        int32_t* ss = segs + s_seg[k];
        for (int64_t j = tid; j < n_seg; j += kEntropyThreads) ss[j] = j == 0 ? 0 : -1;
        if (n_seg == 1) continue;
        const uint8_t* scan = file + s.off;
        const int64_t chunk = (s.len + kEntropyThreads - 1) / kEntropyThreads;
        const int64_t a = min((int64_t)tid * chunk, s.len), b = min(a + chunk, s.len);
        JpegBits r;
        jpeg_bits_init(r, scan, scan, scan + s.len);
        s_count[tid] = jpeg_markers(r, scan, a, b, s.len, nullptr, 0, 0);
        __syncthreads();
        if (tid == 0) {
            int32_t run = 0;
            for (int t = 0; t < kEntropyThreads; ++t) { const int32_t c = s_count[t]; s_count[t] = run; run += c; }
            if (run != n_seg - 1) s_status = JPEG_BAD_RESTART;
        }
        __syncthreads();
        jpeg_markers(r, scan, a, b, s.len, ss, 1 + s_count[tid], n_seg);
        __syncthreads();
    }
    // the image's points, when it takes them and they pass their check
    const JpegSync* pts = nullptr;
    bool use = false;
    if constexpr (kIndexed) {
        const int64_t n_pts = jpeg_prog_indexed(h) && (!kRecord || P.first) ? P.first[img + 1] - P.first[img] : 0;
        if (n_pts > 0) {
            pts = P.points + P.first[img];
            bool ok = jpeg_index_count_ok(h, n_pts);
            if (ok && tid < n_pts) ok = jpeg_prog_point_ok(h, s_scan, n, pts, tid);
            use = __syncthreads_and(ok);
            if (use && tid == 0) jpeg_prog_point_first(s_scan, n, pts, (int)n_pts, s_pfirst);
        }
    }
    int status = 0;
    bool marked = false;
    for (int pass = use ? 0 : 1; pass < 2; ++pass) {     // 0: with the points; 1: without (the plain decode)
        const bool indexed = kIndexed && pass == 0;
        if (kIndexed && pass == 1 && use) {              // a marked image: its work so far is thrown away
            uint4* z = reinterpret_cast<uint4*>(coef);
            const int64_t n16 = jpeg_image_blocks(h) * 8;
            for (int64_t k = tid; k < n16; k += kEntropyThreads) z[k] = make_uint4(0, 0, 0, 0);
            status = 0;
            __syncthreads();
        }
        for (int pos = 0; pos < n;) {
            if (tid == 0) {                              // the next group: scans of one wave, tables in kProgSlots
                int ng = 0, slots = 0, items = 0, q = pos;
                const int w = s_scan[s_order[pos]].wave;
                while (q < n && ng < kProgGroup) {
                    const int k = s_order[q];
                    const JpegScan& s = s_scan[k];
                    const int need = jpeg_scan_tables(s);
                    if (s.wave != w || slots + need > kProgSlots) break;
                    s_gscan[ng] = k; s_gslot[ng] = slots; s_gitem[ng] = items;
                    for (int t = 0; t < need; ++t) s_gtab[slots + t] = s.pool[s.ss == 0 ? t : 3];
                    slots += need;
                    items += indexed && s.restart == 0 ? s_pfirst[k + 1] - s_pfirst[k] + 1 : (int)jpeg_scan_segments(h, s);
                    ++ng; ++q;
                }
                s_gitem[ng] = items; s_ng = ng; s_nslot = slots; s_pos = q;
            }
            __syncthreads();
            const int ng = s_ng, nslot = s_nslot, items = s_gitem[ng];
            pos = s_pos;
            if (tid < nslot) jpeg_huff_codes(P.pool[s_gtab[tid]], s_huff[tid]);
            __syncthreads();
            for (int e = tid; e < nslot << kJpegLookBits; e += kEntropyThreads) {
                const int t = e >> kJpegLookBits;
                s_huff[t].look[e & ((1 << kJpegLookBits) - 1)] = jpeg_huff_look(s_huff[t], e & ((1 << kJpegLookBits) - 1));
            }
            __syncthreads();
            bool linked = true;
            for (int it = tid; it < items; it += kEntropyThreads) {
                int g = 0;
                while (it >= s_gitem[g + 1]) ++g;
                const int k = s_gscan[g];
                const JpegScan& s = s_scan[k];
                const int64_t j = it - s_gitem[g], units = jpeg_scan_units(h, s);
                const JpegHuff* hp[3] = {&s_huff[s_gslot[g]], &s_huff[min(s_gslot[g] + 1, kProgSlots - 1)],
                                         &s_huff[min(s_gslot[g] + 2, kProgSlots - 1)]};
                const uint8_t* scan = file + s.off;
                if (indexed && s.restart == 0) {
                    bool ok = true;
                    status |= jpeg_prog_item(h, s, hp, scan, jpeg_prog_axis(s_scan, k), pts + s_pfirst[k],
                                             s_pfirst[k + 1] - s_pfirst[k], (int)j, coef, &ok);
                    linked = linked && ok;
                    continue;
                }
                const int64_t u0 = s.restart > 0 ? j * s.restart : 0, u1 = s.restart > 0 ? min(u0 + s.restart, units) : units;
                const int32_t at = segs[s_seg[k] + j];
                if constexpr (kRecord) {
                    JpegProgSink sink;
                    const bool r = jpeg_prog_indexed(h) && jpeg_prog_sink(h, s_scan, k, s_rec, sink);
                    status |= jpeg_prog_segment(h, s, hp, scan, at < 0 ? scan + s.len : scan + at, scan + s.len, u0, u1,
                                                coef, nullptr, nullptr, r ? &sink : nullptr);
                } else {
                    status |= jpeg_prog_segment(h, s, hp, scan, at < 0 ? scan + s.len : scan + at, scan + s.len, u0, u1, coef);
                }
            }
            // the wave's coefficients are complete; s_huff is free.  An indexed pass stops at the first failed link.
            if (indexed) {
                marked = __syncthreads_or(!linked);
                if (marked) break;
            } else {
                __syncthreads();
            }
        }
        if (!marked) break;
    }
    if (status) atomicOr(&s_status, status);
    __syncthreads();
    if (tid == 0) {
        P.status[img] = s_status;
        if constexpr (kRecord) {                         // points of the rule when it decoded without usable ones
            const bool rec = jpeg_prog_indexed(h) && (!use || marked) && s_status == 0;
            P.count[img] = rec ? jpeg_prog_compact(s_rec, jpeg_index_parts(h), P.rec_points + P.rec_first[img],
                                                   P.rec_first[img + 1] - P.rec_first[img]) : 0;
        } else {
            if (P.count) P.count[img] = 0;              // (a recording call launches the recording instantiation)
        }
    }
}

cudaError_t launch_jpeg_progressive(const JpegDecodeParams& p, cudaStream_t stream) {
    if (p.batch <= 0) return cudaSuccess;
    if (p.rec_first) faa_jpeg_progressive_kernel<true, true><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    else if (p.first) faa_jpeg_progressive_kernel<true, false><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    else faa_jpeg_progressive_kernel<false, false><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_jpeg_index(const JpegDecodeParams& p, cudaStream_t stream) {
    if (p.batch <= 0) return cudaSuccess;
    faa_jpeg_index_kernel<<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_jpeg_entropy(const JpegDecodeParams& p, cudaStream_t stream, bool found) {
    if (p.batch <= 0) return cudaSuccess;
    if (found) faa_jpeg_entropy_kernel<true, true, true><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    else if (p.rec_first) faa_jpeg_entropy_kernel<true, true><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    else if (p.first) faa_jpeg_entropy_kernel<true, false><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    else faa_jpeg_entropy_kernel<false, false><<<(unsigned)p.batch, kEntropyThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_jpeg_reconstruct(const JpegDecodeParams& p, int n_tiles, cudaStream_t stream) {
    if (p.batch <= 0 || n_tiles <= 0) return cudaSuccess;
    faa_jpeg_reconstruct_kernel<<<(unsigned)n_tiles, kReconThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace faa
