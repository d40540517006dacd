// faa_kernels.cu - sm_90a kernels of the augmentation hot path.
//
// Two launches per batch:
//   faa_resolve_kernel   ONE block: per-sample decisions (given records, or drawn with
//                        Philox4x32-10 keyed by (seed, global sample index)) -> a 96-byte
//                        per-image program: the two applied op records, clipped Cutout boxes,
//                        crop / flip / zero-box and the evaluation CLASS of the image; then a
//                        counting sort of the images by estimated cost, so the pixel kernel
//                        starts the expensive images first (LPT order, no tail).
//   faa_augment_kernel   one thread-block CLUSTER per image, one CTA per row band
//                        (cluster dims (bands,1,1), grid (bands, batch)):
//     0. thread 0 stages the CTA's row band (+1 halo row each side) of the raw uint8 HWC image
//        into shared memory with ONE 1-D TMA bulk copy (cp.async.bulk + mbarrier); all pixel
//        reads below hit shared memory when they fall inside the band and global/L2 otherwise;
//     1. ops that need whole-image statistics (AutoContrast / Equalize histogram, Contrast
//        mean luma): each CTA scans its band of the intermediate image, partial statistics are
//        reduced across the cluster through distributed shared memory, every CTA builds the
//        op's 3x256-byte LUT; LUT-only programs are composed into ONE LUT;
//     2. the CTA streams its band of the OUTPUT with the loop specialised for the image's class:
//          PLAIN   12-byte vector reads -> normalise -> 8-byte plane stores
//          LUT     + one composed per-channel LUT lookup
//          POINT   + pointwise ops in registers (Color, Cutout, LUTs)
//          GENERIC tail index map (zero box, flip, crop) -> lazy evaluation of the op chain
//                  back to the raw pixels (16.16 fixed-point gathers, 3x3 Sharpness ...)
//        followed by ToTensor+Normalize and NCHW fp16/bf16/fp32 (or uint8 HWC) vector stores.
//   With a Mixup partner the same evaluation runs for the partner image and the normalised
//   values are mixed in fp32 before the store (aug_mixup.py:21).
//
// Algorithmic HBM bytes per image: 3*H*W read + out_elem*3*out_h*out_w written.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cassert>
#include <cstdlib>
#include <type_traits>
#include <cstring>

#include "faa_kernels.cuh"

namespace cg = cooperative_groups;

namespace faa {

// Opaque re-reads.  The mid and light kernels run their per-entry body inside a loop (persistent rows); everything in the
// body that only depends on the thread index or on constants (index arithmetic, peer shared-memory addresses) is
// loop-invariant, gets hoisted in front of the loop and then lives across the whole body: ~45 spilled registers at the
// 48 / 64-register budgets.  Reading the thread index through a volatile asm per use (an S2R where it is used, as in
// straight-line code) and passing cluster ranks through opaque_u32 keeps those computations where they are written.
__device__ __forceinline__ uint32_t opaque_u32(uint32_t v) { asm volatile("" : "+r"(v)); return v; }
struct OpaqueTid {
    struct X { __device__ __forceinline__ operator unsigned() const { unsigned t; asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t)); return t; } } x;
};
}  // namespace faa
#define threadIdx (::faa::OpaqueTid{})
namespace faa {

constexpr int kThreads = 256;
constexpr int kMaxDevices = 64;
// Resident CTAs per SM of the single-source cluster kernel and of the light kernel (launch bounds; the persistent light
// grid is sized from it).  3 (an 80-register budget) rather than 4 (64 registers): on sm_90a the 64-register build
// spills (light kernel 232 B stores / 808 B loads, cluster kernel 628 / 720 B), and 3 was faster on every bench.py
// workload on an H100 SXM (DESIGN.md 4.3).
#ifndef FAA_MIN_CTAS
#define FAA_MIN_CTAS 3
#endif
constexpr int kCostBuckets = 8;       // per weight class; heavy programs sort before light ones

struct __align__(16) ImgState {
    Prog prog;                  // 96 B
    uint32_t hist[2][768];      // per-slot local partial histograms (read remotely through DSMEM)
    uint32_t tot[768];          // cluster-reduced histogram of the slot being built
    uint8_t lut[2][768];
    uint8_t lutc[768];          // composed LUT (C_LUT programs)
    HistPart parts[3][32];
    unsigned long long suml[2]; // per-slot local partial luma sums
    uint32_t xpart[8];          // scalar statistics of this CTA's band (read remotely through DSMEM): per-channel
                                // min [0..2], max [3..5] (AutoContrast) or the luma sum [6] lo, [7] hi (Contrast)
    uint32_t xtot[8];           // ... reduced over the cluster
    uint32_t wred[16][8];       // per-warp partials (up to 512 threads)
};

struct FastDiv {
    uint32_t d, rcp;
    __device__ __forceinline__ void init(uint32_t dd, uint32_t r) { d = dd; rcp = r; }     // r = recip32(dd), from the host
    __device__ __forceinline__ uint32_t div(uint32_t q) const { return d == 1u ? q : fastdiv(q, rcp); }
};

// ---------------------------------------------------------------------------------------
// launch 1 (main translation unit only; the pixel kernels are compiled once per output type, in parallel:
// -DFAA_TU_OUT=<OutType> builds just launch_out<that type>, see __graft_entry__.build)
#ifndef FAA_TU_OUT
__device__ __forceinline__ int cost_bucket(uint32_t cost) {     // 0 = most expensive
    int b = kCostBuckets - 1;
    uint32_t th = 4u;
    while (b > 0 && cost >= th) { --b; th *= 2u; }
    return b;
}

// kMulti: a multi-policy TTA call (P.cands); entry i takes candidate tta_candidate(i, per_cand)'s table, probabilities
// and n_sub.  The single-policy instantiation is the kernel of every other call.
template <bool kMulti>
__global__ void __launch_bounds__(1024) faa_resolve_kernel(const __grid_constant__ ResolveParams P) {
    __shared__ int s_count[3 * kCostBuckets], s_base[3 * kCostBuckets];
    // let the dependent pixel kernel start launching (its prologue overlaps this kernel)
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (threadIdx.x < 3 * kCostBuckets) s_count[threadIdx.x] = 0;
    if (P.wait_done != nullptr && threadIdx.x == 0) {            // the slot's previous readers (persistent pixel kernels) are done
        uint32_t v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(P.wait_done) : "memory"); } while ((int32_t)(v - P.wait_target) < 0);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < P.n; t += blockDim.x) {
        const int i = P.first + t;
        const OpRec* ops = P.ops;
        const double* probs = P.probs;
        int n_sub = P.n_sub;
        if (kMulti) {
            const PolicyRef c = P.cands[tta_candidate(i, P.per_cand)];
            ops = c.ops; probs = c.probs; n_sub = c.n_sub;
        }
        Sample s;
        Box bx[8];
        if (P.samples != nullptr) {
            s = P.samples[i];
            for (int j = 0; j < P.n_op; ++j) {
                if (P.boxes != nullptr) bx[j] = P.boxes[(size_t)i * P.n_op + j];
                else { bx[j].x0 = bx[j].y0 = 0; bx[j].x1 = bx[j].y1 = -1; }
            }
        } else {
            const uint64_t at = P.pos != nullptr ? (uint64_t)(uint32_t)P.pos[i] : (uint64_t)i;
            philox_sample(P.rng, P.rng.first_index + at, ops, probs, n_sub, P.n_op, P.H, P.W,
                          P.out_h, P.out_w, s, bx);
        }
        if (P.progs != nullptr) {
            Prog g;
            build_prog(s, bx, ops, P.n_op, P.op_base, P.apply_tail, P.H, P.W, P.out_w, P.allow, g);
            lean_order(g, P.allow);
            // weight class: 0 heavy (cluster kernel), 1 mid (statistics / Sharpness kernel, three-way split only), 2 light
            const int wc = !P.split ? 0 : prog_is_light(g, P.allow) ? 2 : (P.split == 2 && prog_is_mid(g, P.allow)) ? 1 : 0;
            g.bucket = (uint8_t)(cost_bucket(prog_cost(g)) + wc * kCostBuckets);
            P.progs[i] = g;
            atomicAdd(&s_count[g.bucket], 1);
        }
        if (P.samples_out != nullptr) P.samples_out[i] = s;
        if (P.boxes_out != nullptr)
            for (int j = 0; j < P.n_op; ++j) P.boxes_out[(size_t)i * P.n_op + j] = bx[j];
    }
    if (P.order == nullptr || P.progs == nullptr) {
        if (P.ready != nullptr) {
            __syncthreads();
            if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(P.ready), "r"(P.ticket) : "memory"); }
        }
        return;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < 3 * kCostBuckets; ++b) {
            // schedule segments: [0, n_heavy[0]) heavy, [n_heavy[0], n_heavy[1]) mid, [n_heavy[1], n) light
            if (b == kCostBuckets && P.n_heavy != nullptr) P.n_heavy[0] = acc;
            if (b == 2 * kCostBuckets && P.n_heavy != nullptr) P.n_heavy[1] = acc;
            s_base[b] = acc; acc += s_count[b]; s_count[b] = 0;
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < P.n; t += blockDim.x) {        // scheduling order only: any order is correct
        const int b = P.progs[P.first + t].bucket;
        P.order[P.first + s_base[b] + atomicAdd(&s_count[b], 1)] = t;
    }
    if (P.ready != nullptr) {                                    // chained steps: the pixel kernels poll this word
        __syncthreads();
        if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(P.ready), "r"(P.ticket) : "memory"); }
    }
}

// ragged launch (faa_augment_ragged): the same decisions -> program step, image i at its own size with its own op
// table and allow bits (imgs[i]); Philox draws global sample rng.first_index + i.  No schedule: the host orders the images.
// kMulti: a multi-policy TTA call; image i draws with candidate cand_of[i]'s probabilities and n_sub (imgs[i].ops is that
// candidate's table at the image's size).
template <bool kMulti>
__global__ void __launch_bounds__(1024) faa_resolve_ragged_kernel(const __grid_constant__ ResolveParams P, const RaggedImg* imgs) {
    for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
        const RaggedImg m = imgs[i];
        const double* probs = P.probs;
        int n_sub = P.n_sub;
        if (kMulti) {
            const PolicyRef c = P.cands[P.cand_of[i]];
            probs = c.probs; n_sub = c.n_sub;
        }
        Sample s;
        Box bx[8];
        if (P.samples != nullptr) {
            s = P.samples[i];
            for (int j = 0; j < P.n_op; ++j) {
                if (P.boxes != nullptr) bx[j] = P.boxes[(size_t)i * P.n_op + j];
                else { bx[j].x0 = bx[j].y0 = 0; bx[j].x1 = bx[j].y1 = -1; }
            }
        } else {
            philox_sample(P.rng, P.rng.first_index + (uint64_t)i, m.ops, probs, n_sub, P.n_op, m.H, m.W, m.H, m.W, s, bx);
        }
        Prog g;
        build_prog(s, bx, m.ops, P.n_op, P.op_base, P.apply_tail, m.H, m.W, m.W, m.allow, g);
        g.bucket = 0;
        P.progs[i] = g;
    }
}

// the library's aligned copies of ragged inputs whose base breaks the word loads: job blockIdx.y, 4 bytes per thread
// and step (the byte count of an image with W % 4 == 0 is a multiple of 12)
__global__ void __launch_bounds__(256) faa_realign_kernel(const RaggedCopy* jobs) {
    const RaggedCopy j = jobs[blockIdx.y];
    uint32_t* dst = reinterpret_cast<uint32_t*>(j.dst);
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < j.bytes / 4; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* s = j.src + 4 * k;
        dst[k] = (uint32_t)__ldg(s) | ((uint32_t)__ldg(s + 1) << 8) | ((uint32_t)__ldg(s + 2) << 16) | ((uint32_t)__ldg(s + 3) << 24);
    }
}

// faa_gather: every job is cut into kGatherUnit-byte pieces and piece u of the whole list (jobs in order) is copied by
// CTA u % gridDim.x, so a multi-MB job is spread over the SMs and a list of 400-byte jobs over the CTAs.  The list is
// read in tiles of kGatherTile jobs: the CTA scans the tile's piece counts into shared memory and finds its pieces'
// jobs by binary search.  Within a piece, src and dst that agree modulo 16 (modulo 4) move 16-byte (4-byte) words after
// a byte head; anything else moves bytes.  No byte outside [dst, dst + bytes) is written.
constexpr int kGatherTile = 1024;

__device__ __forceinline__ void gather_piece(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint64_t n) {
    const int t = threadIdx.x;
    const uintptr_t rel = ((uintptr_t)src ^ (uintptr_t)dst);
    const int vec = (rel & 15) == 0 ? 16 : (rel & 3) == 0 ? 4 : 1;
    uint64_t head = vec == 1 ? 0 : ((uint64_t)vec - ((uintptr_t)dst & (vec - 1))) & (vec - 1);
    if (head > n) head = n;
    const uint64_t body = (n - head) / vec;
    if ((uint64_t)t < head) dst[t] = src[t];
    if (vec == 16) {
        const uint4* s = reinterpret_cast<const uint4*>(src + head);
        uint4* d = reinterpret_cast<uint4*>(dst + head);
        for (uint64_t k = t; k < body; k += kGatherThreads) d[k] = s[k];
    } else if (vec == 4) {
        const uint32_t* s = reinterpret_cast<const uint32_t*>(src + head);
        uint32_t* d = reinterpret_cast<uint32_t*>(dst + head);
        for (uint64_t k = t; k < body; k += kGatherThreads) d[k] = s[k];
    } else {
        for (uint64_t k = t; k < n; k += kGatherThreads) dst[k] = src[k];
        return;
    }
    for (uint64_t k = head + body * vec + t; k < n; k += kGatherThreads) dst[k] = src[k];
}

__global__ void __launch_bounds__(kGatherThreads) faa_gather_kernel(const RaggedCopy* __restrict__ jobs, int n) {
    __shared__ uint64_t s_end[kGatherTile];          // inclusive prefix of the tile's piece counts
    __shared__ uint64_t s_warp[kGatherThreads / 32];
    constexpr int kPer = kGatherTile / kGatherThreads;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    uint64_t before = 0;                             // pieces of the tiles before this one
    for (int base = 0; base < n; base += kGatherTile) {
        uint64_t c[kPer], sum = 0;
#pragma unroll
        for (int q = 0; q < kPer; ++q) {
            const int j = base + t * kPer + q;
            c[q] = j < n ? (jobs[j].bytes + kGatherUnit - 1) / kGatherUnit : 0;
            sum += c[q];
        }
        uint64_t x = sum;                            // inclusive scan of the threads' sums
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        uint64_t off = 0;
        for (int w = 0; w < warp; ++w) off += s_warp[w];
        uint64_t run = off + x - sum;
#pragma unroll
        for (int q = 0; q < kPer; ++q) { run += c[q]; s_end[t * kPer + q] = run; }
        __syncthreads();
        const uint64_t total = s_end[kGatherTile - 1];
        const int m = min(kGatherTile, n - base);
        // the first piece of this tile that is this CTA's: global piece (before + u) % gridDim.x == blockIdx.x
        uint64_t u = ((uint64_t)blockIdx.x + gridDim.x - before % gridDim.x) % gridDim.x;
        for (; u < total; u += gridDim.x) {
            int lo = 0, hi = m - 1;                  // the job whose pieces hold u: first with s_end > u
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (s_end[mid] > u) hi = mid; else lo = mid + 1;
            }
            const RaggedCopy j = jobs[base + lo];
            const uint64_t at = (u - (s_end[lo] - (j.bytes + kGatherUnit - 1) / kGatherUnit)) * kGatherUnit;
            gather_piece(j.src + at, j.dst + at, min(kGatherUnit, j.bytes - at));
        }
        before += total;
        __syncthreads();                             // s_end and s_warp are rewritten by the next tile
    }
}

#endif  // !FAA_TU_OUT

// ---------------------------------------------------------------------------------------
// TMA 1-D bulk copy + mbarrier (sm_90+ PTX; SASS: UBLKCP / SYNCS)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void tma_stage(uint64_t* bar, void* dst, const void* src, uint32_t bytes) {
    const uint32_t b = smem_u32(bar), d = smem_u32(dst);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(d), "l"(src), "r"(bytes), "r"(b) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    const uint32_t b = smem_u32(bar);
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(b), "r"(phase) : "memory");
    }
}

// schedule words (order / counters / programs) are written by the resolve kernel: in the event-ordered schedule that
// kernel has completed (read-only cache is fine); in the chained schedule it may have run concurrently with earlier
// CTAs of this SM, so the loads bypass L1
__device__ __forceinline__ int ld_sched(const int32_t* p, int chain) { return chain ? __ldcg(p) : __ldg(p); }
__device__ __forceinline__ uint32_t ld_sched(const uint32_t* p, int chain) { return chain ? __ldcg(p) : __ldg(p); }

// TTA replicas (search.py:87-125): schedule entry v of a replicated launch augments input image v % in_mod with
// its own decisions; in_mod == 0: one input image per entry
__device__ __forceinline__ uint32_t src_image(const AugParams& P, int idx) {
    return P.in_mod ? (uint32_t)idx % (uint32_t)P.in_mod : (uint32_t)idx;
}

// chained steps: programs / order / n_heavy of this step are complete once *ready == ticket (written with
// release semantics by the resolve kernel, which precedes this kernel in its stream and has therefore started)
__device__ __forceinline__ void wait_ticket(const int32_t* ready, int32_t ticket) {
    if (ready == nullptr) return;
    if (threadIdx.x == 0) {
        int32_t v;
        do { asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(ready) : "memory"); } while (v != ticket);
    }
    __syncthreads();
}

// persistent launches: schedule row y of grid_y visits entries y, 2*grid_y-1-y, 2*grid_y+y, ... of its (cost-sorted)
// segment - the row that drew the most expensive entry of one round gets the cheapest of the next
__device__ __forceinline__ int sched_entry(int k, int y, int gy) { return k * gy + ((k & 1) ? gy - 1 - y : y); }

// a finished CTA counts itself: the resolve kernel that rewrites this slot's programs waits for the total
__device__ __forceinline__ void count_done(uint32_t* done) {
    if (done == nullptr) return;
    __syncthreads();
    if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(done) : "memory");
}

// ---------------------------------------------------------------------------------------
__device__ __forceinline__ Ctx make_ctx(const AugParams& P, const uint8_t* raw, const uint8_t* sraw, uint32_t s_lo, uint32_t s_len,
                                        int H, int W, const ImgState& st, bool full) {
    Ctx c;
    c.rcp_w = P.rcp_w; c.rcp_wq = P.rcp_wq;
    c.raw = raw; c.sraw = sraw; c.s_lo = s_lo; c.s_len2 = s_len > 2u ? s_len - 2u : 0u; c.H = H; c.W = W;
    if (full) {
        c.op[0] = st.prog.op[0]; c.op[1] = st.prog.op[1];
        c.box[0] = st.prog.box[0]; c.box[1] = st.prog.box[1];
    }
    c.lut[0] = st.lut[0]; c.lut[1] = st.lut[1];
    return c;
}

__device__ __forceinline__ void unpack12(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t q[4]) {
    q[0] = w0 & 0xFFFFFFu;
    q[1] = (w0 >> 24) | ((w1 & 0xFFFFu) << 8);
    q[2] = (w1 >> 16) | ((w2 & 0xFFu) << 16);
    q[3] = w2 >> 8;
}

// pointer to byte `off` of the image: the staged copy when [off-4, off+16) is inside it, else global
__device__ __forceinline__ const uint8_t* src_ptr(const Ctx& c, uint32_t off) {
    const uint32_t rel = off - c.s_lo;
    const uint32_t lim = c.s_len2 > 18u ? c.s_len2 - 14u : 0u;          // rel >= 4 and rel + 16 <= staged length
    return (lim >= 4u && rel - 4u < lim - 4u) ? c.sraw + rel : c.raw + off;
}

// 12 contiguous, 4-byte aligned bytes of the raw image at byte offset `off`
__device__ __forceinline__ void load12(const Ctx& c, uint32_t off, uint32_t q[4]) {
    const uint32_t rel = off - c.s_lo;
    const uint32_t lim = c.s_len2 > 9u ? c.s_len2 - 9u : 0u;
    if (rel < lim) {                   // rel + 11 < staged length (no unsigned wrap)
        const uint32_t* w = reinterpret_cast<const uint32_t*>(c.sraw + rel);
        unpack12(w[0], w[1], w[2], q);
    } else {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(c.raw + off);
        unpack12(__ldg(w), __ldg(w + 1), __ldg(w + 2), q);
    }
}

__device__ __forceinline__ void hist_add(uint32_t* hist, uint32_t p) {
    atomicAdd(&hist[p & 255u], 1u);
    atomicAdd(&hist[256u + ((p >> 8) & 255u)], 1u);
    atomicAdd(&hist[512u + (p >> 16)], 1u);
}

// statistics of the image in front of slot L (0 or 1) over rows [y0, y1):
// per-channel histogram and / or the luma sum
template <int L>
__device__ void accumulate_stats(const Ctx& c_in, bool want_hist, bool want_mean, int y0, int y1, uint32_t* hist,
                                 unsigned long long* suml) {
    const Ctx c = c_in;                 // private copy: no local-memory loads through the reference in the loop
    uint32_t local = 0;
    if (L == 0 && (c.W & 3) == 0) {
        // raw image: 4 pixels per thread from 12 aligned bytes
        const uint32_t nq = (uint32_t)(y1 - y0) * (uint32_t)c.W / 4u;
        const uint32_t base = (uint32_t)y0 * (uint32_t)c.W * 3u;
        for (uint32_t i = threadIdx.x; i < nq; i += blockDim.x) {
            uint32_t q[4];
            load12(c, base + 12u * i, q);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (want_mean) local += luma_of(q[k]);
                if (want_hist) hist_add(hist, q[k]);
            }
        }
    } else {
        const uint32_t n = (uint32_t)(y1 - y0) * (uint32_t)c.W;
        FastDiv dw; dw.init((uint32_t)c.W, c.rcp_w);
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            uint32_t r = dw.div(i);
            uint32_t p = Level<L>::at(c, (int)(i - r * c.W), y0 + (int)r);
            if (want_mean) local += luma_of(p);
            if (want_hist) hist_add(hist, p);
        }
    }
    if (want_mean) {
        for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(suml, (unsigned long long)local);
    }
}

// cluster-wide totals of slot j's partial statistics: histogram -> st.tot (every CTA), luma -> mean
static __device__ uint32_t exchange_stats(int bands, uint32_t n_pixels, bool want_hist, bool want_mean, ImgState& st, int j,
                                   cg::cluster_group& cluster) {
    uint32_t mean = 0;
    if (bands > 1) cluster.sync(); else __syncthreads();         // partials complete everywhere
    if (want_hist) {
        if (bands > 1) {
            // reduce-scatter over distributed shared memory: this CTA sums its slice of the 768
            // bins over all ranks and writes the totals into every rank's `tot`
            const int rank = (int)cluster.block_rank();
            const int slice = (768 + bands - 1) / bands;
            for (int i = threadIdx.x; i < slice; i += blockDim.x) {
                const int bin = rank * slice + i;
                if (bin < 768) {
                    // all remote loads in flight together (each is a ~200-cycle DSMEM round trip)
                    uint32_t v[8];
#pragma unroll
                    for (int r = 0; r < 8; ++r) v[r] = r < bands ? cluster.map_shared_rank(&st.hist[j][0], opaque_u32(r))[bin] : 0u;
                    const uint32_t t = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
#pragma unroll
                    for (int r = 0; r < 8; ++r)
                        if (r < bands) cluster.map_shared_rank(&st.tot[0], opaque_u32(r))[bin] = t;
                }
            }
        } else {
            for (int i = threadIdx.x; i < 768; i += blockDim.x) st.tot[i] = st.hist[j][i];
        }
    }
    if (want_mean) {
        unsigned long long t = 0;
        if (bands > 1) {
            unsigned long long v[8];                                // all remote loads in flight together
#pragma unroll
            for (int r = 0; r < 8; ++r) v[r] = r < bands ? *cluster.map_shared_rank(&st.suml[j], opaque_u32(r)) : 0ull;
            t = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
        } else {
            t = st.suml[j];
        }
        mean = contrast_mean(t, n_pixels);
    }
    // totals visible everywhere; after this barrier no CTA touches a peer's shared memory
    if (bands > 1) cluster.sync(); else __syncthreads();
    return mean;
}

// slot j's 3x256 LUT from st.tot (histogram ops) or from the op's parameters (+ mean)
static __device__ void make_lut(uint32_t n_pixels, ImgState& st, int j, uint32_t mean) {
    const OpRec o = st.prog.op[j];
    const int kind = o.kind;
    if (kind_needs_hist(kind)) {
        const int t = threadIdx.x;
        if (t < 96) st.parts[t >> 5][t & 31] = hist_part(&st.tot[(t >> 5) * 256], t & 31);
        __syncthreads();
        if (t < 96)
            hist_lut_lane(kind, &st.tot[(t >> 5) * 256], st.parts[t >> 5], t & 31, n_pixels, &st.lut[j][(t >> 5) * 256]);
    } else {
        for (int i = threadIdx.x; i < 768; i += blockDim.x)
            st.lut[j][i] = (uint8_t)lut_entry_static(o, (uint32_t)(i & 255), mean);
    }
    __syncthreads();
}

__device__ __forceinline__ void zero_stats(ImgState& st) {
    for (int i = threadIdx.x; i < 2 * 768; i += blockDim.x) (&st.hist[0][0])[i] = 0u;
    if (threadIdx.x < 2) st.suml[threadIdx.x] = 0ull;
    __syncthreads();
}

__device__ __forceinline__ void compose_lut(ImgState& st, uint32_t lut_mask) {
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
        uint32_t v = (uint32_t)(i & 255), base = (uint32_t)(i & ~255);
        if (lut_mask & 1u) v = st.lut[0][base + v];
        if (lut_mask & 2u) v = st.lut[1][base + v];
        st.lutc[i] = (uint8_t)v;
    }
    __syncthreads();
}

// everything before the final pass for one (non-MAT) source image
static __device__ bool prepare_image(const AugParams& P, const Ctx& c, int y0, int y1, ImgState& st, cg::cluster_group& cluster) {
    const uint32_t stat_mask = st.prog.stat_mask, lut_mask = st.prog.lut_mask;
    if (lut_mask == 0) return false;
    const uint32_t n_pixels = (uint32_t)P.H * (uint32_t)P.W;
    const int k0 = st.prog.op[0].kind, k1 = st.prog.op[1].kind;
    // histogram op behind LUT ops: raw histogram pushed forward through the first LUT (no 2nd pass)
    const bool push = k0 != K_NONE && kind_is_lutlike(k0) && kind_needs_hist(k1);
    const bool hist0 = kind_needs_hist(k0) || push, mean0 = kind_needs_mean(k0);
    if (stat_mask || push) zero_stats(st);
    if (lut_mask & 1u) {
        uint32_t mean = 0;
        if (hist0 || mean0) {
            accumulate_stats<0>(c, hist0, mean0, y0, y1, st.hist[0], &st.suml[0]);
            mean = exchange_stats(P.bands, n_pixels, hist0, mean0, st, 0, cluster);
        }
        make_lut(n_pixels, st, 0, mean);
    }
    if (lut_mask & 2u) {
        uint32_t mean = 0;
        if (push) {
            // st.tot holds the cluster totals of the raw histogram; hist[1] is zero
            for (int i = threadIdx.x; i < 768; i += blockDim.x)
                atomicAdd(&st.hist[1][(i & ~255) + st.lut[0][i]], st.tot[i]);
            __syncthreads();
            for (int i = threadIdx.x; i < 768; i += blockDim.x) st.tot[i] = st.hist[1][i];
            __syncthreads();
        } else if ((stat_mask >> 1) & 1u) {      // lazy fallback (no materialisation chunk available)
            accumulate_stats<1>(c, kind_needs_hist(k1), kind_needs_mean(k1), y0, y1, st.hist[1], &st.suml[1]);
            mean = exchange_stats(P.bands, n_pixels, kind_needs_hist(k1), kind_needs_mean(k1), st, 1, cluster);
        }
        make_lut(n_pixels, st, 1, mean);
    }
    if (st.prog.cls == C_LUT) compose_lut(st, lut_mask);
    return stat_mask != 0;
}

// ---------------------------------------------------------------------------------------
// final pass building blocks
struct TailInfo {
    int crop_dy, crop_dx, flip;
    int zb0, zb1, zb2, zb3;      // zero box rows [zb0,zb1) x cols [zb2,zb3); empty when off
};

__device__ __forceinline__ TailInfo make_tail(const AugParams& P, const Prog& g) {
    TailInfo t;
    t.crop_dy = g.crop_dy; t.crop_dx = g.crop_dx; t.flip = g.flip;
    const bool on = P.use_zero_box != 0;
    t.zb0 = on ? g.zero_box[0] : 0; t.zb1 = on ? g.zero_box[1] : 0;
    t.zb2 = on ? g.zero_box[2] : 0; t.zb3 = on ? g.zero_box[3] : 0;
    return t;
}

__device__ __forceinline__ uint32_t zero_mask(const TailInfo& t, int ox0, int oy) {
    if (oy < t.zb0 || oy >= t.zb1) return 0u;
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) m |= (uint32_t)(ox0 + k >= t.zb2 && ox0 + k < t.zb3) << k;
    return m;
}

// one pointwise op with its kind known at compile time (PK: 0 none, 1 LUT, 2 Color, 3 Cutout)
template <int PK>
__device__ __forceinline__ uint32_t point_op(const Ctx& c, int j, uint32_t p, int x, int y) {
    if (PK == 1) return apply_lut(c.lut[j], p);
    if (PK == 2) return color_px(p, bits_to_float(c.op[j].a[0]), c.op[j].a[1] != 0);
    if (PK == 3) { const Box& b = c.box[j]; return (x >= b.x0 && x <= b.x1 && y >= b.y0 && y <= b.y1) ? kCutoutRGB : p; }
    return p;
}
__device__ __forceinline__ int point_kind(int k) { return k == K_NONE ? 0 : k == K_COLOR ? 2 : k == K_CUTOUT ? 3 : 1; }

template <int PK0, int PK1>
__device__ __forceinline__ void point4(const Ctx& c, uint32_t q[4], int sx0, int ay) {
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = point_op<PK1>(c, 1, point_op<PK0>(c, 0, q[k], sx0 + k, ay), sx0 + k, ay);
}
// CTA-uniform dispatch on the two slots' pointwise kinds (pv = 4 * kind0 + kind1)
__device__ __forceinline__ void point4_any(int pv, const Ctx& c, uint32_t q[4], int sx0, int ay) {
    switch (pv) {
    case 1: point4<0, 1>(c, q, sx0, ay); break;   case 2: point4<0, 2>(c, q, sx0, ay); break;
    case 3: point4<0, 3>(c, q, sx0, ay); break;   case 4: point4<1, 0>(c, q, sx0, ay); break;
    case 5: point4<1, 1>(c, q, sx0, ay); break;   case 6: point4<1, 2>(c, q, sx0, ay); break;
    case 7: point4<1, 3>(c, q, sx0, ay); break;   case 8: point4<2, 0>(c, q, sx0, ay); break;
    case 9: point4<2, 1>(c, q, sx0, ay); break;   case 10: point4<2, 2>(c, q, sx0, ay); break;
    case 11: point4<2, 3>(c, q, sx0, ay); break;  case 12: point4<3, 0>(c, q, sx0, ay); break;
    case 13: point4<3, 1>(c, q, sx0, ay); break;  case 14: point4<3, 2>(c, q, sx0, ay); break;
    case 15: point4<3, 3>(c, q, sx0, ay); break;  default: break;
    }
}

// aligned classes: the four source pixels of an output quad are 12 contiguous bytes.
// `slot` is the op slot a C_SHARP program's Sharpness sits in (0) / its pointwise follower (1).
// STAGED (C_SHARP): the three source rows of every quad of the band are inside the staged copy
template <int CLS, bool STAGED = false>
__device__ __forceinline__ void quad_vec(const Ctx& c, const uint8_t* lutc, const TailInfo& t, int out_w, int ox0,
                                         int oy, uint32_t px[4], int pv = 0) {
    const int sx0 = (t.flip ? (out_w - 4 - ox0) : ox0) + t.crop_dx;
    const int ay = oy + t.crop_dy;
    uint32_t q[4] = {0u, 0u, 0u, 0u};
    if ((unsigned)sx0 < (unsigned)c.W && (unsigned)ay < (unsigned)c.H) {
        const uint32_t off = (uint32_t)(ay * c.W + sx0) * 3u;
        if (CLS == C_SHARP) {
            const uint32_t pitch = (uint32_t)c.W * 3u;
            const bool rowb = ay == 0 || ay == c.H - 1;
            const uint8_t* r0 = STAGED ? c.sraw + (off - c.s_lo) : src_ptr(c, off);
            const uint8_t* rm = rowb ? r0 : (STAGED ? r0 - pitch : src_ptr(c, off - pitch));
            const uint8_t* rp = rowb ? r0 : (STAGED ? r0 + pitch : src_ptr(c, off + pitch));
            sharp_quad(rm, r0, rp, sx0 > 0, sx0 + 4 < c.W, rowb, sx0 == 0, sx0 + 4 == c.W,
                       bits_to_float(c.op[0].a[0]), c.op[0].a[1] != 0, q);
            if (pv) {                                   // CTA-uniform: a pointwise op follows the Sharpness
#pragma unroll
                for (int k = 0; k < 4; ++k) q[k] = apply_pointwise(c, 1, q[k], sx0 + k, ay);
            }
        } else {
            load12(c, off, q);
            if (CLS == C_LUT) {
#pragma unroll
                for (int k = 0; k < 4; ++k) q[k] = apply_lut(lutc, q[k]);
            } else if (CLS == C_POINT) {
                point4_any(pv, c, q, sx0, ay);
            }
        }
    }
    if (t.flip) { px[0] = q[3]; px[1] = q[2]; px[2] = q[1]; px[3] = q[0]; }
    else { px[0] = q[0]; px[1] = q[1]; px[2] = q[2]; px[3] = q[3]; }
}

// C_GEOM: exactly one geometric op (slot g) and otherwise pointwise ops: the fixed-point source
// coordinate is stepped along the quad instead of being re-derived per pixel
// The geometric op of a C_GEOM / C_SG program as plain registers (no indexed access to the op array).
struct GeomOp {
    int a0, a1, a2, a3, a4, a5;   // K_AFFINE: 16.16 coefficients; K_SHIFT: a0=dx a1=dy a2=bx a3=by
    int pk;                       // kind of the pointwise op in the other slot (K_NONE: nothing)
};

// Branch-free fetch of source pixel (x, y) when `ok` (else 0): the staged copy or global memory through ONE
// generic pointer, so the twelve byte loads of a quad issue back to back - one exposed load latency per
// quad instead of one per pixel (a warp issues in order and would stall at each pixel's first use).
__device__ __forceinline__ uint32_t load_raw_sel(const Ctx& c, int x, int y, bool ok) {
    const uint32_t off = ok ? (uint32_t)(y * c.W + x) * 3u : 0u;
    const uint32_t rel = off - c.s_lo;
    const uint8_t* p = (rel < c.s_len2) ? c.sraw + rel : c.raw + off;
    const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
    return ok ? v : 0u;
}

// G = slot of the geometric op, AFF = it is a K_AFFINE (else K_SHIFT), SIMPLE = the tail is the identity
// apart from the flip (no crop, out size == image size, out_w % 4 == 0): every pixel of the quad exists.
// COH: the source is the scratch image written by this kernel (plain loads behind the cluster barrier:
// the barrier's fence invalidates L1, so they are coherent with the peers' stores and still L1-cached).
// NB: the branch-free fetch (latency-bound cluster kernel); the streaming kernel has enough warps in flight
// and is issue-bound, there the branchy per-pixel fetch (fewer instructions) is faster.
template <int G, bool AFF, bool SIMPLE, bool COH, bool NB>
__device__ __forceinline__ void quad_geom(const Ctx& c, const GeomOp& o, const TailInfo& t, int out_w, int ox0, int oy,
                                          uint32_t px[4]) {
    const int ay = SIMPLE ? oy : oy + t.crop_dy;
    const int ax0 = (t.flip ? (out_w - 1 - ox0) : ox0) + (SIMPLE ? 0 : t.crop_dx);
    const int sx = t.flip ? -1 : 1;
    const bool row_ok = SIMPLE || (unsigned)ay < (unsigned)c.H;
    int fx = 0, fy = 0, dfx = 0, dfy = 0;               // 16.16 source coordinates of pixel k = 0 and their step
    if (AFF) {
        fx = o.a2 + o.a0 * ax0 + o.a1 * ay; fy = o.a5 + o.a3 * ax0 + o.a4 * ay;
        dfx = sx * o.a0; dfy = sx * o.a3;
    }
    const int ysh = AFF ? 0 : ay + o.a1 + (ay >= o.a3);
    if (!NB) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int ax = ax0 + sx * k;
            uint32_t p = 0u;
            const bool have = SIMPLE || (row_ok && (unsigned)ax < (unsigned)c.W && ox0 + k < out_w);
            if (have) {                                      // (ax, ay) is a pixel of the augmented image
                int xs, ys;
                if (AFF) { xs = (fx + k * dfx) >> 16; ys = (fy + k * dfy) >> 16; }
                else { xs = ax + o.a0 + (ax >= o.a2); ys = ysh; }
                if ((unsigned)xs < (unsigned)c.W && (unsigned)ys < (unsigned)c.H) {
                    p = load_raw(c, xs, ys);
                    if (G == 1 && o.pk != K_NONE) p = apply_pointwise(c, 0, p, xs, ys);     // op0 ran before the gather
                }
                if (G == 0 && o.pk != K_NONE) p = apply_pointwise(c, 1, p, ax, ay);         // op1 runs after it (fill included)
            }
            px[k] = p;
        }
        return;
    }
    uint32_t have_m = 0, ins_m = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {                        // 1. the four fetches, no branches in between
        const int ax = ax0 + sx * k;
        const bool have = SIMPLE || (row_ok && (unsigned)ax < (unsigned)c.W && ox0 + k < out_w);   // a pixel of the augmented image
        int xs, ys;
        if (AFF) { xs = (fx + k * dfx) >> 16; ys = (fy + k * dfy) >> 16; }
        else { xs = ax + o.a0 + (ax >= o.a2); ys = ysh; }
        const bool ins = have && (unsigned)xs < (unsigned)c.W && (unsigned)ys < (unsigned)c.H;
        px[k] = load_raw_sel(c, xs, ys, ins);
        have_m |= (uint32_t)have << k; ins_m |= (uint32_t)ins << k;
    }
    if (o.pk != K_NONE) {                                // 2. the pointwise op of the other slot (CTA-uniform)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int ax = ax0 + sx * k;
            if (G == 1) {                                // op0 ran before the gather: at the source position
                int xs, ys;
                if (AFF) { xs = (fx + k * dfx) >> 16; ys = (fy + k * dfy) >> 16; }
                else { xs = ax + o.a0 + (ax >= o.a2); ys = ysh; }
                if ((ins_m >> k) & 1u) px[k] = apply_pointwise(c, 0, px[k], xs, ys);
            } else {                                     // op1 runs after it (fill included)
                if ((have_m >> k) & 1u) px[k] = apply_pointwise(c, 1, px[k], ax, ay);
            }
        }
    }
}

// runtime -> compile-time dispatch of the variants (CTA-uniform), one call per quad
template <bool COH, bool NB>
__device__ __forceinline__ void quad_geom_any(int variant, const Ctx& c, const GeomOp& o, const TailInfo& t, int out_w,
                                              int ox0, int oy, uint32_t px[4]) {
    switch (variant) {
    case 0: quad_geom<0, false, false, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 1: quad_geom<0, false, true, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 2: quad_geom<0, true, false, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 3: quad_geom<0, true, true, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 4: quad_geom<1, false, false, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 5: quad_geom<1, false, true, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    case 6: quad_geom<1, true, false, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    default: quad_geom<1, true, true, COH, NB>(c, o, t, out_w, ox0, oy, px); break;
    }
}

__device__ __forceinline__ int geom_setup(const Ctx& c, const TailInfo& t, int H, int W, int out_h, int out_w, GeomOp& o) {
    const bool g0 = c.op[0].kind == K_AFFINE || c.op[0].kind == K_SHIFT;
    const OpRec& r = g0 ? c.op[0] : c.op[1];
    o.a0 = r.a[0]; o.a1 = r.a[1]; o.a2 = r.a[2]; o.a3 = r.a[3]; o.a4 = r.a[4]; o.a5 = r.a[5];
    o.pk = g0 ? c.op[1].kind : c.op[0].kind;
    const bool simple = t.crop_dx == 0 && t.crop_dy == 0 && out_h == H && out_w == W && (out_w & 3) == 0;
    return (g0 ? 0 : 4) + (r.kind == K_AFFINE ? 2 : 0) + (simple ? 1 : 0);
}

__device__ __forceinline__ void quad_generic(const Ctx& c, const TailInfo& t, int out_w, int ox0, int oy, uint32_t px[4]) {
    const int ay = oy + t.crop_dy;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int ox = ox0 + k;
        px[k] = 0u;
        const int ax = (t.flip ? (out_w - 1 - ox) : ox) + t.crop_dx;
        if (ox < out_w && (unsigned)ax < (unsigned)c.W && (unsigned)ay < (unsigned)c.H) px[k] = Level<2>::at(c, ax, ay);
    }
}

template <int OUT> struct OutElem { using T = float; };
template <> struct OutElem<OUT_F16> { using T = __half; };
template <> struct OutElem<OUT_BF16> { using T = __nv_bfloat16; };
template <> struct OutElem<OUT_U8_HWC> { using T = uint8_t; };

// ---- output addressing of the lean paths.  Planar float outputs step ONE element per pixel and `plane` elements per
// channel; the uint8 HWC output (Mixup exchange, PIL surface) steps three bytes per pixel.  With OUT_U8_HWC the values the
// paths produce are the augmented BYTES (identity "normalisation": scale 1, bias 0; float tables hold byte values).
template <int OUT> struct PixStep { static constexpr uint32_t v = OUT == OUT_U8_HWC ? 3u : 1u; };
constexpr float kBias15 = 12582912.0f;           // 1.5 * 2^23: float(kBias15 + i) is exact for |i| < 2^22
constexpr uint32_t kBias15Bits = 0x4B400000u;
// a float holding an integer 0..255 -> that integer (no F2I: the conversion unit is 1/8 rate)
__device__ __forceinline__ uint32_t f2b(float v) { return __float_as_uint(__fadd_rn(v, kBias15)) & 255u; }
__device__ __forceinline__ uint32_t pack4(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3) { return b0 | (b1 << 8) | (b2 << 16) | (b3 << 24); }
// 24 bytes = 8 pixels in output order (8-byte aligned: W % 8 == 0) / 12 bytes = 4 pixels (4-byte aligned)
__device__ __forceinline__ void store_oct_u8(uint8_t* o, const uint32_t b[24]) {
    uint2* q = reinterpret_cast<uint2*>(o);
#pragma unroll
    for (int j = 0; j < 3; ++j) q[j] = make_uint2(pack4(b[8 * j], b[8 * j + 1], b[8 * j + 2], b[8 * j + 3]), pack4(b[8 * j + 4], b[8 * j + 5], b[8 * j + 6], b[8 * j + 7]));
}
__device__ __forceinline__ void store_quad_u8(uint8_t* o, const uint32_t b[12]) {
    uint32_t* q = reinterpret_cast<uint32_t*>(o);
#pragma unroll
    for (int j = 0; j < 3; ++j) q[j] = pack4(b[4 * j], b[4 * j + 1], b[4 * j + 2], b[4 * j + 3]);
}

template <int OUT>
__device__ __forceinline__ void store_plane4(typename OutElem<OUT>::T* o, const float v[4], bool vec, int nvalid) {
    if constexpr (OUT == OUT_U8_HWC) {
        (void)o; (void)v; (void)vec; (void)nvalid;                   // (uint8 HWC goes through store_quad_u8 / emit_quad)
    } else if (vec) {
        if constexpr (OUT == OUT_F32) {
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        } else if constexpr (OUT == OUT_F16) {
            __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
            uint2 u; u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
            *reinterpret_cast<uint2*>(o) = u;
        } else {
            __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
            uint2 u; u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
            *reinterpret_cast<uint2*>(o) = u;
        }
    } else {
        for (int k = 0; k < nvalid; ++k) {
            if constexpr (OUT == OUT_F32) o[k] = v[k];
            else if constexpr (OUT == OUT_F16) o[k] = __float2half_rn(v[k]);
            else o[k] = __float2bfloat16_rn(v[k]);
        }
    }
}

template <bool TAB>
__device__ __forceinline__ float normalise(const AugParams& P, const float* s_norm, int ch, uint32_t u) {
    if (TAB) return s_norm[ch * 256 + u];
    return fmaf((float)u, P.scale[ch], P.bias[ch]);
}

// normalise + store one quad (single source); the CutoutDefault box is re-zeroed afterwards (zero_box_rows)
template <int OUT, bool TAB>
__device__ __forceinline__ void emit_quad(const AugParams& P, const float* s_norm, void* out_img, int ox0, int oy,
                                          const uint32_t px[4], bool vec) {
    const int nvalid = min(4, P.out_w - ox0);           // a static bound of 4 keeps the tail stores unrolled
    if constexpr (OUT == OUT_U8_HWC) {
        uint8_t* o = reinterpret_cast<uint8_t*>(out_img) + (uint32_t)(oy * P.out_w + ox0) * 3u;
        if (vec) {
            uint32_t* w = reinterpret_cast<uint32_t*>(o);
            w[0] = px[0] | (px[1] << 24);
            w[1] = (px[1] >> 8) | (px[2] << 16);
            w[2] = (px[2] >> 16) | (px[3] << 8);
        } else {
            for (int k = 0; k < nvalid; ++k) {
                o[3 * k] = (uint8_t)px[k]; o[3 * k + 1] = (uint8_t)(px[k] >> 8); o[3 * k + 2] = (uint8_t)(px[k] >> 16);
            }
        }
    } else {
        using T = typename OutElem<OUT>::T;
        const uint32_t plane = (uint32_t)P.out_h * (uint32_t)P.out_w;
        T* o = reinterpret_cast<T*>(out_img) + (uint32_t)(oy * P.out_w + ox0);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = normalise<TAB>(P, s_norm, ch, (px[k] >> (8 * ch)) & 255u);
            store_plane4<OUT>(o + ch * plane, v, vec, nvalid);
        }
    }
}

// are all source rows of output rows [oy0, oy1) inside the staged copy of the band?
__device__ __forceinline__ bool band_fully_staged(const Ctx& c, const TailInfo& t, int oy0, int oy1) {
    const int a0 = max(oy0 + t.crop_dy, 0), a1 = min(oy1 + t.crop_dy, c.H);        // source rows [a0, a1)
    if (a1 <= a0) return true;
    const uint32_t pitch = (uint32_t)c.W * 3u, s_len = c.s_len2 ? c.s_len2 + 2u : 0u;
    return s_len != 0u && (uint32_t)a0 * pitch >= c.s_lo && (uint32_t)a1 * pitch <= c.s_lo + s_len;
}

// output rows [oy0, oy1) of one image through the class-specialised evaluator
template <int OUT, bool TAB, int CLS, bool NB = true>
__device__ __forceinline__ void final_rows(const AugParams& P, const float* s_norm, const Ctx& c, const uint8_t* lutc,
                                           const TailInfo& t, void* out_img, int oy0, int oy1) {
    const uint32_t qpr = (uint32_t)(P.out_w + 3) >> 2;
    const uint32_t nq = (uint32_t)(oy1 - oy0) * qpr;
    FastDiv dq; dq.init(qpr, P.rcp_out_qpr);
    // aligned classes exist only when out_w % 4 == 0 (build_prog)
    const bool vec = (CLS == C_PLAIN || CLS == C_LUT || CLS == C_POINT || CLS == C_SHARP) ? true : (P.out_w & 3) == 0;
    // incremental (row, quad) walk: one division up front, adds afterwards
    uint32_t r = dq.div(threadIdx.x), qx = threadIdx.x - r * qpr;
    const uint32_t dr = dq.div(blockDim.x), dx = blockDim.x - dr * qpr;
    GeomOp go; int gv = 0;
    if (CLS == C_GEOM || CLS == C_SG) gv = geom_setup(c, t, P.H, P.W, P.out_h, P.out_w, go);
    if (CLS == C_POINT) gv = 4 * point_kind(c.op[0].kind) + point_kind(c.op[1].kind);
    if (CLS == C_SHARP) gv = c.op[1].kind != K_NONE;
    const bool staged = CLS == C_SHARP && band_fully_staged(c, t, oy0 - 1, oy1 + 1);
    for (uint32_t q = threadIdx.x; q < nq; q += blockDim.x) {
        const int ox0 = (int)qx * 4;
        const int oy = oy0 + (int)r;
        uint32_t px[4];
        if (CLS == C_GENERIC) quad_generic(c, t, P.out_w, ox0, oy, px);
        else if (CLS == C_GEOM) quad_geom_any<false, NB>(gv, c, go, t, P.out_w, ox0, oy, px);
        else if (CLS == C_SG) quad_geom_any<true, true>(gv, c, go, t, P.out_w, ox0, oy, px);
        else if (CLS == C_SHARP && staged) quad_vec<CLS, true>(c, lutc, t, P.out_w, ox0, oy, px, gv);
        else quad_vec<CLS>(c, lutc, t, P.out_w, ox0, oy, px, gv);
        emit_quad<OUT, TAB>(P, s_norm, out_img, ox0, oy, px, vec);
        qx += dx; r += dr;
        if (qx >= qpr) { qx -= qpr; ++r; }
    }
}

// CutoutDefault (data.py:235-250) for single-source launches: after its final pass the CTA re-zeroes its
// rows of the image's box (zero on the normalised tensor; byte zero for the raw uint8 output)
template <int OUT>
__device__ __forceinline__ void zero_box_rows(const AugParams& P, const Prog& g, void* out_img, int oy0, int oy1) {
    if (!P.use_zero_box) return;
    const int r0 = max((int)g.zero_box[0], oy0), r1 = min((int)g.zero_box[1], oy1);
    const int c0 = max((int)g.zero_box[2], 0), c1 = min((int)g.zero_box[3], P.out_w);
    const int bw = c1 - c0, n = bw * (r1 - r0);
    if (bw <= 0 || r1 <= r0) return;                    // CTA-uniform
    __syncthreads();                                    // the final pass's stores are ordered before these
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int r = r0 + i / bw, x = c0 + i % bw;
        if constexpr (OUT == OUT_U8_HWC) {
            uint8_t* o = reinterpret_cast<uint8_t*>(out_img) + (uint32_t)(r * P.out_w + x) * 3u;
            o[0] = 0; o[1] = 0; o[2] = 0;
        } else {
            using T = typename OutElem<OUT>::T;
            const uint32_t plane = (uint32_t)P.out_h * (uint32_t)P.out_w;
            T* o = reinterpret_cast<T*>(out_img) + (uint32_t)(r * P.out_w + x);
            o[0] = T(0.0f); o[plane] = T(0.0f); o[2u * plane] = T(0.0f);
        }
    }
}

// ---- streaming loop of the PLAIN / LUT classes -------------------------------------------------
// When every source row of the band is staged, the twelve bytes of a quad go straight from the staged
// words to the three planes: value = tab[ch][byte] (LUT composed with the normalisation) or the fma.

template <int OUT, bool USE_TAB, bool FLIP>
__device__ __forceinline__ void stream_quad(const AugParams& P, const uint32_t* w, const float* tab,
                                            typename OutElem<OUT>::T* o, uint32_t plane) {
    const uint32_t w3[3] = {w[0], w[1], w[2]};
    if constexpr (OUT == OUT_U8_HWC) {
        if (!USE_TAB && !FLIP) {
            uint32_t* q = reinterpret_cast<uint32_t*>(o);
            q[0] = w3[0]; q[1] = w3[1]; q[2] = w3[2];
        } else {
            uint32_t ob[12];
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const int b = 3 * (FLIP ? 3 - k : k) + ch;
                    const uint32_t u = (w3[b >> 2] >> (8 * (b & 3))) & 255u;
                    ob[3 * k + ch] = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
                }
            store_quad_u8(o, ob);
        }
    } else {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int b = 3 * (FLIP ? 3 - k : k) + ch;                  // which of the 12 bytes
            const uint32_t u = (w3[b >> 2] >> (8 * (b & 3))) & 255u;
            v[k] = USE_TAB ? tab[ch * 256 + u] : fmaf((float)u, P.scale[ch], P.bias[ch]);
        }
        store_plane4<OUT>(o + ch * plane, v, true, 4);
    }
    }
}

// pad[ch] = normalised value of a zero byte (RandomCrop padding is applied to the augmented image)
template <int OUT, bool USE_TAB>
__device__ __forceinline__ void final_rows_stream(const AugParams& P, const float* tab, const float pad[3], const Ctx& c,
                                                  const TailInfo& t, void* out_img, int oy0, int oy1) {
    using T = typename OutElem<OUT>::T;
    const uint32_t qpr = (uint32_t)P.out_w >> 2;
    const uint32_t nq = (uint32_t)(oy1 - oy0) * qpr;
    FastDiv dq; dq.init(qpr, P.rcp_out_qpr);
    uint32_t r = dq.div(threadIdx.x), qx = threadIdx.x - r * qpr;
    const uint32_t dr = dq.div(blockDim.x), dx = blockDim.x - dr * qpr;
    const uint32_t plane = (uint32_t)P.out_h * (uint32_t)P.out_w;
    const bool flip = t.flip != 0;
    for (uint32_t q = threadIdx.x; q < nq; q += blockDim.x) {
        const int ox0 = (int)qx * 4, oy = oy0 + (int)r;
        const int sx0 = (flip ? (P.out_w - 4 - ox0) : ox0) + t.crop_dx, ay = oy + t.crop_dy;
        T* o = reinterpret_cast<T*>(out_img) + PixStep<OUT>::v * (uint32_t)(oy * P.out_w + ox0);
        if ((unsigned)sx0 < (unsigned)c.W && (unsigned)ay < (unsigned)c.H) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(c.sraw + ((uint32_t)(ay * c.W + sx0) * 3u - c.s_lo));
            if (flip) stream_quad<OUT, USE_TAB, true>(P, w, tab, o, plane);
            else stream_quad<OUT, USE_TAB, false>(P, w, tab, o, plane);
        } else if constexpr (OUT == OUT_U8_HWC) {
            uint32_t ob[12];
#pragma unroll
            for (int k = 0; k < 12; ++k) ob[k] = f2b(pad[k % 3]);
            store_quad_u8(o, ob);
        } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float v[4] = {pad[ch], pad[ch], pad[ch], pad[ch]};
                store_plane4<OUT>(o + ch * plane, v, true, 4);
            }
        }
        qx += dx; r += dr;
        if (qx >= qpr) { qx -= qpr; ++r; }
    }
}

// ---- octet (8-pixel) streaming: W % 8 == 0, output size == image size, no crop --------------------
// Eight consecutive pixels of one row are 24 contiguous, 8-byte aligned bytes; each plane gets ONE 16-byte
// store (fp16 / bf16) and the normalisation is one fused multiply-add per value.
template <int OUT>
__device__ __forceinline__ void store_plane8(typename OutElem<OUT>::T* o, const float v[8]) {
    if constexpr (OUT == OUT_U8_HWC) {
        (void)o; (void)v;                                            // (uint8 HWC goes through store_oct_u8)
    } else if constexpr (OUT == OUT_F32) {
        reinterpret_cast<float4*>(o)[0] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4*>(o)[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else if constexpr (OUT == OUT_F16) {
        __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
        __half2 c = __floats2half2_rn(v[4], v[5]), d = __floats2half2_rn(v[6], v[7]);
        uint4 u; u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
        u.z = *reinterpret_cast<uint32_t*>(&c); u.w = *reinterpret_cast<uint32_t*>(&d);
        *reinterpret_cast<uint4*>(o) = u;
    } else {
        __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
        __nv_bfloat162 c = __floats2bfloat162_rn(v[4], v[5]), d = __floats2bfloat162_rn(v[6], v[7]);
        uint4 u; u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
        u.z = *reinterpret_cast<uint32_t*>(&c); u.w = *reinterpret_cast<uint32_t*>(&d);
        *reinterpret_cast<uint4*>(o) = u;
    }
}

// normalised values of one plane from eight byte values: table lookups, or fma
template <bool USE_TAB>
__device__ __forceinline__ void norm8(const AugParams& P, const float* tab, int ch, const uint32_t u[8], float v[8]) {
    if (USE_TAB) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = tab[ch * 256 + u[k]];
    } else {
        const float sc = P.scale[ch], bi = P.bias[ch];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __fmaf_rn((float)u[k], sc, bi);
    }
}

// w[6]: the 24 source bytes of the octet in memory order; FLIP reverses the pixel order
template <int OUT, bool USE_TAB, bool FLIP>
__device__ __forceinline__ void stream_oct(const AugParams& P, const uint32_t w[6], const float* tab,
                                           typename OutElem<OUT>::T* o, uint32_t plane) {
    if constexpr (OUT == OUT_U8_HWC) {
        if (!USE_TAB && !FLIP) {                                     // the bytes themselves
            uint2* q = reinterpret_cast<uint2*>(o);
            q[0] = make_uint2(w[0], w[1]); q[1] = make_uint2(w[2], w[3]); q[2] = make_uint2(w[4], w[5]);
        } else {
            uint32_t ob[24];
#pragma unroll
            for (int k = 0; k < 8; ++k)
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const int b = 3 * (FLIP ? 7 - k : k) + ch;
                    const uint32_t u = (w[b >> 2] >> (8 * (b & 3))) & 255u;
                    ob[3 * k + ch] = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
                }
            store_oct_u8(o, ob);
        }
    } else {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        uint32_t u[8]; float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int b = 3 * (FLIP ? 7 - k : k) + ch;                  // which of the 24 bytes
            u[k] = (w[b >> 2] >> (8 * (b & 3))) & 255u;
        }
        norm8<USE_TAB>(P, tab, ch, u, v);
        store_plane8<OUT>(o + ch * plane, v);
    }
    }
}

// px[8]: eight 24-bit pixels already in OUTPUT order
template <int OUT, bool TAB>
__device__ __forceinline__ void emit_oct(const AugParams& P, const float* s_norm, typename OutElem<OUT>::T* o, uint32_t plane,
                                         const uint32_t px[8]) {
    if constexpr (OUT == OUT_U8_HWC) {                               // (TAB: a LUT's table of byte values)
        uint32_t ob[24];
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const uint32_t u = (px[k] >> (8 * ch)) & 255u;
                ob[3 * k + ch] = TAB ? f2b(s_norm[ch * 256 + u]) : u;
            }
        store_oct_u8(o, ob);
    } else {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        uint32_t u[8]; float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) u[k] = (px[k] >> (8 * ch)) & 255u;
        norm8<TAB>(P, s_norm, ch, u, v);
        store_plane8<OUT>(o + ch * plane, v);
    }
    }
}

// the launch geometry allows octets: W % 8 == 0 and the output is the (possibly mirrored) image itself
__device__ __forceinline__ bool octet_geometry(const AugParams& P, const TailInfo& t) {
    return P.octets != 0 && t.crop_dx == 0 && t.crop_dy == 0;      // P.octets: W % 8 == 0, out size == image size, 16-byte aligned output
}

template <int OUT, bool USE_TAB, bool FLIP>
__device__ __forceinline__ void final_rows_stream8(const AugParams& P, const float* tab, const Ctx& c, void* out_img,
                                                   int oy0, int oy1) {
    using T = typename OutElem<OUT>::T;
    const uint32_t opr = (uint32_t)P.W >> 3;                      // octets per row
    const uint32_t n8 = (uint32_t)(oy1 - oy0) * opr;
    const uint32_t plane = (uint32_t)P.H * (uint32_t)P.W;
    const uint8_t* src = c.sraw + ((uint32_t)oy0 * (uint32_t)P.W * 3u - c.s_lo);   // first byte of row oy0 (staged)
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)P.W;
    if (!FLIP) {                                                  // source and output both advance linearly
        for (uint32_t i = threadIdx.x; i < n8; i += blockDim.x) {
            const uint2* s8 = reinterpret_cast<const uint2*>(src + 24u * i);
            const uint2 a = s8[0], b = s8[1], d = s8[2];
            const uint32_t w[6] = {a.x, a.y, b.x, b.y, d.x, d.y};
            stream_oct<OUT, USE_TAB, false>(P, w, tab, dst + PS * 8u * i, plane);
        }
    } else {
        FastDiv dq; dq.init(opr, P.rcp_opr);
        uint32_t r = dq.div(threadIdx.x), ox = threadIdx.x - r * opr;
        const uint32_t dr = dq.div(blockDim.x), dx = blockDim.x - dr * opr;
        for (uint32_t i = threadIdx.x; i < n8; i += blockDim.x) {
            const uint2* s8 = reinterpret_cast<const uint2*>(src + 24u * (r * opr + (opr - 1u - ox)));
            const uint2 a = s8[0], b = s8[1], d = s8[2];
            const uint32_t w[6] = {a.x, a.y, b.x, b.y, d.x, d.y};
            stream_oct<OUT, USE_TAB, true>(P, w, tab, dst + PS * 8u * i, plane);
            ox += dx; r += dr;
            if (ox >= opr) { ox -= opr; ++r; }
        }
    }
}

// PLAIN / LUT octet streaming (octet geometry, band staged)
template <int OUT, bool TAB, bool LUT>
__device__ __forceinline__ void final_rows_plain_lut8(const AugParams& P, const float* s_norm, const float* ftab, const Ctx& c,
                                                      int flip, void* out_img, int oy0, int oy1) {
    if (flip) {
        if (LUT) final_rows_stream8<OUT, true, true>(P, ftab, c, out_img, oy0, oy1);
        else final_rows_stream8<OUT, TAB, true>(P, s_norm, c, out_img, oy0, oy1);
    } else {
        if (LUT) final_rows_stream8<OUT, true, false>(P, ftab, c, out_img, oy0, oy1);
        else final_rows_stream8<OUT, TAB, false>(P, s_norm, c, out_img, oy0, oy1);
    }
}

// PLAIN / LUT final pass: the streaming loop when possible, else the generic aligned loop.
// `ftab` (768 floats) is only read for LUT programs and must hold normalise(ch, lutc[ch][b]).
template <int OUT, bool TAB, bool LUT, bool OCT = false>
__device__ __forceinline__ void final_rows_plain_lut(const AugParams& P, const float* s_norm, const float* ftab, const Ctx& c,
                                                     const uint8_t* lutc, const TailInfo& t, void* out_img, int oy0, int oy1) {
    if constexpr (OUT != OUT_U8_HWC || OCT) {                       // (uint8 HWC: only the octet paths of the light kernel)
        if ((!LUT || ftab != nullptr) && band_fully_staged(c, t, oy0, oy1) && (OUT != OUT_U8_HWC || (OCT && octet_geometry(P, t)))) {
            if (OCT && octet_geometry(P, t)) {                 // (the light kernel: 8 pixels per thread and iteration)
                final_rows_plain_lut8<OUT, TAB, LUT>(P, s_norm, ftab, c, t.flip, out_img, oy0, oy1);
                return;
            }
            const float pad[3] = {normalise<TAB>(P, s_norm, 0, 0u), normalise<TAB>(P, s_norm, 1, 0u), normalise<TAB>(P, s_norm, 2, 0u)};
            if (LUT) final_rows_stream<OUT, true>(P, ftab, pad, c, t, out_img, oy0, oy1);
            else final_rows_stream<OUT, TAB>(P, s_norm, pad, c, t, out_img, oy0, oy1);
            return;
        }
    }
    final_rows<OUT, TAB, LUT ? C_LUT : C_PLAIN>(P, s_norm, c, lutc, t, out_img, oy0, oy1);
}

// ftab[ch][b] = normalise(ch, lutc[ch][b]) (all threads; ends with a barrier)
template <bool TAB>
__device__ __forceinline__ void build_ftab(const AugParams& P, const float* s_norm, const uint8_t* lutc, float* ftab) {
    for (int i = threadIdx.x; i < 768; i += blockDim.x) ftab[i] = normalise<TAB>(P, s_norm, i >> 8, (uint32_t)lutc[i]);
    __syncthreads();
}

template <int OUT, bool TAB>
__device__ __forceinline__ void final_rows_cls(int cls, const AugParams& P, const float* s_norm, const Ctx& c,
                                               const uint8_t* lutc, const TailInfo& t, void* out_img, int oy0, int oy1,
                                               const float* ftab = nullptr) {
    switch (cls) {
    case C_PLAIN: final_rows_plain_lut<OUT, TAB, false>(P, s_norm, ftab, c, lutc, t, out_img, oy0, oy1); break;
    case C_LUT:   final_rows_plain_lut<OUT, TAB, true>(P, s_norm, ftab, c, lutc, t, out_img, oy0, oy1); break;
    case C_POINT: final_rows<OUT, TAB, C_POINT>(P, s_norm, c, lutc, t, out_img, oy0, oy1); break;
    case C_SHARP: final_rows<OUT, TAB, C_SHARP>(P, s_norm, c, lutc, t, out_img, oy0, oy1); break;
    case C_GEOM:  final_rows<OUT, TAB, C_GEOM>(P, s_norm, c, lutc, t, out_img, oy0, oy1); break;
    case C_SG:    final_rows<OUT, TAB, C_SG>(P, s_norm, c, lutc, t, out_img, oy0, oy1); break;
    default:      final_rows<OUT, TAB, C_GENERIC>(P, s_norm, c, lutc, t, out_img, oy0, oy1); break;
    }
}

// (the chunk has a 16-byte guard band on both sides so that the vector paths' "is the 16-byte
//  neighbourhood resident" tests succeed for its first and last pixels; guards are never used)
constexpr uint32_t kMatGuard = 16;

// C_MAT: op0's output is materialised chunk by chunk into `mat` (uint8 HWC rows), then op1 - a
// Sharpness or a statistics op - runs on the chunk as a single-op program.  Never re-evaluates
// op0 nine times (lazy Sharpness) and keeps shared memory bounded for any image size.
// rows [r0, r1) of op0's output (op1 disabled in `c`) -> dst (+ row pitch), through the
// class-specialised single-op evaluators (cls0) when the width allows 4-pixel quads
static __device__ void fill_rows(const Ctx& c_in, int cls0, const uint8_t* lut0, uint8_t* dst, int r0, int r1) {
    // a private copy: through the reference every field read in the loop is a local-memory load (the caller's
    // stack frame), and with most of the SM's L1 carved out as shared memory those go to L2
    const Ctx c = c_in;
    const int W = c.W;
    if ((W & 3) == 0) {
        const uint32_t qpr = (uint32_t)W >> 2, nq = (uint32_t)(r1 - r0) * qpr;
        FastDiv dq; dq.init(qpr, c.rcp_wq);
        TailInfo id; id.crop_dy = id.crop_dx = id.flip = 0; id.zb0 = id.zb1 = id.zb2 = id.zb3 = 0;
        GeomOp go; int gv = 0;
        if (cls0 == C_GEOM) gv = geom_setup(c, id, c.H, W, c.H, W, go);
        for (uint32_t q = threadIdx.x; q < nq; q += blockDim.x) {
            const uint32_t r = dq.div(q);
            const int x0 = (int)(q - r * qpr) * 4, y = r0 + (int)r;
            uint32_t p[4];
            switch (cls0) {
            case C_LUT:   quad_vec<C_LUT>(c, lut0, id, W, x0, y, p); break;
            case C_POINT: quad_vec<C_POINT>(c, lut0, id, W, x0, y, p, 4 * point_kind(c.op[0].kind) + point_kind(c.op[1].kind)); break;
            case C_SHARP: quad_vec<C_SHARP>(c, lut0, id, W, x0, y, p, c.op[1].kind != K_NONE); break;
            case C_GEOM:  quad_geom_any<false, true>(gv, c, go, id, W, x0, y, p); break;
            default:
#pragma unroll
                for (int k = 0; k < 4; ++k) p[k] = Level<1>::at(c, x0 + k, y);
            }
            uint32_t* w = reinterpret_cast<uint32_t*>(dst + (r * (uint32_t)W + (uint32_t)x0) * 3u);
            w[0] = p[0] | (p[1] << 24);
            w[1] = (p[1] >> 8) | (p[2] << 16);
            w[2] = (p[2] >> 16) | (p[3] << 8);
        }
    } else {
        const uint32_t n = (uint32_t)(r1 - r0) * (uint32_t)W;
        FastDiv dw; dw.init((uint32_t)W, c.rcp_w);
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t r = dw.div(i);
            const uint32_t p = Level<1>::at(c, (int)(i - r * W), r0 + (int)r);
            uint8_t* o = dst + i * 3u;
            o[0] = (uint8_t)p; o[1] = (uint8_t)(p >> 8); o[2] = (uint8_t)(p >> 16);
        }
    }
}

__device__ __forceinline__ int single_op_class(int kind, int W) {
    if (W & 3) return C_GENERIC;
    if (kind == K_SHARPNESS) return C_SHARP;
    if (kind == K_AFFINE || kind == K_SHIFT) return C_GEOM;
    if (kind_uses_lut(kind)) return C_LUT;
    return C_POINT;
}

template <int OUT, bool TAB>
__device__ bool run_materialised(const AugParams& P, const float* s_norm, ImgState& st, const Ctx& c, uint8_t* mat,
                                 void* out_img, int band, cg::cluster_group& cluster) {
    const int H = P.H, W = P.W;
    const uint32_t pitch = (uint32_t)W * 3u;
    const int k1 = st.prog.op[1].kind;
    const bool stat1 = kind_needs_hist(k1) || kind_needs_mean(k1);
    const int halo = (k1 == K_SHARPNESS) ? 1 : 0;
    const int rows_cap = (P.mat_cap - 2 * (int)kMatGuard) / (int)pitch;      // >= 3
    const int step = rows_cap - 2 * halo;
    const int y0 = P.geo[0].y[band], y1 = P.geo[0].y[band + 1];
    bool exchanged = false;

    // op0's own LUT (and statistics over the raw band) first
    const uint32_t n_pixels = (uint32_t)H * (uint32_t)W;
    const int k0 = st.prog.op[0].kind;
    if (st.prog.stat_mask) zero_stats(st);
    if (st.prog.lut_mask & 1u) {
        uint32_t mean = 0;
        if (st.prog.stat_mask & 1u) {
            accumulate_stats<0>(c, kind_needs_hist(k0), kind_needs_mean(k0), y0, y1, st.hist[0], &st.suml[0]);
            mean = exchange_stats(P.bands, n_pixels, kind_needs_hist(k0), kind_needs_mean(k0), st, 0, cluster);
            exchanged = true;
        }
        make_lut(n_pixels, st, 0, mean);
    }
    Ctx c0 = c;                                                   // op0 alone, evaluated into the chunk
    c0.op[1].kind = K_NONE;
    const int cls0 = single_op_class(k0, W);
    // the op1-only program that runs on the materialised rows
    Ctx c2;
    c2.raw = nullptr; c2.sraw = mat; c2.H = H; c2.W = W; c2.rcp_w = c.rcp_w; c2.rcp_wq = c.rcp_wq;
    c2.op[0] = st.prog.op[1]; c2.box[0] = st.prog.box[1];
    c2.op[1].kind = K_NONE; c2.box[1] = st.prog.box[1];
    c2.lut[0] = st.lut[1]; c2.lut[1] = st.lut[1];

    const TailInfo t = make_tail(P, st.prog);
    const int oy0 = P.geo[0].oy[band], oy1 = P.geo[0].oy[band + 1];
    // resident mode: every row of op0's output this CTA needs fits the buffer -> evaluate op0 ONCE
    int ra = min(y0, oy0 + t.crop_dy - halo), rb = max(y1, oy1 + t.crop_dy + halo);
    if (ra < 0) ra = 0;
    if (rb > H) rb = H;
    const bool resident = rb - ra <= rows_cap;
    if (resident) {
        fill_rows(c0, cls0, st.lut[0], mat + kMatGuard, ra, rb);
        c2.s_lo = (uint32_t)ra * pitch - kMatGuard; c2.s_len2 = (uint32_t)(rb - ra) * pitch + 2u * kMatGuard - 2u;
        __syncthreads();
    }
    if (stat1) {                                                  // pass A: statistics of op0's output
        if (resident) {
            accumulate_stats<0>(c2, kind_needs_hist(k1), kind_needs_mean(k1), y0, y1, st.hist[1], &st.suml[1]);
        } else {
            for (int r = y0; r < y1; r += rows_cap) {
                const int re = min(r + rows_cap, y1);
                fill_rows(c0, cls0, st.lut[0], mat + kMatGuard, r, re);
                __syncthreads();
                c2.s_lo = (uint32_t)r * pitch - kMatGuard; c2.s_len2 = (uint32_t)(re - r) * pitch + 2u * kMatGuard - 2u;
                accumulate_stats<0>(c2, kind_needs_hist(k1), kind_needs_mean(k1), r, re, st.hist[1], &st.suml[1]);
                __syncthreads();
            }
        }
        exchanged = true;
        const uint32_t mean1 = exchange_stats(P.bands, n_pixels, kind_needs_hist(k1), kind_needs_mean(k1), st, 1, cluster);
        make_lut(n_pixels, st, 1, mean1);
        if (st.prog.cls2 == C_LUT) {                              // op1-only program: one LUT
            for (int i = threadIdx.x; i < 768; i += blockDim.x) st.lutc[i] = st.lut[1][i];
            __syncthreads();
        }
    }
    // pass B: output rows
    if (resident) {
        final_rows_cls<OUT, TAB>(st.prog.cls2, P, s_norm, c2, st.lutc, t, out_img, oy0, oy1);
    } else {
        for (int o = oy0; o < oy1; o += step) {                   // chunk by chunk
            const int oe = min(o + step, oy1);
            int r0 = o + t.crop_dy - halo, r1 = oe + t.crop_dy + halo;      // source rows of this chunk
            if (r0 < 0) r0 = 0;
            if (r1 > H) r1 = H;
            if (r1 > r0) {
                fill_rows(c0, cls0, st.lut[0], mat + kMatGuard, r0, r1);
                c2.s_lo = (uint32_t)r0 * pitch - kMatGuard; c2.s_len2 = (uint32_t)(r1 - r0) * pitch + 2u * kMatGuard - 2u;
            } else { c2.s_lo = 0; c2.s_len2 = 0; }
            __syncthreads();
            final_rows_cls<OUT, TAB>(st.prog.cls2, P, s_norm, c2, st.lutc, t, out_img, o, oe);
            __syncthreads();
        }
    }
    return exchanged;
}

// two sources mixed in fp32 (fused Mixup): class dispatch per quad, both contexts live
template <int OUT, bool TAB>
__device__ void final_pass_mix(const AugParams& P, const float* s_norm, const ImgState* st, const Ctx& c0,
                               const Ctx& c1, void* out_img, int band) {
    using T = typename OutElem<OUT>::T;
    const int oy0 = P.geo[0].oy[band], oy1 = P.geo[0].oy[band + 1];
    const uint32_t qpr = (uint32_t)(P.out_w + 3) >> 2;
    const uint32_t nq = (uint32_t)(oy1 - oy0) * qpr;
    FastDiv dq; dq.init(qpr, P.rcp_out_qpr);
    const bool vec = (P.out_w & 3) == 0;
    const TailInfo t0 = make_tail(P, st[0].prog), t1 = make_tail(P, st[1].prog);
    const int cls0 = st[0].prog.cls, cls1 = st[1].prog.cls;
    const uint32_t plane = (uint32_t)P.out_h * (uint32_t)P.out_w;
    for (uint32_t q = threadIdx.x; q < nq; q += blockDim.x) {
        const uint32_t r = dq.div(q);
        const int ox0 = (int)(q - r * qpr) * 4;
        const int oy = oy0 + (int)r;
        uint32_t pa[4], pb[4];
        if (cls0 == C_GENERIC || cls0 == C_GEOM || cls0 == C_SG) quad_generic(c0, t0, P.out_w, ox0, oy, pa);
        else if (cls0 == C_LUT) quad_vec<C_LUT>(c0, st[0].lutc, t0, P.out_w, ox0, oy, pa);
        else if (cls0 == C_SHARP) quad_vec<C_SHARP>(c0, st[0].lutc, t0, P.out_w, ox0, oy, pa, c0.op[1].kind != K_NONE);
        else quad_vec<C_POINT>(c0, st[0].lutc, t0, P.out_w, ox0, oy, pa, 4 * point_kind(c0.op[0].kind) + point_kind(c0.op[1].kind));
        if (cls1 == C_GENERIC || cls1 == C_GEOM || cls1 == C_SG) quad_generic(c1, t1, P.out_w, ox0, oy, pb);
        else if (cls1 == C_LUT) quad_vec<C_LUT>(c1, st[1].lutc, t1, P.out_w, ox0, oy, pb);
        else if (cls1 == C_SHARP) quad_vec<C_SHARP>(c1, st[1].lutc, t1, P.out_w, ox0, oy, pb, c1.op[1].kind != K_NONE);
        else quad_vec<C_POINT>(c1, st[1].lutc, t1, P.out_w, ox0, oy, pb, 4 * point_kind(c1.op[0].kind) + point_kind(c1.op[1].kind));
        const uint32_t za = zero_mask(t0, ox0, oy), zb = zero_mask(t1, ox0, oy);
        const int nvalid = min(4, P.out_w - ox0);
        T* o = reinterpret_cast<T*>(out_img) + (uint32_t)(oy * P.out_w + ox0);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float a = ((za >> k) & 1u) ? 0.0f : normalise<TAB>(P, s_norm, ch, (pa[k] >> (8 * ch)) & 255u);
                float b = ((zb >> k) & 1u) ? 0.0f : normalise<TAB>(P, s_norm, ch, (pb[k] >> (8 * ch)) & 255u);
                v[k] = f_add(f_mul(a, P.lam), f_mul(b, P.one_minus_lam));          // aug_mixup.py:21
            }
            store_plane4<OUT>(o + ch * plane, v, vec, nvalid);
        }
    }
}

}  // namespace faa
#include "faa_fast.cuh"
namespace faa {

// ---- scalar statistics: AutoContrast needs only per-channel min / max, Contrast only the luma sum ----------
// (PIL ImageOps.autocontrast with cutoff 0 uses the first / last non-zero histogram bin, augmentations.py:64-65;
//  ImageEnhance.Contrast the rounded mean luma, :97-99.)  For programs "statistics op [+ static per-channel LUT]"
// the band is scanned with packed 16-bit min / max (VIMNMX3.U16x2) or a luma sum - no shared-memory atomics -,
// the per-band scalars (32 bytes) are exchanged with ONE cluster barrier and every CTA builds the float table
// tab[ch][b] = normalise(lut1(lut0(b))) directly.
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

__device__ __forceinline__ bool scalar_stats_program(const Prog& g) {
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    return (g.cls == C_LUT || g.cls == C_GEOM || g.cls == C_MAT) && (k0 == K_AUTOCONTRAST || k0 == K_CONTRAST) &&
           (k1 == K_NONE || k1 == K_LUT || k1 == K_BRIGHTNESS || k1 == K_AFFINE || k1 == K_SHIFT || k1 == K_SHARPNESS);
}

// returns with ftab / st.lutc complete (barrier included); the caller must call cluster_wait() once more before
// the CTA exits when `bands > 1` (peers may still be reading this CTA's record)
template <bool TAB>
__device__ void build_scalar_stats_table(const AugParams& P, const float* s_norm, ImgState& st, const Ctx& c, int y0, int y1,
                                         cg::cluster_group& cluster, float* ftab) {
    const int k0 = st.prog.op[0].kind;
    const bool ac = k0 == K_AUTOCONTRAST;
    const uint32_t nq = (uint32_t)(y1 - y0) * (uint32_t)P.W / 4u;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(c.sraw + ((uint32_t)y0 * (uint32_t)P.W * 3u - c.s_lo));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (ac) {
        // quad = 12 bytes R G B R | G B R G | B R G B: even / odd bytes of each word as 16-bit lanes
        uint32_t mnA = 0x00FF00FFu, mnB = 0x00FF00FFu, mnC = 0x00FF00FFu, mxA = 0u, mxB = 0u, mxC = 0u;   // lanes (R,B) (G,R) (B,G)
        for (uint32_t i = threadIdx.x; i < nq; i += blockDim.x) {
            const uint32_t w0 = src[3u * i], w1 = src[3u * i + 1u], w2 = src[3u * i + 2u];
            const uint32_t e0 = __byte_perm(w0, 0u, 0x4240), o0 = __byte_perm(w0, 0u, 0x4341);
            const uint32_t e1 = __byte_perm(w1, 0u, 0x4240), o1 = __byte_perm(w1, 0u, 0x4341);
            const uint32_t e2 = __byte_perm(w2, 0u, 0x4240), o2 = __byte_perm(w2, 0u, 0x4341);
            mnA = __vimin3_u16x2(mnA, e0, o2); mxA = __vimax3_u16x2(mxA, e0, o2);
            mnB = __vimin3_u16x2(mnB, o0, e1); mxB = __vimax3_u16x2(mxB, o0, e1);
            mnC = __vimin3_u16x2(mnC, o1, e2); mxC = __vimax3_u16x2(mxC, o1, e2);
        }
        uint32_t v[6];
        v[0] = min(mnA & 0xFFFFu, mnB >> 16); v[1] = min(mnB & 0xFFFFu, mnC >> 16); v[2] = min(mnA >> 16, mnC & 0xFFFFu);
        v[3] = max(mxA & 0xFFFFu, mxB >> 16); v[4] = max(mxB & 0xFFFFu, mxC >> 16); v[5] = max(mxA >> 16, mxC & 0xFFFFu);
#pragma unroll
        for (int j = 0; j < 3; ++j) { v[j] = __reduce_min_sync(0xffffffffu, v[j]); v[3 + j] = __reduce_max_sync(0xffffffffu, v[3 + j]); }
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 6; ++j) st.wred[warp][j] = v[j];
        }
    } else {
        uint32_t local = 0;
        for (uint32_t i = threadIdx.x; i < nq; i += blockDim.x) {
            uint32_t q[4];
            unpack12(src[3u * i], src[3u * i + 1u], src[3u * i + 2u], q);
#pragma unroll
            for (int k = 0; k < 4; ++k) local += luma_of(q[k]);
        }
        local = __reduce_add_sync(0xffffffffu, local);                     // < 2^32: a warp covers < 2^24 pixels of a band
        if (lane == 0) st.wred[warp][6] = local;
    }
    __syncthreads();
    const int nwarp = (int)(blockDim.x >> 5);
    if (threadIdx.x < 8) {
        const int j = threadIdx.x;
        if (ac) {
            uint32_t r = j < 3 ? 255u : 0u;
            if (j < 6) for (int w = 0; w < nwarp; ++w) r = j < 3 ? min(r, st.wred[w][j]) : max(r, st.wred[w][j]);
            st.xpart[j] = r;
        } else if (j == 6) {
            unsigned long long t = 0;
            for (int w = 0; w < nwarp; ++w) t += st.wred[w][6];
            st.xpart[6] = (uint32_t)t; st.xpart[7] = (uint32_t)(t >> 32);
        }
    }
    const int bands = P.bands;
    if (bands > 1) { cluster_arrive(); cluster_wait(); } else __syncthreads();       // every band's record is complete
    if (threadIdx.x < 8) {
        const int j = threadIdx.x;
        uint32_t v[8];
#pragma unroll
        for (int r = 0; r < 8; ++r)                                        // remote loads in flight together
            v[r] = r < bands ? (bands > 1 ? cluster.map_shared_rank(&st.xpart[0], opaque_u32(r))[j] : st.xpart[j]) : (j < 3 ? 255u : 0u);
        uint32_t t;
        if (j < 3) t = min(min(min(v[0], v[1]), min(v[2], v[3])), min(min(v[4], v[5]), min(v[6], v[7])));
        else if (j < 6) t = max(max(max(v[0], v[1]), max(v[2], v[3])), max(max(v[4], v[5]), max(v[6], v[7])));
        else t = 0u;
        st.xtot[j] = t;
        if (j == 6) {                                                      // 64-bit luma total
            unsigned long long tot = 0;
            for (int r = 0; r < bands; ++r) {
                const uint32_t* xp = bands > 1 ? cluster.map_shared_rank(&st.xpart[0], opaque_u32(r)) : &st.xpart[0];
                tot += (unsigned long long)xp[6] | ((unsigned long long)xp[7] << 32);
            }
            st.xtot[6] = (uint32_t)tot; st.xtot[7] = (uint32_t)(tot >> 32);
        }
    }
    __syncthreads();
    if (bands > 1) cluster_arrive();                                       // this CTA is done reading its peers
    // the table: entry i of channel ch by thread i (blockDim.x == 256)
    const OpRec o0 = st.prog.op[0], o1 = st.prog.op[1];
    const uint32_t n_pixels = (uint32_t)P.H * (uint32_t)P.W;
    const uint32_t mean = ac ? 0u : contrast_mean((unsigned long long)st.xtot[6] | ((unsigned long long)st.xtot[7] << 32), n_pixels);
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
        const int ch = i >> 8, ix = i & 255;
        uint32_t v;
        if (ac) {                                                          // == hist_lut_lane(K_AUTOCONTRAST)
            const int lo = (int)st.xtot[ch], hi = (int)st.xtot[3 + ch];
            if (hi <= lo) v = (uint32_t)ix;
            else {
                const double scale = 255.0 / (double)(hi - lo);
                const double offset = d_mul(-(double)lo, scale);
                const int t = (int)d_add(d_mul((double)ix, scale), offset);
                v = (uint32_t)(t < 0 ? 0 : t > 255 ? 255 : t);
            }
        } else {
            v = lut_entry_static(o0, (uint32_t)ix, mean);
        }
        if (o1.kind != K_NONE) v = lut_entry_static(o1, v, 0u);
        st.lutc[i] = (uint8_t)v;
        ftab[i] = normalise<TAB>(P, s_norm, ch, v);
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------
// launch 2
// self-resolving launches: one image's decisions and program, by one thread (kept out of line: its registers and
// code must not weigh on the pixel paths)
static __device__ __noinline__ void self_resolve_prog(const AugParams& P, int i, Prog* dst) {
    Sample s;
    Box bx[8];
    philox_sample(P.sr_rng, P.sr_rng.first_index + (uint64_t)i, P.sr_ops, P.sr_probs, P.sr_n_sub, P.sr_n_op, P.H, P.W,
                  P.out_h, P.out_w, s, bx);
    Prog g;
    build_prog(s, bx, P.sr_ops, P.sr_n_op, P.sr_op_base, P.sr_apply_tail, P.H, P.W, P.out_w, P.sr_allow, g);
    g.bucket = 0;
    *dst = g;
}

// entry: this cluster's schedule row (blockIdx.y of a uniform launch)
template <int OUT, int NSRC, bool TAB>
static __device__ __forceinline__ void cluster_kernel_body(const AugParams& P, int entry) {
    extern __shared__ __align__(128) uint8_t s_dyn[];           // NSRC staged row bands [+ materialisation chunk]
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ ImgState st[NSRC];
    __shared__ float s_norm[TAB ? 768 : 1];
    __shared__ __align__(8) uint64_t s_bar[NSRC];

    const int band = blockIdx.x;
    const uint32_t img_bytes = (uint32_t)P.H * (uint32_t)P.W * 3u;
    const uint32_t s_lo = P.geo[0].lo[band], s_len = P.geo[0].len[band];
    if (TAB && !P.norm_stride)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + i);

    // Programmatic dependent launch: everything above overlaps the resolve kernel's tail; the
    // schedule and the programs it writes are only read after this point.
    if (P.chain == CHAIN_STREAM_ORDERED) asm volatile("griddepcontrol.wait;" ::: "memory");
    if (P.chain == CHAIN_SELF_RESOLVING) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // nothing shared between steps
    wait_ticket(P.ready, P.ticket);

    // split launches: this (cluster) kernel owns the first n_heavy entries of the schedule
    if (P.n_heavy != nullptr && entry >= ld_sched(P.n_heavy, P.chain)) return;      // cluster-uniform
    // LPT schedule entry: a uniform load per warp (no shared-memory hand-off, no barrier)
    const int img = P.order ? ld_sched(P.order + P.first + entry, P.chain) : entry;
    int src_idx[NSRC];
    src_idx[0] = P.first + img;
    if constexpr (NSRC == 2) src_idx[1] = P.partner[img];
    if (TAB && P.norm_stride)                                   // Lighting: this image's own normalisation table
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + (size_t)src_idx[0] * P.norm_stride + i);

    // 0. stage the raw row band(s): one TMA bulk copy each, in flight while the program loads
    if (threadIdx.x == 0 && s_len) {
#pragma unroll
        for (int s = 0; s < NSRC; ++s)
            tma_stage(&s_bar[s], s_dyn + (size_t)s * P.band_cap, P.in + (size_t)src_image(P, src_idx[s]) * img_bytes + s_lo, s_len);
    }
    // per-image programs -> shared memory (24 words each)
    if (P.self_resolve) {
        if (threadIdx.x == 0) {
#pragma unroll
            for (int s = 0; s < NSRC; ++s) self_resolve_prog(P, src_idx[s], &st[s].prog);
        }
    } else {
#pragma unroll
        for (int s = 0; s < NSRC; ++s)
            if (threadIdx.x < sizeof(Prog) / 4)
                reinterpret_cast<uint32_t*>(&st[s].prog)[threadIdx.x] =
                    ld_sched(reinterpret_cast<const uint32_t*>(P.progs + src_idx[s]) + threadIdx.x, P.chain);
    }
    __syncthreads();
    // chained steps: the next kernel of the stream may start once every CTA of this one has copied its program
    // (it may overwrite the OTHER program slot only); Sharpness->gather programs also own a scratch image that
    // the next step reuses, so they only release at exit.  (A chained step is tested as "neither stream-ordered nor
    // self-resolving": `== CHAIN_STEP` compiles to one instruction less, and the shifted code made the self-resolving
    // CIFAR step 0.5% slower on an H100 80GB HBM3 at 400 W.)
    if (P.chain != CHAIN_STREAM_ORDERED && P.chain != CHAIN_SELF_RESOLVING && st[0].prog.cls != C_SG) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (s_len) {
#pragma unroll
        for (int s = 0; s < NSRC; ++s) mbar_wait(&s_bar[s], 0);
    }

    const int y0 = P.geo[0].y[band], y1 = P.geo[0].y[band + 1];
    const int oy0 = P.geo[0].oy[band], oy1 = P.geo[0].oy[band + 1];
    const size_t out_elem = OUT == OUT_F32 ? 4 : (OUT == OUT_U8_HWC ? 1 : 2);
    void* out_img = reinterpret_cast<uint8_t*>(P.out) + (size_t)img * 3u * (size_t)P.out_h * (size_t)P.out_w * out_elem;
    const uint8_t* raw0 = P.in + (size_t)src_image(P, src_idx[0]) * img_bytes;
    bool any_stats = false;

    if constexpr (NSRC == 1) {
        const int cls = st[0].prog.cls;
        // C_PLAIN / C_LUT final passes only read the composed LUT; but a C_LUT program with slot-1 statistics (Contrast
        // behind a LUT op, in a launch without a materialisation chunk) takes them lazily through Level<1>, which
        // evaluates op 0 from the records
        const bool full = (cls != C_PLAIN && cls != C_LUT) || (st[0].prog.stat_mask & 2u);
        const Ctx c = make_ctx(P, raw0, s_dyn, s_lo, s_len, P.H, P.W, st[0], full);
        if (cls == C_MAT) {
            any_stats = run_materialised<OUT, TAB>(P, s_norm, st[0], c, s_dyn + P.band_cap, out_img, band, cluster);
        } else if (cls == C_SG) {
            // Sharpness then a gather: the band of the sharpened image goes to the global scratch
            // image, the whole cluster synchronises, then the gather reads scratch (coherent loads)
            uint8_t* scr = P.scratch + (size_t)src_idx[0] * img_bytes;
            Ctx cs = c; cs.op[1].kind = K_NONE;
            fill_rows(cs, C_SHARP, st[0].lut[0], scr + (uint32_t)y0 * (uint32_t)P.W * 3u, y0, y1);
            __threadfence();
            cluster.sync();                                      // also for one band: orders the scratch stores
            Ctx cg2 = c;
            cg2.raw = scr; cg2.s_len2 = 0;
            cg2.op[0] = c.op[1]; cg2.box[0] = c.box[1]; cg2.op[1].kind = K_NONE;
            final_rows_cls<OUT, TAB>(C_SG, P, s_norm, cg2, st[0].lutc, make_tail(P, st[0].prog), out_img, oy0, oy1);
        } else {
            any_stats = prepare_image(P, c, y0, y1, st[0], cluster);
            // LUT programs: composed LUT o normalisation table in the (now idle) slot-0 histogram
            float* ftab = nullptr;
            if (OUT != OUT_U8_HWC && cls == C_LUT) {
                ftab = reinterpret_cast<float*>(&st[0].hist[0][0]);
                build_ftab<TAB>(P, s_norm, st[0].lutc, ftab);
            }
            final_rows_cls<OUT, TAB>(cls, P, s_norm, c, st[0].lutc, make_tail(P, st[0].prog), out_img, oy0, oy1, ftab);
        }
        zero_box_rows<OUT>(P, st[0].prog, out_img, oy0, oy1);
    } else {
        const uint8_t* raw1 = P.in + (size_t)src_image(P, src_idx[1]) * img_bytes;
        const Ctx c0 = make_ctx(P, raw0, s_dyn, s_lo, s_len, P.H, P.W, st[0], true);
        const Ctx c1 = make_ctx(P, raw1, s_dyn + P.band_cap, s_lo, s_len, P.H, P.W, st[1], true);
        any_stats = prepare_image(P, c0, y0, y1, st[0], cluster);
        any_stats |= prepare_image(P, c1, y0, y1, st[1], cluster);
        final_pass_mix<OUT, TAB>(P, s_norm, st, c0, c1, out_img, band);
    }

    (void)any_stats;   // statistics exchanges end with their own cluster barrier (build_slot_lut)
}

// a pointwise op applied in place to rows [r0, r1) of a uint8 HWC band whose byte 0 is pixel (0, ra): per-channel LUT
// (`lut`), Color (augmentations.py:102-104) or the Cutout box (augmentations.py:142-143).  No barrier inside.
__device__ __forceinline__ void inplace_pointwise(const AugParams& P, uint8_t* band, int ra, int r0, int r1, int kind, const OpRec& op,
                                                  const Box bx, const uint8_t* lut) {
    const uint32_t qpr = (uint32_t)P.W >> 2, nq = (uint32_t)(r1 - r0) * qpr;
    uint32_t* rows = reinterpret_cast<uint32_t*>(band + (uint32_t)(r0 - ra) * (uint32_t)P.W * 3u);
    const float alpha = bits_to_float(op.a[0]);
    const bool clip = op.a[1] != 0;
    FastDiv dq; dq.init(qpr, P.rcp_wq);
    for (uint32_t i = threadIdx.x; i < nq; i += blockDim.x) {
        uint32_t q[4];
        unpack12(rows[3u * i], rows[3u * i + 1u], rows[3u * i + 2u], q);
        if (kind == K_CUTOUT) {
            const uint32_t r = dq.div(i);
            const int y = r0 + (int)r, x0 = (int)(i - r * qpr) * 4;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (y >= bx.y0 && y <= bx.y1 && x0 + k >= bx.x0 && x0 + k <= bx.x1) q[k] = kCutoutRGB;
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) q[k] = kind == K_COLOR ? color_px(q[k], alpha, clip) : apply_lut(lut, q[k]);
        }
        rows[3u * i] = q[0] | (q[1] << 24);
        rows[3u * i + 1u] = (q[1] >> 8) | (q[2] << 16);
        rows[3u * i + 2u] = (q[2] >> 16) | (q[3] << 8);
    }
}

template <int OUT, int NSRC, bool TAB>
__global__ void __launch_bounds__(kThreads, (NSRC == 1 ? FAA_MIN_CTAS : 2)) faa_augment_kernel(const __grid_constant__ AugParams P) {
    cluster_kernel_body<OUT, NSRC, TAB>(P, (int)blockIdx.y);
    count_done(P.done);                                          // (CTAs without an entry included)
}

#if defined(FAA_TU_OUT) && FAA_TU_OUT == 3   // OUT_U8_HWC
// Ragged policy launch (faa_augment_ragged): cluster blockIdx.y runs image list[blockIdx.y] at its own size.  The
// image's per-size launch parameters are copied into shared memory once per CTA and its pointers patched in; the body
// is the uniform cluster kernel's, reading them from there (no order, no split, no chaining, uint8 HWC, one source).
__global__ void __launch_bounds__(kThreads, FAA_MIN_CTAS) faa_augment_ragged_kernel(const __grid_constant__ RaggedParams R) {
    __shared__ AugParams sP;
    const int i = __ldg(R.list + blockIdx.y);
    const RaggedImg& m = R.imgs[i];
    const uint32_t* src = reinterpret_cast<const uint32_t*>(R.geoms + m.geom);
    for (int k = threadIdx.x; k < (int)(sizeof(AugParams) / 4); k += blockDim.x) reinterpret_cast<uint32_t*>(&sP)[k] = __ldg(src + k);
    __syncthreads();
    if (threadIdx.x == 0) {
        sP.in = m.realigned ? m.realigned : R.in[i].data;
        sP.out = const_cast<uint8_t*>(R.out[i].data);
        sP.scratch = m.scratch;
        sP.progs = R.progs + i;
    }
    __syncthreads();
    cluster_kernel_body<OUT_U8_HWC, 1, false>(sP, 0);
}
#endif

// ---------------------------------------------------------------------------------------
// launch 2b: the "mid" kernel of a three-way split: statistics -> per-channel LUT programs (AutoContrast, Equalize,
// Contrast, with static LUT partners) and Sharpness (+ static LUT).  One cluster per image like the cluster kernel
// (P.bands / P.geo[0] of THIS launch: fewer, taller bands - the per-CTA overhead of a statistics program is
// amortised over more pixels), but only the lean paths: scalar statistics with one cluster barrier, the shared
// histogram path for Equalize and pushed-forward histograms, the byte-stream Sharpness, the streaming final pass.
// Preconditions (host, three-way split only): float output of the image's own size, no crop, W % 4 == 0, staged bands.
// It owns schedule entries [n_heavy[0], n_heavy[1]).
constexpr int kMidThreadsMax = 512;     // two tall bands per image, 512 threads each: 2 CTAs / SM at 224x224
template <int OUT, bool TAB>
__global__ void __launch_bounds__(kMidThreadsMax, 2) faa_augment_mid_kernel(const __grid_constant__ AugParams P) {
    extern __shared__ __align__(128) uint8_t s_dyn[];           // staged row band (+ halo rows)
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ ImgState st;
    __shared__ float s_norm[TAB ? 768 : 1];
    __shared__ __align__(16) uint32_t s_tile[(kMidThreadsMax / 32) * 128];      // gather tiles (128 px per warp)
    __shared__ __align__(8) uint64_t s_bar;

    if (TAB && !P.norm_stride)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + i);
    wait_ticket(P.ready, P.ticket);
    if (P.chain == CHAIN_STEP) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // persistent: see count_done
    const int e0 = ld_sched(P.n_heavy, P.chain), n_ent = ld_sched(P.n_heavy + 1, P.chain) - e0;
    // One entry per row, or a persistent row's entries.  The body is written for ONE entry; so that the compiler does not
    // hoist its loop-invariant parts (thread-index arithmetic, peer addresses) in front of the loop, where they would live
    // across the whole body and spill, thread and band indices are re-read opaquely per use (threadIdx macro above).
    for (int round = 0;; ++round) {
    const int ent = sched_entry(round, (int)blockIdx.y, (int)gridDim.y);
    if (ent >= n_ent) break;                                     // cluster-uniform
    if (round) {                                                 // shared memory (and the staging buffer, for the TMA) is free again
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
    }
    const int band = (int)opaque_u32(blockIdx.x);
    const uint32_t img_bytes = (uint32_t)P.H * (uint32_t)P.W * 3u;
    const uint32_t s_lo = P.geo[0].lo[band], s_len = P.geo[0].len[band];
    const int img = ld_sched(P.order + P.first + e0 + ent, P.chain);
    const int idx = P.first + img;
    if (TAB && P.norm_stride)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + (size_t)idx * P.norm_stride + i);
    if (threadIdx.x == 0 && s_len) tma_stage(&s_bar, s_dyn, P.in + (size_t)src_image(P, idx) * img_bytes + s_lo, s_len);
    if (threadIdx.x < sizeof(Prog) / 4)
        reinterpret_cast<uint32_t*>(&st.prog)[threadIdx.x] = ld_sched(reinterpret_cast<const uint32_t*>(P.progs + idx) + threadIdx.x, P.chain);
    __syncthreads();
    if (s_len) mbar_wait(&s_bar, 0);

    const int y0 = P.geo[0].y[band], y1 = P.geo[0].y[band + 1];
    const int oy0 = P.geo[0].oy[band], oy1 = P.geo[0].oy[band + 1];
    const size_t out_elem = OUT == OUT_F32 ? 4 : (OUT == OUT_U8_HWC ? 1 : 2);
    void* out_img = reinterpret_cast<uint8_t*>(P.out) + (size_t)img * 3u * (size_t)P.out_h * (size_t)P.out_w * out_elem;
    const int cls = st.prog.cls;
    const Ctx c = make_ctx(P, P.in + (size_t)src_image(P, idx) * img_bytes, s_dyn, s_lo, s_len, P.H, P.W, st, true);
    const TailInfo t = make_tail(P, st.prog);
    float* ftab = reinterpret_cast<float*>(&st.hist[0][0]);      // 768 floats; the slot-0 histogram is idle by then
    if (prog_two_stage(st.prog, P.allow)) {
        // Stage A materialises op0 in the band buffer: a per-channel LUT (static or from statistics), Color or Cutout in
        // place (the raw bytes are not needed again; halo rows included); a gather straight from global memory; Sharpness
        // through the global scratch image (its neighbours' rows come back from there).  Stage B runs op1 on the band as a
        // single-op program: Sharpness, a statistics LUT, Color / Cutout - or, for Sharpness -> gather, reads the scratch.
        bool peers_pending = false;
        const int k0 = st.prog.op[0].kind, k1 = st.prog.op[1].kind;
        const int ra = max(oy0 - 1, 0), rb = min(oy1 + 1, P.H);
        const uint32_t pitch = (uint32_t)P.W * 3u;
        uint8_t* rows_b = s_dyn + ((uint32_t)ra * pitch - s_lo);
        bool done = false;
        if (k0 == K_AFFINE || k0 == K_SHIFT) {
            gather_rows_to_band(P, c.raw, &st.prog.op[0], rows_b, ra, rb, s_tile);
        } else if (k0 == K_SHARPNESS) {
            uint8_t* scr = P.scratch + (size_t)idx * img_bytes;
            const float alpha0 = bits_to_float(st.prog.op[0].a[0]);
            if (st.prog.op[0].a[1]) final_rows_sharp4<OUT, false, true>(P, nullptr, c, alpha0, 0, nullptr, y0, y1, scr);
            else final_rows_sharp4<OUT, false, false>(P, nullptr, c, alpha0, 0, nullptr, y0, y1, scr);
            __threadfence();
            if (P.bands > 1) cluster.sync(); else __syncthreads();        // every band of the sharpened image is in the scratch
            if (k1 == K_AFFINE || k1 == K_SHIFT) {                        // Sharpness -> gather: straight from the scratch image
                Ctx cs = c; cs.raw = scr;
                const float pad[3] = {normalise<TAB>(P, s_norm, 0, 0u), normalise<TAB>(P, s_norm, 1, 0u), normalise<TAB>(P, s_norm, 2, 0u)};
                final_rows_gather_coh<OUT, TAB>(P, s_norm, pad, cs, &st.prog.op[1], t.flip, out_img, oy0, oy1, s_tile);
                done = true;
            } else {                                                      // back into the band buffer, halo rows from the peers' bands
                const uint32_t n16 = ((uint32_t)(rb - ra) * pitch) >> 4;  // rows are multiples of 8 bytes; the pair of rows is 16
                const uint4* g = reinterpret_cast<const uint4*>(scr + (uint32_t)ra * pitch);
                uint4* d = reinterpret_cast<uint4*>(rows_b);
                if ((((uint32_t)ra * pitch) & 15u) == 0u && (((uint32_t)(rb - ra) * pitch) & 15u) == 0u && ((reinterpret_cast<uintptr_t>(rows_b)) & 15u) == 0u) {
                    for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) d[i] = __ldcg(g + i);
                } else {
                    const uint32_t n4 = ((uint32_t)(rb - ra) * pitch) >> 2;
                    const uint32_t* g4 = reinterpret_cast<const uint32_t*>(scr + (uint32_t)ra * pitch);
                    uint32_t* d4 = reinterpret_cast<uint32_t*>(rows_b);
                    for (uint32_t i = threadIdx.x; i < n4; i += blockDim.x) d4[i] = __ldcg(g4 + i);
                }
            }
        } else {
            const uint8_t* lut0 = st.lut[0];
            if (kind_uses_lut(k0)) {
                if (scalar_stats_program(st.prog)) {
                    build_scalar_stats_table<TAB>(P, s_norm, st, c, y0, y1, cluster, ftab);     // (the float table is not used here)
                    peers_pending = P.bands > 1;
                    lut0 = st.lutc;
                } else if (st.prog.stat_mask & 1u) {
                    // histogram path of slot 0 only (prepare_image would also try slot 1)
                    const uint32_t n_pixels = (uint32_t)P.H * (uint32_t)P.W;
                    zero_stats(st);
                    accumulate_stats<0>(c, kind_needs_hist(k0), kind_needs_mean(k0), y0, y1, st.hist[0], &st.suml[0]);
                    const uint32_t mean = exchange_stats(P.bands, n_pixels, kind_needs_hist(k0), kind_needs_mean(k0), st, 0, cluster);
                    make_lut(n_pixels, st, 0, mean);
                } else {
                    make_lut((uint32_t)P.H * (uint32_t)P.W, st, 0, 0u);                          // static LUT
                }
            }
            inplace_pointwise(P, rows_b, ra, ra, rb, k0, st.prog.op[0], st.prog.box[0], lut0);
        }
        __syncthreads();
        if (done) {
        } else if (k1 == K_SHARPNESS) {
            const float alpha = bits_to_float(st.prog.op[1].a[0]);
            if (st.prog.op[1].a[1]) final_rows_sharp4<OUT, TAB, true>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
            else final_rows_sharp4<OUT, TAB, false>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
        } else if (k1 == K_COLOR || k1 == K_CUTOUT) {
            inplace_pointwise(P, rows_b, ra, oy0, oy1, k1, st.prog.op[1], st.prog.box[1], nullptr);
            __syncthreads();
            const float pad[3] = {0.0f, 0.0f, 0.0f};
            final_rows_stream<OUT, TAB>(P, s_norm, pad, c, t, out_img, oy0, oy1);
        } else {
            // a statistics LUT on the materialised band: the program continues as the single-op program of slot 1
            if (peers_pending) { cluster_wait(); peers_pending = false; }      // the record of slot 0's exchange is free again
            if (threadIdx.x == 0) {
                st.prog.op[0] = st.prog.op[1]; st.prog.op[1].kind = K_NONE;
                st.prog.stat_mask = 1; st.prog.lut_mask = 1; st.prog.cls = C_LUT;
            }
            __syncthreads();
            if (scalar_stats_program(st.prog)) {
                build_scalar_stats_table<TAB>(P, s_norm, st, c, y0, y1, cluster, ftab);
                peers_pending = P.bands > 1;
            } else {
                prepare_image(P, c, y0, y1, st, cluster);
                build_ftab<TAB>(P, s_norm, st.lutc, ftab);
            }
            const float pad[3] = {0.0f, 0.0f, 0.0f};
            final_rows_stream<OUT, true>(P, ftab, pad, c, t, out_img, oy0, oy1);
        }
        if (peers_pending) cluster_wait();
    } else if (cls == C_SHARP) {
        const float alpha = bits_to_float(st.prog.op[0].a[0]);
        const bool clip = st.prog.op[0].a[1] != 0;
        if (st.prog.op[1].kind != K_NONE) {                      // static LUT partner: rides in the float table
            make_lut((uint32_t)P.H * (uint32_t)P.W, st, 1, 0u);
            build_ftab<TAB>(P, s_norm, st.lut[1], ftab);
            if (clip) final_rows_sharp4<OUT, true, true>(P, ftab, c, alpha, t.flip, out_img, oy0, oy1);
            else final_rows_sharp4<OUT, true, false>(P, ftab, c, alpha, t.flip, out_img, oy0, oy1);
        } else {
            if (clip) final_rows_sharp4<OUT, TAB, true>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
            else final_rows_sharp4<OUT, TAB, false>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
        }
    } else {                                                     // C_LUT with statistics
        bool peers_pending = false;
        if (scalar_stats_program(st.prog)) {
            build_scalar_stats_table<TAB>(P, s_norm, st, c, y0, y1, cluster, ftab);
            peers_pending = P.bands > 1;
        } else {
            prepare_image(P, c, y0, y1, st, cluster);
            if (cls == C_LUT) build_ftab<TAB>(P, s_norm, st.lutc, ftab);
        }
        if (cls == C_GEOM) {
            // statistics LUT then a gather: the LUT ran BEFORE the gather, so pixels without a source are plain zero
            if (!scalar_stats_program(st.prog)) build_ftab<TAB>(P, s_norm, st.lut[0], ftab);      // (not a C_LUT program: no composed lutc)
            const float pad[3] = {normalise<TAB>(P, s_norm, 0, 0u), normalise<TAB>(P, s_norm, 1, 0u), normalise<TAB>(P, s_norm, 2, 0u)};
            RowShift rs;
            if (rowshift_of(st.prog.op[1], rs)) {
                if (t.flip) final_rows_rowshift<OUT, true, true>(P, ftab, pad, c, rs, out_img, oy0, oy1);
                else final_rows_rowshift<OUT, true, false>(P, ftab, pad, c, rs, out_img, oy0, oy1);
            } else {
                final_rows_gather<OUT, true>(P, ftab, pad, c, &st.prog.op[1], nullptr, t.flip, out_img, oy0, oy1, s_tile);
            }
        } else {
            const float pad[3] = {0.0f, 0.0f, 0.0f};             // never used: there is no crop padding in this kernel
            final_rows_stream<OUT, true>(P, ftab, pad, c, t, out_img, oy0, oy1);
        }
        if (peers_pending) cluster_wait();                       // peers have read this CTA's statistics record
    }
    zero_box_rows<OUT>(P, st.prog, out_img, oy0, oy1);
    }   // rounds
    count_done(P.done);
}

// ---------------------------------------------------------------------------------------
// launch 3: the streaming kernel for "light" images (no statistics, no neighbourhood ops):
// PLAIN / LUT / POINT / GEOM classes only - no cluster, 3 KB of static shared memory, a fraction of
// the cluster kernel's registers and code.  It owns schedule entries [n_heavy, B).
// LEAN: the variant for launches whose every light entry takes an octet path (LaunchPlan::lean_light, allow bit 3 of
// prog_is_light).  Without the generic evaluators it fits 64 registers: four CTAs per SM, and two beside a mid CTA.
#ifndef FAA_LIGHT_CTAS
#define FAA_LIGHT_CTAS 3                  // (see FAA_MIN_CTAS)
#endif
constexpr int kLeanLightCtas = 4;
template <int OUT, bool TAB, bool LEAN>
__global__ void __launch_bounds__(kThreads, LEAN ? kLeanLightCtas : FAA_LIGHT_CTAS) faa_augment_light_kernel(const __grid_constant__ AugParams P) {
    extern __shared__ __align__(128) uint8_t s_dyn[];           // staged row band
    __shared__ Prog s_prog;
    __shared__ __align__(16) uint8_t s_lut[2][768];
    __shared__ __align__(16) uint8_t s_lutc[768];
    __shared__ float s_ftab[768];                                // LUT programs: normalise(ch, lutc[ch][b])
    __shared__ __align__(16) uint32_t s_tile[(kThreads / 32) * 128];   // affine gather tiles (128 px per warp)
    __shared__ float s_norm[TAB ? 768 : 1];
    __shared__ __align__(8) uint64_t s_bar;

    if (TAB && !P.norm_stride)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + i);
    wait_ticket(P.ready, P.ticket);
    if (P.chain == CHAIN_STEP) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // persistent: see count_done
    const int n_heavy = ld_sched(P.n_heavy + 1, P.chain);       // entries in front of the light segment (heavy + mid)
    for (int round = 0;; ++round) {                              // one entry per row, or a persistent row's entries (see the mid kernel)
    const int ent = sched_entry(round, (int)blockIdx.y, (int)gridDim.y);
    if (ent >= P.B - n_heavy) break;
    if (round) {                                                 // shared memory (and the staging buffer, for the TMA) is free again
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
    }
    const int band = (int)opaque_u32(blockIdx.x);
    const uint32_t img_bytes = (uint32_t)P.H * (uint32_t)P.W * 3u;
    const uint32_t s_lo = P.geo[1].lo[band], s_len = P.geo[1].len[band];
    const int img = ld_sched(P.order + P.first + n_heavy + ent, P.chain);     // uniform load per warp
    const int idx = P.first + img;
    if (TAB && P.norm_stride)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) s_norm[i] = __ldg(P.norm_tab + (size_t)idx * P.norm_stride + i);
    if (threadIdx.x == 0 && s_len) tma_stage(&s_bar, s_dyn, P.in + (size_t)src_image(P, idx) * img_bytes + s_lo, s_len);
    if (threadIdx.x < sizeof(Prog) / 4)
        reinterpret_cast<uint32_t*>(&s_prog)[threadIdx.x] = ld_sched(reinterpret_cast<const uint32_t*>(P.progs + idx) + threadIdx.x, P.chain);
    __syncthreads();
    const uint32_t lut_mask = s_prog.lut_mask;
    if (lut_mask) {                                   // static LUTs only (no statistics in light programs)
#pragma unroll
        for (int j = 0; j < 2; ++j)
            if ((lut_mask >> j) & 1u)
                for (int i = threadIdx.x; i < 768; i += blockDim.x)
                    s_lut[j][i] = (uint8_t)lut_entry_static(s_prog.op[j], (uint32_t)(i & 255), 0u);
        __syncthreads();
        // (GEOM: the one LUT slot rides in the float table; lean POINT: the static LUT behind Color / Cutout)
        if (s_prog.cls == C_LUT || s_prog.cls == C_GEOM || (LEAN && s_prog.cls == C_POINT)) {
            for (int i = threadIdx.x; i < 768; i += blockDim.x) {
                uint32_t v = (uint32_t)(i & 255), base = (uint32_t)(i & ~255);
                if (lut_mask & 1u) v = s_lut[0][base + v];
                if (lut_mask & 2u) v = s_lut[1][base + v];
                s_lutc[i] = (uint8_t)v;
                s_ftab[i] = normalise<TAB>(P, s_norm, i >> 8, v);      // (uint8 HWC output: scale 1, bias 0 - the byte as a float)
            }
            __syncthreads();
        }
    }
    if (s_len) mbar_wait(&s_bar, 0);

    const int cls = s_prog.cls;
    Ctx c;
    c.raw = P.in + (size_t)src_image(P, idx) * img_bytes; c.sraw = s_dyn; c.s_lo = s_lo; c.s_len2 = s_len > 2u ? s_len - 2u : 0u;
    c.H = P.H; c.W = P.W; c.rcp_w = P.rcp_w; c.rcp_wq = P.rcp_wq;
    if (cls == C_POINT || cls == C_GEOM || cls == C_GEOM2) {
        c.op[0] = s_prog.op[0]; c.op[1] = s_prog.op[1]; c.box[0] = s_prog.box[0]; c.box[1] = s_prog.box[1];
    }
    c.lut[0] = s_lut[0]; c.lut[1] = s_lut[1];
    const TailInfo t = make_tail(P, s_prog);
    const int oy0 = P.geo[1].oy[band], oy1 = P.geo[1].oy[band + 1];
    const size_t out_elem = OUT == OUT_F32 ? 4 : (OUT == OUT_U8_HWC ? 1 : 2);
    void* out_img = reinterpret_cast<uint8_t*>(P.out) + (size_t)img * 3u * (size_t)P.out_h * (size_t)P.out_w * out_elem;
    bool done = false;
    {
        // lean octet paths (faa_fast.cuh) for the common geometry; everything else takes the generic evaluators
        // (C_GEOM2 only exists in launches whose geometry the lean gather handles: build_prog, allow bit 2)
        if (cls == C_GEOM2 || ((cls == C_GEOM || cls == C_POINT) && (LEAN || (octet_geometry(P, t) && band_fully_staged(c, t, oy0, oy1))))) {
            const int k0 = s_prog.op[0].kind, k1 = s_prog.op[1].kind;
            if (cls == C_GEOM2) {
                // two gathers: out(x) = raw(map0(map1(x))), zero wherever either map leaves the image
                const float pad[3] = {normalise<TAB>(P, s_norm, 0, 0u), normalise<TAB>(P, s_norm, 1, 0u), normalise<TAB>(P, s_norm, 2, 0u)};
                final_rows_gather<OUT, TAB>(P, s_norm, pad, c, &s_prog.op[1], &s_prog.op[0], t.flip, out_img, oy0, oy1, s_tile);
                done = true;
            } else if (cls == C_GEOM) {
                const bool g0 = k0 == K_AFFINE || k0 == K_SHIFT;          // geometric op first, partner after it
                const int pk = g0 ? k1 : k0;
                if (pk == K_NONE || kind_uses_lut(pk)) {
                    const bool has_lut = pk != K_NONE;
                    const OpRec gop = g0 ? s_prog.op[0] : s_prog.op[1];
                    float pad[3];
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch)                           // fill colour: lut(0) if the LUT runs after the gather
                        pad[ch] = (has_lut && g0) ? s_ftab[ch * 256] : normalise<TAB>(P, s_norm, ch, 0u);
                    RowShift rs;
                    if (rowshift_of(gop, rs)) {
                        if (has_lut) {
                            if (t.flip) final_rows_rowshift<OUT, true, true>(P, s_ftab, pad, c, rs, out_img, oy0, oy1);
                            else final_rows_rowshift<OUT, true, false>(P, s_ftab, pad, c, rs, out_img, oy0, oy1);
                        } else {
                            if (t.flip) final_rows_rowshift<OUT, TAB, true>(P, s_norm, pad, c, rs, out_img, oy0, oy1);
                            else final_rows_rowshift<OUT, TAB, false>(P, s_norm, pad, c, rs, out_img, oy0, oy1);
                        }
                    } else {
                        const OpRec* gp = g0 ? &s_prog.op[0] : &s_prog.op[1];
                        if (has_lut) final_rows_gather<OUT, true>(P, s_ftab, pad, c, gp, nullptr, t.flip, out_img, oy0, oy1, s_tile);
                        else final_rows_gather<OUT, TAB>(P, s_norm, pad, c, gp, nullptr, t.flip, out_img, oy0, oy1, s_tile);
                    }
                    done = true;
                } else if (LEAN) {                                       // Cutout, then the gather (prog_is_light)
                    const float pad[3] = {normalise<TAB>(P, s_norm, 0, 0u), normalise<TAB>(P, s_norm, 1, 0u), normalise<TAB>(P, s_norm, 2, 0u)};
                    final_rows_gather<OUT, TAB>(P, s_norm, pad, c, &s_prog.op[1], nullptr, t.flip, out_img, oy0, oy1, s_tile, &s_prog.box[0]);
                    done = true;
                }
            } else if (LEAN && k1 != K_NONE) {                           // Color / Cutout, then a static LUT: the float table
                if (k0 == K_COLOR) {
                    const float alpha = bits_to_float(s_prog.op[0].a[0]);
                    if (s_prog.op[0].a[1]) final_rows_color<OUT, true, true>(P, s_ftab, c, alpha, t.flip, out_img, oy0, oy1);
                    else final_rows_color<OUT, true, false>(P, s_ftab, c, alpha, t.flip, out_img, oy0, oy1);
                } else {
                    final_rows_cutout<OUT, true>(P, s_ftab, c, s_prog.box[0], t.flip, out_img, oy0, oy1);
                }
                done = true;
            } else if (k1 == K_NONE && k0 == K_COLOR) {
                const float alpha = bits_to_float(s_prog.op[0].a[0]);
                if (s_prog.op[0].a[1]) final_rows_color<OUT, TAB, true>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
                else final_rows_color<OUT, TAB, false>(P, s_norm, c, alpha, t.flip, out_img, oy0, oy1);
                done = true;
            } else if (k1 == K_NONE && k0 == K_CUTOUT) {
                final_rows_cutout<OUT, TAB>(P, s_norm, c, s_prog.box[0], t.flip, out_img, oy0, oy1);
                done = true;
            }
        }
    }
    if (LEAN && !done) {                                         // C_PLAIN / C_LUT
        if (cls == C_LUT) final_rows_plain_lut8<OUT, TAB, true>(P, s_norm, s_ftab, c, t.flip, out_img, oy0, oy1);
        else final_rows_plain_lut8<OUT, TAB, false>(P, s_norm, s_ftab, c, t.flip, out_img, oy0, oy1);
    } else if (!done) {
        switch (cls) {
        case C_PLAIN: final_rows_plain_lut<OUT, TAB, false, true>(P, s_norm, s_ftab, c, s_lutc, t, out_img, oy0, oy1); break;
        case C_LUT:   final_rows_plain_lut<OUT, TAB, true, true>(P, s_norm, s_ftab, c, s_lutc, t, out_img, oy0, oy1); break;
        case C_POINT: final_rows<OUT, TAB, C_POINT>(P, s_norm, c, s_lutc, t, out_img, oy0, oy1); break;
        default:      final_rows<OUT, TAB, C_GEOM, false>(P, s_norm, c, s_lutc, t, out_img, oy0, oy1); break;
        }
    }
    zero_box_rows<OUT>(P, s_prog, out_img, oy0, oy1);
    }   // rounds
    count_done(P.done);
}

#ifndef FAA_TU_OUT
// out[i] = data[i]*lam + data[perm[i]]*(1-lam), fp32 math (aug_mixup.py:13-23)
template <typename T>
__global__ void faa_mixup_kernel(const T* __restrict__ data, T* __restrict__ out, const int64_t* __restrict__ perm,
                                 int64_t n_per, float lam, float oml) {
    const int b = blockIdx.y;
    const T* a = data + (size_t)b * n_per;
    const T* p = data + (size_t)perm[b] * n_per;
    T* o = out + (size_t)b * n_per;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per; i += (int64_t)gridDim.x * blockDim.x) {
        float x = (float)a[i], y = (float)p[i];
        o[i] = (T)f_add(f_mul(x, lam), f_mul(y, oml));
    }
}

// 16-byte vectorised variant (n_per % VEC == 0, 16-byte aligned rows): the op is pure HBM streaming,
// 2 reads + 1 write per element
template <typename T, int VEC>
__global__ void __launch_bounds__(256) faa_mixup_kernel_v(const T* __restrict__ data, T* __restrict__ out,
                                                          const int64_t* __restrict__ perm, int64_t n_vec, int64_t n_per,
                                                          float lam, float oml) {
    const int b = blockIdx.y;
    const uint4* a = reinterpret_cast<const uint4*>(data + (size_t)b * n_per);
    const uint4* p = reinterpret_cast<const uint4*>(data + (size_t)perm[b] * n_per);
    uint4* o = reinterpret_cast<uint4*>(out + (size_t)b * n_per);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (int64_t)gridDim.x * blockDim.x) {
        const uint4 xa = __ldg(a + i), xp = __ldg(p + i);
        uint4 r;
        const uint32_t* ua = &xa.x; const uint32_t* up = &xp.x; uint32_t* ur = &r.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if constexpr (VEC == 4) {
                ur[k] = __float_as_uint(f_add(f_mul(__uint_as_float(ua[k]), lam), f_mul(__uint_as_float(up[k]), oml)));
            } else if constexpr (sizeof(T) == 2 && VEC == 8) {
                float x0, x1, y0, y1;
                if constexpr (std::is_same<T, __half>::value) {
                    const float2 fx = __half22float2(*reinterpret_cast<const __half2*>(&ua[k]));
                    const float2 fy = __half22float2(*reinterpret_cast<const __half2*>(&up[k]));
                    x0 = fx.x; x1 = fx.y; y0 = fy.x; y1 = fy.y;
                    const __half2 h = __floats2half2_rn(f_add(f_mul(x0, lam), f_mul(y0, oml)), f_add(f_mul(x1, lam), f_mul(y1, oml)));
                    ur[k] = *reinterpret_cast<const uint32_t*>(&h);
                } else {
                    const float2 fx = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ua[k]));
                    const float2 fy = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&up[k]));
                    x0 = fx.x; x1 = fx.y; y0 = fy.x; y1 = fy.y;
                    const __nv_bfloat162 h = __floats2bfloat162_rn(f_add(f_mul(x0, lam), f_mul(y0, oml)), f_add(f_mul(x1, lam), f_mul(y1, oml)));
                    ur[k] = *reinterpret_cast<const uint32_t*>(&h);
                }
            }
        }
        o[i] = r;
    }
}

// ---------------------------------------------------------------------------------------
// torchvision ColorJitter(brightness, contrast, saturation) of the ImageNet train chain (data.py:65-69) on uint8 HWC
// images: per image a random order of up to three ImageEnhance blends with per-image factors - Brightness (with
// black), Contrast (with the rounded mean luma of the CURRENT image), Color (with the pixel's luma) - i.e. the
// arithmetic of the policy ops K_BRIGHTNESS / K_CONTRAST / K_COLOR (faa_core.cuh) with magnitudes that are not
// policy constants.  One CTA per image; every op is one pass over the image in place (Contrast: a reduction first).
struct JitterRec { float alpha[3]; uint8_t order[4]; };     // == faa_jitter_t; order[]: torch.randperm(4), id 3 = hue (absent)

__global__ void __launch_bounds__(1024) faa_color_jitter_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                                                                const JitterRec* __restrict__ recs, int H, int W) {
    __shared__ uint8_t s_lut[256];
    __shared__ unsigned long long s_sum;
    const int img = blockIdx.x;
    const uint32_t npx = (uint32_t)H * (uint32_t)W;
    const uint8_t* src = in + (size_t)img * npx * 3u;
    uint8_t* dst = out + (size_t)img * npx * 3u;
    const JitterRec r = recs[img];
    bool first = true;
    for (int step = 0; step < 4; ++step) {
        const int id = r.order[step];
        if (id > 2) continue;
        const float alpha = r.alpha[id];
        const bool clip = !(alpha >= 0.0f && alpha <= 1.0f);
        const uint8_t* cur = first ? src : dst;
        if (id == 2) {                                       // saturation: ImageEnhance.Color
            for (uint32_t i = threadIdx.x; i < npx; i += blockDim.x) {
                const uint32_t p = (uint32_t)cur[3u * i] | ((uint32_t)cur[3u * i + 1u] << 8) | ((uint32_t)cur[3u * i + 2u] << 16);
                const uint32_t q = color_px(p, alpha, clip);
                dst[3u * i] = (uint8_t)q; dst[3u * i + 1u] = (uint8_t)(q >> 8); dst[3u * i + 2u] = (uint8_t)(q >> 16);
            }
        } else {
            uint32_t mean = 0u;
            if (id == 1) {                                   // contrast: mean luma of the current image
                if (threadIdx.x == 0) s_sum = 0ull;
                __syncthreads();
                unsigned long long local = 0ull;
                for (uint32_t i = threadIdx.x; i < npx; i += blockDim.x)
                    local += luma_of((uint32_t)cur[3u * i] | ((uint32_t)cur[3u * i + 1u] << 8) | ((uint32_t)cur[3u * i + 2u] << 16));
                for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
                if ((threadIdx.x & 31) == 0) atomicAdd(&s_sum, local);
                __syncthreads();
                mean = contrast_mean(s_sum, npx);
            }
            if (threadIdx.x < 256) s_lut[threadIdx.x] = (uint8_t)blend_u8(mean, threadIdx.x, alpha, clip);
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < npx * 3u; i += blockDim.x) dst[i] = s_lut[cur[i]];
        }
        first = false;
        __syncthreads();                                     // the next op reads what this one wrote (same CTA: block scope)
    }
    if (first && src != dst)                                 // no op applied: plain copy
        for (uint32_t i = threadIdx.x; i < npx * 3u; i += blockDim.x) dst[i] = src[i];
}

cudaError_t launch_color_jitter(const uint8_t* in, uint8_t* out, const void* recs, int batch, int H, int W, cudaStream_t stream) {
    if (batch <= 0) return cudaSuccess;
    faa_color_jitter_kernel<<<(unsigned)batch, 1024, 0, stream>>>(in, out, reinterpret_cast<const JitterRec*>(recs), H, W);
    return cudaGetLastError();
}

// Lighting (augmentations.py:197-215) sits between ToTensor and Normalize (data.py:70-72): x = u8/255 ; x += rgb[c] ;
// (x - mean) / std - a per-IMAGE normalisation table [3][256] in fp32 with torch's operation order and IEEE division
__global__ void faa_lighting_tables_kernel(const float* __restrict__ rgb, float* __restrict__ tabs, int n, float m0, float m1, float m2,
                                           float s0, float s1, float s2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * 768) return;
    const int img = i / 768, e = i - img * 768, ch = e >> 8, u = e & 255;
    const float mean = ch == 0 ? m0 : ch == 1 ? m1 : m2, sd = ch == 0 ? s0 : ch == 1 ? s1 : s2;
    const float x = __fdiv_rn((float)u, 255.0f);
    const float y = __fadd_rn(x, rgb[img * 3 + ch]);
    tabs[i] = __fdiv_rn(__fadd_rn(y, -mean), sd);
}

cudaError_t launch_lighting_tables(const float* rgb, float* tabs, int n, const float mean[3], const float std[3], cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    faa_lighting_tables_kernel<<<(unsigned)((n * 768 + 255) / 256), 256, 0, stream>>>(rgb, tabs, n, mean[0], mean[1], mean[2], std[0], std[1], std[2]);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------
// EfficientNet crop + Pillow bicubic Resize (data.py:61-62, 76-77, 267-345; faa_core.cuh crop_attempt /
// resize_coeffs).  One CTA per (tile_w x tile_h) output tile of one image, no whole-image state: thread 0 fixes the
// crop box (given, or drawn with philox_crop_box), the CTA builds the horizontal coefficients of its tile's columns
// and the vertical ones of its rows in shared memory, runs the horizontal pass over exactly the crop rows its rows
// read into a uint8 intermediate (one packed RGB word per pixel), then the vertical pass from there, and writes
// uint8 HWC or ToTensor + Normalize (exact fp32 table, then one rounding to fp16 / bf16) NCHW.
// A ragged batch (images != nullptr) differs only in where thread 0 finds the image and its size: every per-image
// quantity (box, coefficients, rows) already derives from the box, and the plan is made for the batch's largest height
// and largest width (see launch_crop_resize).
struct CropResizeParams {
    const uint8_t* in;           // [B][H][W][3] (uniform batch)
    const CropImage* images;     // [B] descriptors (ragged batch) or nullptr
    void* out;                   // [B][out_h][out_w][3] uint8 or [B][3][out_h][out_w]
    const CropBox* boxes;        // [B] or nullptr: draw with cfg
    CropCfg cfg;
    int32_t H, W, out_h, out_w;  // H x W: every image's size (uniform) or the largest height / width (ragged)
    int32_t tile_w, tile_h, tw_shift;   // tile_w = 1 << tw_shift
    int32_t kx_cap, ky_cap, rows_cap;   // taps per column / row and intermediate rows a CTA can hold
    float mean[3], std[3];
};

// (not inlined: the fp64 division / sqrt slow paths inside would otherwise make the kernel spill)
__device__ __noinline__ CropBox draw_crop_box(const CropCfg* c, uint64_t index, int H, int W) {
    return philox_crop_box(*c, index, H, W);
}

template <int OUT>
__global__ void __launch_bounds__(256, 4) faa_crop_resize_kernel(const __grid_constant__ CropResizeParams P) {
    extern __shared__ int32_t cr_smem[];
    __shared__ float s_norm[OUT == OUT_U8_HWC ? 1 : 768];
    __shared__ CropBox s_box;
    __shared__ const uint8_t* s_src;
    __shared__ int32_t s_src_w;
    const int img = blockIdx.z, tid = threadIdx.x;
    const int ox0 = blockIdx.x * P.tile_w, oy0 = blockIdx.y * P.tile_h;
    const int ncols = min(P.tile_w, P.out_w - ox0), nrows = min(P.tile_h, P.out_h - oy0);
    int32_t* hk = cr_smem;                                   // [tile_w][kx_cap]
    int32_t* hmin = hk + P.tile_w * P.kx_cap;                // [tile_w]
    int32_t* hn = hmin + P.tile_w;
    int32_t* vk = hn + P.tile_w;                             // [tile_h][ky_cap]
    int32_t* vmin = vk + P.tile_h * P.ky_cap;
    int32_t* vn = vmin + P.tile_h;
    uint32_t* inter = reinterpret_cast<uint32_t*>(vn + P.tile_h);   // [rows_cap][tile_w]
    if (tid == 0) {
        CropImage d;
        if (P.images != nullptr) d = P.images[img];
        else { d.data = P.in + (size_t)img * P.H * P.W * 3u; d.h = P.H; d.w = P.W; }
        s_src = d.data; s_src_w = d.w;
        s_box = P.boxes ? P.boxes[img] : draw_crop_box(&P.cfg, P.cfg.rng.first_index + (uint64_t)img, d.h, d.w);
    }
    if (OUT != OUT_U8_HWC) {                                 // data.py:76-78: x = u8 / 255 ; (x - mean) / std in fp32
        for (int i = tid; i < 768; i += blockDim.x) {
            const int ch = i >> 8;
            s_norm[i] = __fdiv_rn(__fadd_rn(__fdiv_rn((float)(i & 255), 255.0f), -P.mean[ch]), P.std[ch]);
        }
    }
    __syncthreads();
    const CropBox b = s_box;
    if (tid < ncols) {
        int xm;
        hn[tid] = resize_coeffs(b.w, P.out_w, ox0 + tid, &xm, hk + tid * P.kx_cap);
        hmin[tid] = xm;
    } else if (tid >= 128 && tid - 128 < nrows) {
        const int r = tid - 128;
        int ym;
        vn[r] = resize_coeffs(b.h, P.out_h, oy0 + r, &ym, vk + r * P.ky_cap);
        vmin[r] = ym;
    }
    __syncthreads();
    const int r0 = vmin[0];
    // crop rows this tile reads: at most (tile_h - 1) * scale_y + taps + 1 <= rows_cap (plan_crop_resize bounds them
    // for every crop of the source, with one row to spare)
    const int rows = vmin[nrows - 1] + vn[nrows - 1] - r0;
    assert(rows <= P.rows_cap);
    // horizontal pass: crop rows [r0, r0 + rows) x this tile's columns -> inter
    const uint8_t* const img_src = s_src;
    const size_t pitch = (size_t)s_src_w * 3u;
    const int tmask = P.tile_w - 1;
    for (int i = tid; i < (rows << P.tw_shift); i += blockDim.x) {
        const int r = i >> P.tw_shift, c = i & tmask;
        if (c >= ncols) continue;
        const uint8_t* src = img_src + (size_t)(b.y0 + r0 + r) * pitch + (size_t)(b.x0 + hmin[c]) * 3u;
        const int32_t* k = hk + c * P.kx_cap;
        const int n = hn[c];
        int32_t s0 = 1 << (kResPrecisionBits - 1), s1 = s0, s2 = s0;
        for (int t = 0; t < n; ++t) {
            const int32_t w = k[t];
            s0 += (int32_t)__ldg(src + 3 * t) * w;
            s1 += (int32_t)__ldg(src + 3 * t + 1) * w;
            s2 += (int32_t)__ldg(src + 3 * t + 2) * w;
        }
        inter[(r << P.tw_shift) + c] = resize_clip8(s0) | (resize_clip8(s1) << 8) | (resize_clip8(s2) << 16);
    }
    __syncthreads();
    // vertical pass: inter -> output
    for (int i = tid; i < (nrows << P.tw_shift); i += blockDim.x) {
        const int r = i >> P.tw_shift, c = i & tmask;
        if (c >= ncols) continue;
        const uint32_t* col = inter + ((vmin[r] - r0) << P.tw_shift) + c;
        const int32_t* k = vk + r * P.ky_cap;
        const int n = vn[r];
        int32_t s0 = 1 << (kResPrecisionBits - 1), s1 = s0, s2 = s0;
        for (int t = 0; t < n; ++t) {
            const int32_t w = k[t];
            const uint32_t p = col[t << P.tw_shift];
            s0 += (int32_t)(p & 255u) * w;
            s1 += (int32_t)((p >> 8) & 255u) * w;
            s2 += (int32_t)((p >> 16) & 255u) * w;
        }
        const uint32_t v0 = resize_clip8(s0), v1 = resize_clip8(s1), v2 = resize_clip8(s2);
        const int oy = oy0 + r, ox = ox0 + c;
        if constexpr (OUT == OUT_U8_HWC) {
            uint8_t* o = reinterpret_cast<uint8_t*>(P.out) + (((size_t)img * P.out_h + oy) * P.out_w + ox) * 3u;
            o[0] = (uint8_t)v0; o[1] = (uint8_t)v1; o[2] = (uint8_t)v2;
        } else {
            const size_t plane = (size_t)P.out_h * P.out_w;
            const size_t off = (size_t)img * 3u * plane + (size_t)oy * P.out_w + ox;
            const float f0 = s_norm[v0], f1 = s_norm[256 + v1], f2 = s_norm[512 + v2];
            if constexpr (OUT == OUT_F32) {
                float* o = reinterpret_cast<float*>(P.out) + off;
                o[0] = f0; o[plane] = f1; o[2 * plane] = f2;
            } else if constexpr (OUT == OUT_F16) {
                __half* o = reinterpret_cast<__half*>(P.out) + off;
                o[0] = __float2half_rn(f0); o[plane] = __float2half_rn(f1); o[2 * plane] = __float2half_rn(f2);
            } else {
                __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(P.out) + off;
                o[0] = __float2bfloat16_rn(f0); o[plane] = __float2bfloat16_rn(f1); o[2 * plane] = __float2bfloat16_rn(f2);
            }
        }
    }
}

// Tile of a crop-resize launch: the largest tile whose coefficients and intermediate fit, for ANY crop of the
// h x w source (a crop's scale, taps and rows are bounded by the full image's).  Prefers <= 48 KB (several CTAs
// per SM); the 1 x 1 tile of an 8192 x 8192 source needs ~96 KB, so every valid size has a tile.
// A ragged batch is planned at (largest height, largest width), which may come from two different images.  That plan
// holds every image h x w with h <= H and w <= W: its crop box is at most w wide and h high, resize_ksize is
// non-decreasing in the input size (scale, support and their ceiling all grow with it), so the taps of a column are at
// most min(w, ksize(w)) <= kx and those of a row at most ky; the vertical scale is box_h / out_h <= H / out_h, so the
// rows a tile reads are at most min(h, ceil((th - 1) * sy) + ky + 2) <= rows.  The kernel's assert keeps checking it.
CropResizeTile plan_crop_resize(int H, int W, int out_h, int out_w) {
    const int kx = min(W, resize_ksize(W, out_w)), ky = min(H, resize_ksize(H, out_h));
    const double sy = (double)H / out_h > 1.0 ? (double)H / out_h : 1.0;
    int tw0 = 1, shift0 = 0;
    while (tw0 < 32 && tw0 < out_w) { tw0 *= 2; ++shift0; }
    CropResizeTile best; best.smem = 0;
    for (int pass = 0; pass < 2 && best.smem == 0; ++pass) {
        const size_t limit = pass == 0 ? 48u * 1024u : 220u * 1024u;
        for (int tw = tw0, sh = shift0; tw >= 1 && best.smem == 0; tw /= 2, --sh)
            for (int th = 32; th >= 1; th /= 2) {
                if (th > 1 && th / 2 >= out_h) continue;
                const int rows = min(H, (int)ceil((th - 1) * sy) + ky + 2);
                const size_t smem = 4u * ((size_t)tw * (kx + 2) + (size_t)th * (ky + 2) + (size_t)rows * tw);
                if (smem <= limit) {
                    best.tile_w = tw; best.tile_h = th; best.tw_shift = sh; best.kx_cap = kx; best.ky_cap = ky;
                    best.rows_cap = rows; best.smem = smem;
                    break;
                }
            }
    }
    return best;
}

template <auto Kernel> static cudaError_t reserve_dyn_smem(size_t dyn);     // (defined below)

// The dynamic shared memory limit is always raised to the plan's size: the kernel's static shared memory (the
// normalisation table) counts against the default 48 KB too, so a plan just under 48 KB of dynamic memory would not
// launch without it.
template <int OUT>
static cudaError_t launch_crop_resize_as(const CropResizeParams& P, dim3 grid, size_t smem, cudaStream_t stream) {
    if (cudaError_t e = reserve_dyn_smem<faa_crop_resize_kernel<OUT>>(smem)) return e;
    faa_crop_resize_kernel<OUT><<<grid, 256, smem, stream>>>(P);
    return cudaGetLastError();
}

cudaError_t launch_crop_resize(const uint8_t* in, const CropImage* images, void* out, int batch, int H, int W, int out_h,
                               int out_w, int out_type, const float mean[3], const float std[3], const CropBox* boxes,
                               const CropCfg& cfg, const CropResizeTile& t, cudaStream_t stream) {
    if (batch <= 0) return cudaSuccess;
    CropResizeParams P;
    P.in = in; P.images = images; P.out = out; P.boxes = boxes; P.cfg = cfg;
    P.H = H; P.W = W; P.out_h = out_h; P.out_w = out_w;
    P.tile_w = t.tile_w; P.tile_h = t.tile_h; P.tw_shift = t.tw_shift;
    P.kx_cap = t.kx_cap; P.ky_cap = t.ky_cap; P.rows_cap = t.rows_cap;
    for (int c = 0; c < 3; ++c) { P.mean[c] = mean[c]; P.std[c] = std[c]; }
    const dim3 grid((unsigned)((out_w + t.tile_w - 1) / t.tile_w), (unsigned)((out_h + t.tile_h - 1) / t.tile_h), (unsigned)batch);
    switch (out_type) {
    case OUT_F16:    return launch_crop_resize_as<OUT_F16>(P, grid, t.smem, stream);
    case OUT_BF16:   return launch_crop_resize_as<OUT_BF16>(P, grid, t.smem, stream);
    case OUT_F32:    return launch_crop_resize_as<OUT_F32>(P, grid, t.smem, stream);
    case OUT_U8_HWC: return launch_crop_resize_as<OUT_U8_HWC>(P, grid, t.smem, stream);
    default: return cudaErrorInvalidValue;
    }
}

// ---------------------------------------------------------------------------------------
// Mixup of AUGMENTED uint8 images (aug_mixup.py:13-23 behind data.py's ToTensor + Normalize + CutoutDefault):
//     out[i] = norm(a_i) * lam + norm(b_i) * (1 - lam)           (fp32, separate roundings, then the output dtype)
// a = this sample's augmented uint8 HWC image, b = its partner's (same array or a received one); the CutoutDefault
// boxes act on the normalised values, so each source brings its own zero box.  The op streams: 6 bytes in, 3 values
// out per pixel; one quad per thread and iteration, 8-byte plane stores.
struct MixU8Params {
    const uint8_t* a;            // [batch][H][W][3]
    const uint8_t* b;            // partner pool [nb][H][W][3]
    const int32_t* partner;      // [batch] index into b
    const uint8_t* const* b_ptrs;  // optional [batch]: the partner IMAGE of every sample (may be another GPU's memory, mapped
                                 // through NVLink peer access: the exchange happens inside this kernel's loads); then zb_b is
                                 // indexed per sample and b / partner are unused
    const int16_t* zb_a;         // [batch][4] zero boxes (y0, y1, x0, x1; half-open) or nullptr
    const int16_t* zb_b;         // [nb][4] or nullptr
    const float* norm_tab;       // [3][256] exact ToTensor+Normalize values
    void* out;                   // [batch][3][H][W]
    int32_t H, W;
    float lam, oml;
};

template <typename T>
__global__ void __launch_bounds__(256) faa_mix_u8_kernel(const __grid_constant__ MixU8Params P) {
    // both products of aug_mixup.py:21 as tables: round(norm(b) * lam), round(norm(b) * (1 - lam)) - the same two roundings
    // as the reference's tensor ops, then ONE add per value in the loop
    __shared__ float s_la[768], s_ob[768];
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
        const float t = __ldg(P.norm_tab + i);
        s_la[i] = f_mul(t, P.lam); s_ob[i] = f_mul(t, P.oml);
    }
    __syncthreads();
    const float za_val = f_mul(0.0f, P.lam), zb_val = f_mul(0.0f, P.oml);     // a zeroed (CutoutDefault) value, scaled
    const int img = blockIdx.y, pi = P.b_ptrs ? img : __ldg(P.partner + img);
    const uint32_t npx = (uint32_t)P.H * (uint32_t)P.W, nq = npx >> 2;
    const uint32_t* a = reinterpret_cast<const uint32_t*>(P.a + (size_t)img * npx * 3u);
    const uint32_t* b = P.b_ptrs ? reinterpret_cast<const uint32_t*>(__ldg(reinterpret_cast<const unsigned long long*>(P.b_ptrs) + img))
                                 : reinterpret_cast<const uint32_t*>(P.b + (size_t)pi * npx * 3u);
    T* o = reinterpret_cast<T*>(P.out) + (size_t)img * npx * 3u;
    int za[4] = {0, 0, 0, 0}, zb[4] = {0, 0, 0, 0};
    if (P.zb_a) for (int k = 0; k < 4; ++k) za[k] = P.zb_a[img * 4 + k];
    if (P.zb_b) for (int k = 0; k < 4; ++k) zb[k] = P.zb_b[pi * 4 + k];
    const bool boxes = (za[1] > za[0] && za[3] > za[2]) || (zb[1] > zb[0] && zb[3] > zb[2]);
    const uint32_t qpr = (uint32_t)P.W >> 2;
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
        uint32_t pa[4], pb[4];
        unpack12(__ldg(a + 3u * q), __ldg(a + 3u * q + 1u), __ldg(a + 3u * q + 2u), pa);
        unpack12(__ldg(b + 3u * q), __ldg(b + 3u * q + 1u), __ldg(b + 3u * q + 2u), pb);
        uint32_t ma = 0u, mb = 0u;                           // pixels of the quad inside the zero boxes
        if (boxes) {
            const int y = (int)(q / qpr), x0 = (int)(q - (uint32_t)y * qpr) * 4;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                ma |= (uint32_t)(y >= za[0] && y < za[1] && x0 + k >= za[2] && x0 + k < za[3]) << k;
                mb |= (uint32_t)(y >= zb[0] && y < zb[1] && x0 + k >= zb[2] && x0 + k < zb[3]) << k;
            }
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float v[4];
            if (ma | mb) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float fa = ((ma >> k) & 1u) ? za_val : s_la[ch * 256 + ((pa[k] >> (8 * ch)) & 255u)];
                    const float fb = ((mb >> k) & 1u) ? zb_val : s_ob[ch * 256 + ((pb[k] >> (8 * ch)) & 255u)];
                    v[k] = f_add(fa, fb);                                         // aug_mixup.py:21
                }
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    v[k] = f_add(s_la[ch * 256 + ((pa[k] >> (8 * ch)) & 255u)], s_ob[ch * 256 + ((pb[k] >> (8 * ch)) & 255u)]);
            }
            T* op = o + (size_t)ch * npx + 4u * q;
            if constexpr (sizeof(T) == 4) {
                *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
            } else if constexpr (std::is_same<T, __half>::value) {
                __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
                uint2 u; u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(op) = u;
            } else {
                __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
                uint2 u; u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
                *reinterpret_cast<uint2*>(op) = u;
            }
        }
    }
}

cudaError_t launch_mix_u8(const uint8_t* a, const uint8_t* b, const int32_t* partner, const int16_t* zb_a, const int16_t* zb_b,
                          const float* norm_tab, void* out, int batch, int H, int W, int dtype, float lam, float oml,
                          cudaStream_t stream, const uint8_t* const* b_ptrs) {
    if (batch <= 0) return cudaSuccess;
    MixU8Params P; P.a = a; P.b = b; P.partner = partner; P.zb_a = zb_a; P.zb_b = zb_b; P.norm_tab = norm_tab; P.out = out;
    P.b_ptrs = b_ptrs;
    P.H = H; P.W = W; P.lam = lam; P.oml = oml;
    const uint32_t nq = (uint32_t)H * (uint32_t)W / 4u;
    unsigned gx = (nq + 255u) / 256u;
    if (gx > 8) gx = 8;                                      // ~6 quads per thread at 224x224
    dim3 grid(gx, (unsigned)batch, 1);
    switch (dtype) {
    case OUT_F16:  faa_mix_u8_kernel<__half><<<grid, 256, 0, stream>>>(P); break;
    case OUT_BF16: faa_mix_u8_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(P); break;
    case OUT_F32:  faa_mix_u8_kernel<float><<<grid, 256, 0, stream>>>(P); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

#endif  // !FAA_TU_OUT

// raise Kernel's dynamic shared memory limit to `dyn` bytes on the current device if it is below that
// (the attribute is per kernel AND per device)
template <auto Kernel>
static cudaError_t reserve_dyn_smem(size_t dyn) {
    static size_t configured[kMaxDevices] = {};
    int dev = 0;
    if (cudaError_t e = cudaGetDevice(&dev)) return e;
    if (dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (dyn > configured[dev]) {
        if (cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn)) return e;
        configured[dev] = dyn;
    }
    return cudaSuccess;
}

template <int OUT, int NSRC, bool TAB>
static cudaError_t launch_one(const AugParams& p, cudaStream_t stream) {
    const size_t dyn = (size_t)p.geo[0].band_cap * NSRC + (size_t)p.mat_cap;
    if (cudaError_t e = reserve_dyn_smem<faa_augment_kernel<OUT, NSRC, TAB>>(dyn)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)p.bands, (unsigned)p.B, 1);
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)p.bands;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;    // overlap with the resolve kernel
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (p.pdl || p.chain) ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, faa_augment_kernel<OUT, NSRC, TAB>, p);
}

#if defined(FAA_TU_OUT) && FAA_TU_OUT == 3   // OUT_U8_HWC
cudaError_t launch_augment_ragged(const RaggedParams& r, int bands, int count, size_t smem, cudaStream_t stream) {
    if (count <= 0) return cudaSuccess;
    if (cudaError_t e = reserve_dyn_smem<faa_augment_ragged_kernel>(smem)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)bands, (unsigned)count, 1);
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)bands;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, faa_augment_ragged_kernel, r);
}
#endif

static inline int rows_of(const AugParams& p) { return (p.grid_y > 0 && p.grid_y < p.B) ? p.grid_y : p.B; }

template <int OUT, bool TAB, bool LEAN>
static cudaError_t launch_light(const AugParams& p, cudaStream_t stream) {
    const size_t dyn = (size_t)p.geo[1].band_cap;
    if (cudaError_t e = reserve_dyn_smem<faa_augment_light_kernel<OUT, TAB, LEAN>>(dyn)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)p.geo[1].bands, (unsigned)rows_of(p), 1);
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = p.chain ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, faa_augment_light_kernel<OUT, TAB, LEAN>, p);
}

template <int OUT, bool TAB>
static cudaError_t launch_mid(const AugParams& p, cudaStream_t stream) {
    const size_t dyn = (size_t)p.geo[0].band_cap;
    if (cudaError_t e = reserve_dyn_smem<faa_augment_mid_kernel<OUT, TAB>>(dyn)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)p.bands, (unsigned)rows_of(p), 1);
    cfg.blockDim = dim3((unsigned)mid_kernel_threads((uint32_t)dyn), 1, 1);
    cfg.dynamicSmemBytes = dyn;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)p.bands;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = p.chain ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, faa_augment_mid_kernel<OUT, TAB>, p);
}

template <int OUT>
cudaError_t launch_out(const AugParams& p, bool mix, bool tab, int which, cudaStream_t stream) {
    if (which == 2) return tab ? launch_mid<OUT, true>(p, stream) : launch_mid<OUT, false>(p, stream);
    if (which == 1) return tab ? launch_light<OUT, true, false>(p, stream) : launch_light<OUT, false, false>(p, stream);
    if (which == 3) return tab ? launch_light<OUT, true, true>(p, stream) : launch_light<OUT, false, true>(p, stream);
    if constexpr (OUT != OUT_U8_HWC) {                   // fused Mixup needs a float output
        if (mix) return tab ? launch_one<OUT, 2, true>(p, stream) : launch_one<OUT, 2, false>(p, stream);
    }
    return tab ? launch_one<OUT, 1, true>(p, stream) : launch_one<OUT, 1, false>(p, stream);
}

#ifdef FAA_TU_OUT
template cudaError_t launch_out<FAA_TU_OUT>(const AugParams&, bool, bool, int, cudaStream_t);
#else
extern template cudaError_t launch_out<OUT_F16>(const AugParams&, bool, bool, int, cudaStream_t);
extern template cudaError_t launch_out<OUT_BF16>(const AugParams&, bool, bool, int, cudaStream_t);
extern template cudaError_t launch_out<OUT_F32>(const AugParams&, bool, bool, int, cudaStream_t);
extern template cudaError_t launch_out<OUT_U8_HWC>(const AugParams&, bool, bool, int, cudaStream_t);

// which == 0: the cluster kernel (all images, or the heavy part of a split launch);
// which == 1: the streaming kernel for the light part of a split launch (p.n_heavy != nullptr);
// which == 2: the statistics / Sharpness kernel for the mid part of a three-way split;
// which == 3: the lean variant of the streaming kernel (LaunchPlan::lean_light)
cudaError_t launch_augment(const AugParams& p, int out_type, bool use_tab, int which, cudaStream_t stream) {
    if (p.B <= 0) return cudaSuccess;
    const bool mix = p.partner != nullptr;
    switch (out_type) {
    case OUT_F16:  return launch_out<OUT_F16>(p, mix, use_tab, which, stream);
    case OUT_BF16: return launch_out<OUT_BF16>(p, mix, use_tab, which, stream);
    case OUT_F32:  return launch_out<OUT_F32>(p, mix, true, which, stream);
    case OUT_U8_HWC: return launch_out<OUT_U8_HWC>(p, false, false, which, stream);
    default: return cudaErrorInvalidValue;
    }
}

int resident_ctas_per_sm(int which) { return which == 1 ? FAA_LIGHT_CTAS : which == 3 ? kLeanLightCtas : which == 2 ? 2 : FAA_MIN_CTAS; }

unsigned augment_cta_count(const AugParams& p, int which) {
    if (p.B <= 0) return 0u;
    if (which == 1 || which == 3) return (unsigned)p.geo[1].bands * (unsigned)rows_of(p);
    if (which == 2) return (unsigned)p.bands * (unsigned)rows_of(p);
    return (unsigned)p.bands * (unsigned)p.B;
}

cudaError_t launch_resolve(const ResolveParams& p, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    int threads = p.n >= 1024 ? 1024 : ((p.n + 31) / 32) * 32;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1, 1, 1);
    cfg.blockDim = dim3((unsigned)threads, 1, 1);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = p.pdl ? 1 : 0;
    return p.cands != nullptr ? cudaLaunchKernelEx(&cfg, faa_resolve_kernel<true>, p)
                              : cudaLaunchKernelEx(&cfg, faa_resolve_kernel<false>, p);
}

cudaError_t launch_resolve_ragged(const ResolveParams& p, const RaggedImg* imgs, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    const int threads = p.n >= 1024 ? 1024 : ((p.n + 31) / 32) * 32;
    if (p.cands != nullptr) faa_resolve_ragged_kernel<true><<<1, threads, 0, stream>>>(p, imgs);
    else faa_resolve_ragged_kernel<false><<<1, threads, 0, stream>>>(p, imgs);
    return cudaGetLastError();
}

cudaError_t launch_realign(const RaggedCopy* jobs, int n, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    faa_realign_kernel<<<dim3(64, (unsigned)n, 1), 256, 0, stream>>>(jobs);
    return cudaGetLastError();
}

cudaError_t launch_gather(const RaggedCopy* jobs, int n, int ctas, cudaStream_t stream) {
    if (n <= 0 || ctas <= 0) return cudaSuccess;
    faa_gather_kernel<<<ctas, kGatherThreads, 0, stream>>>(jobs, n);
    return cudaGetLastError();
}

cudaError_t launch_mixup(const void* data, void* out, const int64_t* perm, int batch, int64_t n_per_sample,
                         int dtype, float lam, float oml, cudaStream_t stream) {
    if (batch <= 0 || n_per_sample <= 0) return cudaSuccess;
    const int vec = dtype == OUT_F32 ? 4 : 8;
    if (n_per_sample % vec == 0 && ((uintptr_t)data % 16) == 0 && ((uintptr_t)out % 16) == 0) {
        const int64_t n_vec = n_per_sample / vec;
        unsigned gv = (unsigned)((n_vec + 255) / 256);
        if (gv > 32) gv = 32;
        dim3 gridv(gv, (unsigned)batch, 1);
        switch (dtype) {
        case OUT_F16:  faa_mixup_kernel_v<__half, 8><<<gridv, 256, 0, stream>>>((const __half*)data, (__half*)out, perm, n_vec, n_per_sample, lam, oml); break;
        case OUT_BF16: faa_mixup_kernel_v<__nv_bfloat16, 8><<<gridv, 256, 0, stream>>>((const __nv_bfloat16*)data, (__nv_bfloat16*)out, perm, n_vec, n_per_sample, lam, oml); break;
        case OUT_F32:  faa_mixup_kernel_v<float, 4><<<gridv, 256, 0, stream>>>((const float*)data, (float*)out, perm, n_vec, n_per_sample, lam, oml); break;
        default: return cudaErrorInvalidValue;
        }
        return cudaGetLastError();
    }
    unsigned gx = (unsigned)((n_per_sample + 255) / 256);
    if (gx > 64) gx = 64;
    dim3 grid(gx, (unsigned)batch, 1);
    switch (dtype) {
    case OUT_F16:  faa_mixup_kernel<__half><<<grid, 256, 0, stream>>>((const __half*)data, (__half*)out, perm, n_per_sample, lam, oml); break;
    case OUT_BF16: faa_mixup_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)data, (__nv_bfloat16*)out, perm, n_per_sample, lam, oml); break;
    case OUT_F32:  faa_mixup_kernel<float><<<grid, 256, 0, stream>>>((const float*)data, (float*)out, perm, n_per_sample, lam, oml); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

#endif  // FAA_TU_OUT

}  // namespace faa
