// faa_kernels.cuh - launch-side declarations shared by faa_kernels.cu and faa_cabi.cu
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "faa_core.cuh"
#include "faa_jpeg.cuh"

namespace faa {

enum OutType : int32_t { OUT_F16 = 0, OUT_BF16 = 1, OUT_F32 = 2, OUT_U8_HWC = 3 };

// step 1 (one thread per image): decisions -> per-image program
struct ResolveParams {
    const OpRec* ops;           // compiled policy [n_sub][n_op][2]
    const double* probs;        // [n_sub][n_op]
    const Sample* samples;      // [n] resolved decisions, or nullptr -> draw with Philox
    const Box* boxes;           // [n][n_op] (may be nullptr when no Cutout box is needed)
    Prog* progs;                // [n] out
    int32_t* order;             // [n] out: local image indices, most expensive first (optional)
    int32_t* n_heavy;           // out (optional): [0] = end of the heavy segment of the order, [1] = end of the mid segment
    int32_t split;              // 1: sort light programs behind heavy ones (two pixel launches); 2: heavy | mid | light
    Sample* samples_out;        // optional [n]
    Box* boxes_out;             // optional [n][n_op]
    RngCfg rng;
    const int32_t* pos;         // Philox: record t draws global sample rng.first_index + pos[t] (nullptr: + t)
    int32_t first, n;           // images [first, first+n) of the arrays above
    int32_t H, W, out_h, out_w, n_sub, n_op, op_base, apply_tail;
    int32_t allow;              // bit 0: the pixel kernel has a materialisation chunk, bit 1: a global scratch image
    int32_t* ready;             // optional: set to `ticket` (release) once programs / order / n_heavy are written
    int32_t ticket;
    int32_t pdl;                // launch with programmatic stream serialization (chained steps)
    const uint32_t* wait_done;  // optional: before writing anything, spin until *wait_done has reached wait_target (the pixel
    uint32_t wait_target;       // CTAs that read this slot's previous programs count themselves there when they finish)
};
cudaError_t launch_resolve(const ResolveParams& p, cudaStream_t stream);

// AugParams::chain: how a pixel launch is ordered against the kernel in front of it in its stream
enum ChainMode : int32_t {
    CHAIN_STREAM_ORDERED = 0,   // griddepcontrol.wait before the schedule is read (or no programmatic launch at all)
    CHAIN_STEP = 1,             // chained step (resolve, pixel kernels and the next step on ONE stream, programmatic
                                // dependent launches): no griddepcontrol.wait - the ticket orders the programs; the persistent
                                // mid / light kernels release their dependents at once and the slot's next writer waits for
                                // `done`; the cluster kernel releases them once its program is copied
    CHAIN_SELF_RESOLVING = 2,   // self-resolving step: nothing is shared between steps, every CTA releases the next at once
};

// step 2 (one cluster per image): pixels
struct AugParams {
    const uint8_t* in;          // [n_all][H][W][3] uint8
    void* out;                  // [B][3][out_h][out_w] OutT  (or [B][out_h][out_w][3] uint8)
    const Prog* progs;          // [n_all]
    const int32_t* partner;     // [B] index into [0, n_all) or nullptr (no mixup)
    const int32_t* order;       // [n_all] LPT schedule written by the resolve kernel, or nullptr
    const int32_t* n_heavy;     // device counters: schedule entries [0, n_heavy[0]) -> cluster kernel, [n_heavy[0], n_heavy[1]) -> mid
                                // kernel (empty in a two-way split), rest -> light kernel; nullptr = no split
    const float* norm_tab;      // [3][256] exact fp32 ToTensor+Normalize values ([n_all][3][256] when norm_stride != 0)
    int32_t norm_stride;        // 768: one table per image (Lighting, augmentations.py:197-215); 0: one table per launch
    uint8_t* scratch;           // [n_all][H][W][3] uint8 scratch image for Sharpness->gather programs, or nullptr
    int32_t B, H, W, out_h, out_w;
    int32_t first;              // index of this launch's image 0 inside the n_all arrays
    int32_t in_mod;             // > 0: replicated launch (TTA): entry v reads input image v % in_mod
    int32_t use_zero_box;
    int32_t bands;              // CTAs (== cluster size) per image of the cluster kernel (== geo[0].bands)
    BandGeom geo[2];            // [0] cluster kernel, [1] light streaming kernel
    uint32_t rcp_out_qpr, rcp_w, rcp_wq;   // 2^32 / ceil(out_w/4), 2^32 / W, 2^32 / (W/4)  (rounded up) for fastdiv
    uint32_t rcp_opr;           // 2^32 / (W/8) (octet fast paths; 0 when W % 8 != 0)
    int32_t octets;             // 1: 8-pixel fast paths allowed (W % 8 == 0, out size == image size, float output 16-byte aligned)
    int32_t stage;              // 1: TMA-stage the raw row band into shared memory
    int32_t band_cap;           // bytes of dynamic shared memory per staged band
    int32_t crop_pad;           // max |crop_dy| (RandomCrop padding)
    int32_t mat_cap;            // bytes of the materialisation chunk (0: none), a whole number of rows >= 3
    int32_t allow;              // ResolveParams::allow of this launch (the mid kernel's two-stage programs depend on it)
    int32_t pdl;                // launched with programmatic stream serialization
    const int32_t* ready;       // chained steps: spin until *ready == ticket before reading programs / order / n_heavy
    int32_t ticket;
    int32_t chain;              // ChainMode
    int32_t grid_y;             // > 0: launch this many schedule rows (CTAs / clusters per band); each one loops over the
                                // entries row, row + grid_y, ... of its segment.  0: one row per image (B)
    uint32_t* done;             // optional completion counter: every CTA adds 1 when it has finished (release)
    // self-resolving launches (small batches, cluster kernel only): no resolve kernel, no program array - thread 0 of each
    // CTA draws its image's decisions (Philox, the same counters as faa_resolve_kernel) and builds the program itself
    int32_t self_resolve;
    const OpRec* sr_ops; const double* sr_probs;
    RngCfg sr_rng;
    int32_t sr_n_sub, sr_n_op, sr_op_base, sr_apply_tail, sr_allow;
    float scale[3], bias[3];
    float lam, one_minus_lam;   // mixup weights (fp32 of the Python floats)
};
// number of CTAs launch_augment starts for (p, which): what `done` advances by
unsigned augment_cta_count(const AugParams& p, int which);
int resident_ctas_per_sm(int which);     // the launch bounds of the light (1, lean variant 3) / mid (2) / cluster (0) kernel
// which: 0 cluster, 1 light, 2 mid, 3 the light kernel's lean variant (LaunchPlan::lean_light)
cudaError_t launch_augment(const AugParams& p, int out_type, bool use_tab, int which, cudaStream_t stream);

struct CropImage { const uint8_t* data; int32_t h, w; };               // == faa_image_t: one image of a ragged batch

// ragged policy launch (faa_augment_ragged): what the resolve and cluster kernels need per image, by batch position
struct RaggedImg {
    const uint8_t* realigned;   // the library's 4-byte aligned copy of the input, or nullptr: the caller's descriptor
    uint8_t* scratch;           // scratch image of the image's own size for Sharpness -> gather programs, or nullptr
    const OpRec* ops;           // compiled table of the image's size [n_sub][n_op][2]
    int32_t H, W;
    int32_t allow;              // ResolveParams::allow of the image's geometry
    int32_t geom;               // index of the image's per-size AugParams
};
// one launch of the cluster kernel over images list[0, count) of a ragged batch (grid (bands, count))
struct RaggedParams {
    const AugParams* geoms;     // per-size launch parameters (in / out / progs / scratch are per image)
    const RaggedImg* imgs;      // [batch]
    const CropImage* in;        // [batch] the caller's device descriptors
    const CropImage* out;
    const Prog* progs;          // [batch]
    const int32_t* list;        // this launch's images, largest first
};
cudaError_t launch_resolve_ragged(const ResolveParams& p, const RaggedImg* imgs, cudaStream_t stream);
cudaError_t launch_augment_ragged(const RaggedParams& r, int bands, int count, size_t smem, cudaStream_t stream);
// copies n images to 4-byte aligned buffers: src[k] -> dst[k], bytes[k] (device arrays) in one launch
struct RaggedCopy { const uint8_t* src; uint8_t* dst; uint64_t bytes; };
cudaError_t launch_realign(const RaggedCopy* jobs, int n, cudaStream_t stream);

cudaError_t launch_mixup(const void* data, void* out, const int64_t* perm, int batch, int64_t n_per_sample,
                         int dtype, float lam, float one_minus_lam, cudaStream_t stream);

cudaError_t launch_mix_u8(const uint8_t* a, const uint8_t* b, const int32_t* partner, const int16_t* zb_a, const int16_t* zb_b,
                          const float* norm_tab, void* out, int batch, int H, int W, int dtype, float lam, float one_minus_lam,
                          cudaStream_t stream, const uint8_t* const* b_ptrs = nullptr);

cudaError_t launch_color_jitter(const uint8_t* in, uint8_t* out, const void* recs, int batch, int H, int W, cudaStream_t stream);
// EfficientNet crop + bicubic resize (faa_crop_resize_kernel): output tile and shared-memory plan
struct CropResizeTile { int32_t tile_w, tile_h, tw_shift, kx_cap, ky_cap, rows_cap; size_t smem; };
CropResizeTile plan_crop_resize(int H, int W, int out_h, int out_w);     // smem == 0: nothing fits
// images == nullptr: `in` is [batch][H][W][3]; else image i is images[i] (device array) and H x W is only the plan's size
cudaError_t launch_crop_resize(const uint8_t* in, const CropImage* images, void* out, int batch, int H, int W, int out_h,
                               int out_w, int out_type, const float mean[3], const float std[3], const CropBox* boxes,
                               const CropCfg& cfg, const CropResizeTile& t, cudaStream_t stream);
cudaError_t launch_lighting_tables(const float* rgb, float* tabs, int n, const float mean[3], const float std[3], cudaStream_t stream);

// baseline JPEG decode (faa_jpeg.cu): what one faa_jpeg_decode call hands its two kernels
struct JpegJob {                // per image of the call, plus one sentinel entry holding the total tile count
    int64_t coef;               // first block of the image's coefficient planes in `coef`
    int32_t seg;                // first entry of the image's restart-segment starts in `segs`
    int32_t tile0;              // first reconstruct CTA of the image
};
struct JpegDecodeParams {
    const JpegHeader* hdrs;     // [batch] (device copy)
    const JpegTable* pool;      // table pool the headers index
    const uint8_t* src;         // file i is bytes [hdrs[i].offset, + hdrs[i].len)
    const JpegJob* jobs;        // [batch + 1]
    const CropImage* out;       // [batch] uint8 HWC destinations
    int16_t* coef;              // coefficient buffer (the decoder handle's)
    int32_t* segs;              // restart-segment starts, relative to each scan (-1: marker not found)
    int32_t* status;            // [batch] JpegStatus bits
    int32_t batch;
    // scan index: image i's points are points[first[i], first[i + 1]) (decode: null = none; index build: the
    // capacities, with the points written in count[i])
    const int64_t* first;
    JpegSync* points;
    int32_t* count;             // [batch] (index build, recording decode)
    // recording decode only (null otherwise): image i's recorded points go to rec_points[rec_first[i], rec_first[i + 1])
    const int64_t* rec_first;
    JpegSync* rec_points;
};
// found: the found decode's instantiation (counts from faa_jpeg_find_kernel, faa_jpeg_decode's find)
cudaError_t launch_jpeg_entropy(const JpegDecodeParams& p, cudaStream_t stream, bool found = false);
cudaError_t launch_jpeg_reconstruct(const JpegDecodeParams& p, int n_tiles, cudaStream_t stream);
cudaError_t launch_jpeg_index(const JpegDecodeParams& p, cudaStream_t stream);
// finds scan indexes into rec_points / rec_first, counts into count, skipping images with input points (first, may be
// null); mark: a prefix that did not converge gets count ~n
cudaError_t launch_jpeg_find(const JpegDecodeParams& p, bool mark, cudaStream_t stream);
// progressive entropy decode (faa_jpeg_decode_progressive): one CTA per image; the reconstruct kernel follows it
struct JpegProgressiveParams {
    const JpegHeader* hdrs;     // [batch] (device copy)
    const JpegTable* pool;
    const uint8_t* src;
    const JpegJob* jobs;        // [batch + 1]; seg: first entry of the image's segment starts (all its scans)
    const JpegScan* scans;      // image i's scans are scans[scan_first[i], scan_first[i + 1])
    const int64_t* scan_first;
    int16_t* coef;
    int32_t* segs;
    int32_t* status;
    int32_t batch;
};
cudaError_t launch_jpeg_progressive(const JpegProgressiveParams& p, cudaStream_t stream);

}  // namespace faa
