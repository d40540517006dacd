/*
 * faa_b200.h - C ABI of the H100-native Fast AutoAugment augmentation hot path.
 *
 * Plain C: opaque handle, plain pointers and sizes, int status returns, no C++
 * or torch types, no exceptions across the boundary.  Every device entry point
 * takes an explicit CUDA stream (passed as void*, i.e. a cudaStream_t) and is
 * asynchronous with respect to the host; the caller owns every device buffer,
 * the library owns only the policy handle and its small device-side tables.
 *
 * The reference (kakaobrain/fast-autoaugment @ 2424224) has no FFI: its
 * boundary for this path is a set of Python callables.  Each entry point below
 * names the reference interface it replaces (file:line relative to the
 * reference root).  The Python mirror of that surface lives in
 * fast_autoaugment_b200/ and binds this header with ctypes; INTEGRATION.md
 * shows the binding a reference maintainer would add.
 */
#ifndef FAA_B200_H
#define FAA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FAA_ABI_VERSION 2
#define FAA_MAX_FUSED_OPS 2      /* ops of one sub-policy applied by one launch */
#define FAA_MAX_POLICY_OPS 8     /* ops per sub-policy (search.py --num-op); >2 runs as chained launches */
#define FAA_MAX_DIM 8192         /* max H or W */

/* status codes; the Python layer maps them to the reference's exceptions */
enum faa_status {
    FAA_OK = 0,
    FAA_ERR_UNKNOWN_OP = 1,   /* KeyError      - augmentations.py:189 get_augment */
    FAA_ERR_MAGNITUDE = 2,    /* AssertionError- augmentations.py:14,21,28,36,44,51,58,81,86,92,98,103,108,113,118 */
    FAA_ERR_VALUE = 3,        /* ValueError    - bad argument */
    FAA_ERR_CUDA = 4,         /* RuntimeError  - CUDA runtime error, see faa_last_error() */
    FAA_ERR_NO_DEVICE = 5,    /* RuntimeError  - no CUDA device: there is NO CPU fallback */
    FAA_ERR_UNSUPPORTED = 6   /* RuntimeError  - shape / option outside what the kernels handle */
};

/* op ids = position in augment_list(for_autoaug=True), augmentations.py:156-182 */
enum faa_op_id {
    FAA_SHEAR_X = 0, FAA_SHEAR_Y = 1, FAA_TRANSLATE_X = 2, FAA_TRANSLATE_Y = 3, FAA_ROTATE = 4,
    FAA_AUTOCONTRAST = 5, FAA_INVERT = 6, FAA_EQUALIZE = 7, FAA_SOLARIZE = 8, FAA_POSTERIZE = 9,
    FAA_CONTRAST = 10, FAA_COLOR = 11, FAA_BRIGHTNESS = 12, FAA_SHARPNESS = 13, FAA_CUTOUT = 14,
    FAA_CUTOUT_ABS = 15, FAA_POSTERIZE2 = 16, FAA_TRANSLATE_X_ABS = 17, FAA_TRANSLATE_Y_ABS = 18,
    FAA_NUM_OPS = 19
};

/* which random draws an applied op consumes (augmentations.py:15,22,29,37,45,52,59,131-132) */
enum faa_draw { FAA_DRAW_NONE = 0, FAA_DRAW_MIRROR = 1, FAA_DRAW_BOX = 2 };

enum faa_dtype { FAA_F16 = 0, FAA_BF16 = 1, FAA_F32 = 2, FAA_U8_HWC = 3 };

/*
 * Per-sample resolved decisions: what the reference's RNG draws decided for one
 * image (data.py:257-264 Augmentation.__call__, torchvision RandomCrop /
 * RandomHorizontalFlip data.py:40-41, CutoutDefault data.py:235-244).
 * Filled on the host by the parity sampler or on the device by the Philox one.
 */
typedef struct faa_sample {
    uint16_t sub;          /* chosen sub-policy (random.choice, data.py:259)              */
    uint8_t  gate;         /* bit j: op j passed its `random.random() > pr` gate (:261)    */
    uint8_t  sign;         /* bit j: op j drew the mirrored (-v) variant                   */
    int8_t   crop_dy;      /* RandomCrop: top  - padding  (source row = out row + crop_dy) */
    int8_t   crop_dx;      /* RandomCrop: left - padding                                   */
    uint8_t  flip;         /* RandomHorizontalFlip fired                                   */
    uint8_t  reserved;
    int16_t  zero_box[4];  /* CutoutDefault half-open, clipped: y1, y2, x1, x2 (data.py:241-246) */
} faa_sample_t;            /* 16 bytes */

/* per-sample, per-op inclusive Cutout rectangle x0, y0, x1, y1 (augmentations.py:134-143),
 * already truncated to integers, NOT yet clipped to the image */
typedef struct faa_box { int16_t x0, y0, x1, y1; } faa_box_t;

/* the part of the train chain behind the policy (data.py:39-44, 64, 70-72, 111-112) */
typedef struct faa_tail {
    int32_t out_h, out_w;     /* RandomCrop size (== H, W when there is no crop)            */
    int32_t out_dtype;        /* enum faa_dtype; FAA_U8_HWC skips ToTensor/Normalize         */
    int32_t use_zero_box;     /* apply faa_sample.zero_box (CutoutDefault)                   */
    float   mean[3], std[3];  /* Normalize                                                  */
    int32_t crop_pad;         /* RandomCrop padding = bound on |crop_dy| (sizes the staged band; a hint) */
    int32_t reserved;
} faa_tail_t;

/* parameters of the device-side (Philox4x32-10) sampler: the distribution of every draw
 * is the reference's, the stream is not (statistical equivalence, not replay) */
typedef struct faa_rng {
    uint64_t seed;            /* key                                                        */
    uint64_t first_index;     /* global index of sample 0 of this call (shard offset)        */
    int32_t  crop_pad;        /* RandomCrop padding (0 = no crop)                            */
    int32_t  hflip;           /* RandomHorizontalFlip present                                */
    int32_t  zero_box_len;    /* CutoutDefault length (0 = off)                              */
    int32_t  reserved;
} faa_rng_t;

typedef struct faa_policy faa_policy_t;

/* ---- misc ------------------------------------------------------------------ */
int         faa_abi_version(void);
const char* faa_last_error(void);          /* thread-local message of the last failing call */
int         faa_device_count(void);        /* 0 when no usable CUDA device */
int         faa_op_id_from_name(const char* name);   /* -1 if unknown; names of augment_list() */
const char* faa_op_name(int op_id);
int         faa_op_range(int op_id, double* low, double* high);   /* augmentations.py:157-181 */

/* ---- policy: replaces Augmentation.__init__ (data.py:254-255) over the archive.py
 *      list-of-sub-policies format.  ops/probs/levels are row-major [n_sub][n_op].
 *      Like the reference, an unknown op / out-of-range magnitude is only an error when the op
 *      is actually applied: the host sampler reports it then (KeyError / AssertionError); the
 *      device sampler, which cannot raise, refuses such a policy up front.            */
int faa_policy_create(const int32_t* op_ids, const double* probs, const double* levels,
                      int n_sub, int n_op, faa_policy_t** out);
int faa_policy_destroy(faa_policy_t* p);
int faa_policy_dims(const faa_policy_t* p, int* n_sub, int* n_op);
/* host-side compiled op record (32 bytes) for (sub, op, sign) at image size (h, w):
 * exposes the level->magnitude->fixed-point compilation (augmentations.py:192-194 + Pillow
 * matrix set-up) for tests and foreign hosts.  No GPU needed. */
int faa_policy_compiled_op(faa_policy_t* p, int h, int w, int sub, int op, int sign, int32_t out8[8]);
int faa_policy_draw_kind(const faa_policy_t* p, int sub, int op);     /* enum faa_draw */
/* CutoutAbs box from the two uniforms (augmentations.py:131-137), host helper */
int faa_cutout_box(const faa_policy_t* p, int h, int w, int sub, int op, double ux, double uy,
                   faa_box_t* out);

/* ---- host parity sampler: replays Augmentation.__call__'s draws (data.py:257-264) for
 *      `batch` images drawn one after another, from explicit MT19937 states of Python's
 *      `random` (624 words + index) and numpy's legacy global RandomState (same layout).
 *      States are advanced in place.  Tail draws (torch generator) are not covered here. */
int faa_sample_policy_mt(const faa_policy_t* p, int batch, int h, int w,
                         uint32_t py_state[625], uint32_t np_state[625],
                         faa_sample_t* out_samples, faa_box_t* out_boxes /* [batch][n_op] */);

/* ---- device sampler (Philox): fills samples/boxes on the device -------------- */
int faa_sample_philox(faa_policy_t* p, int batch, int h, int w, const faa_tail_t* tail,
                      const faa_rng_t* rng, faa_sample_t* d_samples, faa_box_t* d_boxes,
                      void* stream);
/* the same sampler at given positions: record k (k < n) holds the decisions of global sample
 * rng->first_index + d_pos[k] (d_pos: n non-negative int32 on the device; NULL = 0..n-1, which is
 * faa_sample_philox), drawn for an h x w image.  The per-image Augmentation(policy) draws of the
 * ImageNet train chain (data.py:60, 257-264) on a batch of mixed source sizes: the images of one
 * size are augmented together, each with the decisions of its position in the batch. */
int faa_sample_philox_at(faa_policy_t* p, int n, int h, int w, const faa_tail_t* tail,
                         const faa_rng_t* rng, const int32_t* d_pos, faa_sample_t* d_samples,
                         faa_box_t* d_boxes, void* stream);
/* how many per-size device tables of compiled ops the handle holds, and their bytes (one per image
 * size it has augmented or sampled; they live as long as the handle) */
int faa_policy_cached_tables(faa_policy_t* p, int* n_tables, uint64_t* bytes);

/* ---- the hot path: replaces, for a whole batch, Augmentation.__call__ (data.py:257-264)
 *      -> apply_augment (augmentations.py:192-194) -> the 19 ops (augmentations.py:13-144)
 *      -> RandomCrop/HFlip/ToTensor/Normalize (data.py:40-43, 64, 70-72)
 *      -> CutoutDefault (data.py:235-250).
 *      d_in : uint8 [batch][h][w][3] (HWC, contiguous) on the device
 *      d_out: [batch][3][out_h][out_w] of tail->out_dtype (or uint8 HWC)
 *      d_samples / d_boxes: resolved decisions; if d_samples == NULL the kernel draws them
 *      itself from `rng` (fused Philox mode).  op_base selects which FAA_MAX_FUSED_OPS-wide
 *      window of the sub-policy this launch applies (chained launches for n_op > 2).
 *      Alignment (all policy entries): d_in 4-byte aligned when w % 4 == 0; d_out 16-byte (fp32),
 *      8-byte (fp16 / bf16) or 4-byte (uint8 HWC) aligned when out_w % 4 == 0; else
 *      FAA_ERR_UNSUPPORTED. */
int faa_augment(faa_policy_t* p, const uint8_t* d_in, void* d_out, int batch, int h, int w,
                const faa_tail_t* tail, const faa_sample_t* d_samples, const faa_box_t* d_boxes,
                const faa_rng_t* rng, int op_base, void* stream);

/* fused Mixup variant: out[i] = lam*aug(in[i]) + one_minus_lam*aug(in[partner[i]]) in fp32
 * (lam and one_minus_lam are the fp32 casts of the Python floats lam and 1-lam)
 * (aug_mixup.py:13-23 with the pairing resolved by the caller; partner indexes d_in_all,
 * which may be an all-gathered or peer-mapped array of n_all images with its own
 * samples/boxes).  d_partner == NULL or lam == 1 degenerates to faa_augment. */
int faa_augment_mixup(faa_policy_t* p, const uint8_t* d_in_all, int n_all, int first, void* d_out,
                      int batch, int h, int w, const faa_tail_t* tail,
                      const faa_sample_t* d_samples_all, const faa_box_t* d_boxes_all,
                      const faa_rng_t* rng, const int32_t* d_partner, float lam, float one_minus_lam,
                      void* stream);

/* ---- overlap of consecutive calls.  The kernels of one call are chained with programmatic dependent launches and
 * overlap each other; with on != 0 the kernels of call N+1 may also start while call N (same handle, same stream,
 * disjoint buffers) is still running - worth ~15 % at 224x224 b512.  The caller promises that the INPUT batch of every
 * call was complete before the previous call on that stream was issued (e.g. device-resident data, or a producer that
 * runs one batch ahead): the first kernel of an overlapping call does not wait for the kernel right in front of it in
 * the stream.  Default: off (the first kernel of every call is an ordinary stream-ordered launch). */
int faa_policy_set_overlap(faa_policy_t* p, int on);

/* ---- several consecutive batches in one call: the loop `for data, label in loader:` of train.py:47-49 when the
 * dataset is device-resident (data.py:114-224 replaced by a DeviceDataset) - the caller knows the next n_steps
 * batches in advance, so their launches are issued back to back without returning to the interpreter (small-image
 * steps are bound by the host's launch rate otherwise).  Step k reads d_in[k] ([batch][h][w][3] uint8), writes
 * d_out[k] and draws the decisions of global samples rng->first_index + k*index_stride + i; it equals
 * faa_augment(..., rng with that first_index, ...).  Policies of at most FAA_MAX_FUSED_OPS ops. */
int faa_augment_many(faa_policy_t* p, int n_steps, const uint8_t* const* d_in, void* const* d_out,
                     int batch, int h, int w, const faa_tail_t* tail, const faa_rng_t* rng,
                     uint64_t index_stride, void* stream);

/* ---- test-time-augmentation batching: replaces the `num_policy` validation loaders of
 * eval_tta (search.py:87-90: one get_dataloaders call per replica, each drawing its own
 * sub-policies for the SAME validation batch, the losses reduced per sample at :116-125).
 * ONE launch augments d_in [batch] `replicas` times: d_out [replicas][batch][3][out_h][out_w];
 * replica r uses the decisions of global samples rng->first_index + r*batch + i, i.e. it equals
 * faa_augment called with first_index + r*batch.  Policies of at most FAA_MAX_FUSED_OPS ops. */
int faa_augment_tta(faa_policy_t* p, const uint8_t* d_in, void* d_out, int batch, int replicas,
                    int h, int w, const faa_tail_t* tail, const faa_rng_t* rng, void* stream);

/* same call with HOST buffers: pinned staging, chunked H2D / kernel / D2H pipeline inside.
 * h_out may be NULL (result stays on the device in d_out_keep, which may also be NULL). */
int faa_augment_host(faa_policy_t* p, const uint8_t* h_in, void* h_out, void* d_out_keep,
                     int batch, int h, int w, const faa_tail_t* tail, const faa_rng_t* rng,
                     void* stream);

/* ---- standalone Mixup on already-augmented device tensors: replaces mixup()
 *      (aug_mixup.py:13-23) given the resolved permutation and lambda.
 *      out[i] = data[i]*lam + data[perm[i]]*(1-lam), fp32 math, n_per_sample elements each.
 *      d_out must not overlap d_data (FAA_ERR_VALUE: a sample would be overwritten while another
 *      reads it as its partner); batch <= 65535 (FAA_ERR_UNSUPPORTED). */
int faa_mixup(const void* d_data, void* d_out, const int64_t* d_perm, int batch,
              int64_t n_per_sample, int dtype, float lam, float one_minus_lam, void* stream);

/* ---- Mixup of AUGMENTED uint8 images (the multi-GPU / large-batch route): the policy part of the
 * chain ran with a uint8 HWC output (faa_augment with tail.out_dtype = FAA_U8_HWC: policy + crop +
 * flip), possibly on another GPU; this call finishes data.py:42-43 (ToTensor, Normalize), data.py:228-250
 * (CutoutDefault: one half-open zero box [y0,y1)x[x0,x1) per SOURCE image, int16[4] each, may be NULL) and
 * aug_mixup.py:21 in one streaming pass:
 *     d_out[i] = norm(d_a[i]) * lam + norm(d_b[d_partner[i]]) * one_minus_lam      (fp32, then tail->out_dtype)
 * Same values as faa_augment_mixup on the raw images.  W % 4 == 0. */
int faa_mix_u8(faa_policy_t* p, const uint8_t* d_a, const uint8_t* d_b, const int32_t* d_partner,
               const int16_t* d_zero_box_a, const int16_t* d_zero_box_b, void* d_out, int batch, int h, int w,
               const faa_tail_t* tail, float lam, float one_minus_lam, void* stream);

/* ---- the same pass with the partner exchange INSIDE the kernel: d_partner_ptrs[i] (device array of `batch` pointers)
 * is the address of sample i's partner image - local, or in the memory of another GPU of the node mapped into this
 * process (CUDA IPC / symmetric memory; NVLink peer access enabled).  The partner's bytes travel over NVSwitch as the
 * kernel's loads: no all-to-all, no staging copy.  The caller orders it behind the partners' augmentation (a barrier
 * across the ranks) and keeps their buffers alive until it has run.  d_zero_box_b: one box PER SAMPLE (its partner's). */
int faa_enable_peer_access(int peer_device);      /* cudaDeviceEnablePeerAccess from the current device (idempotent) */
/* a device buffer that the other processes of the node can map (cudaMalloc + cudaIpcGetMemHandle; 64-byte handle),
 * the mapping of such a buffer under the current device (cudaIpcOpenMemHandle, lazy peer access), and their release */
int faa_peer_alloc(size_t bytes, void** d_ptr, unsigned char* handle64);
int faa_peer_open(const unsigned char* handle64, void** d_ptr);
int faa_peer_close(void* d_ptr);
int faa_peer_free(void* d_ptr);
int faa_mix_u8_peer(faa_policy_t* p, const uint8_t* d_a, const uint8_t* const* d_partner_ptrs,
                    const int16_t* d_zero_box_a, const int16_t* d_zero_box_b, void* d_out, int batch, int h, int w,
                    const faa_tail_t* tail, float lam, float one_minus_lam, void* stream);

/* ---- ImageNet train chain pieces (data.py:60-73), "next" row N2 --------------------------------
 * torchvision ColorJitter(brightness, contrast, saturation) (data.py:65-69) on uint8 HWC images, in place
 * allowed (d_out == d_in): per image the ops of order[] (torch.randperm(4): 0 brightness, 1 contrast,
 * 2 saturation, 3 hue = absent) with the factors alpha[] as PIL ImageEnhance blends - the arithmetic of
 * the policy ops Brightness / Contrast / Color with per-image magnitudes. */
typedef struct faa_jitter { float alpha[3]; uint8_t order[4]; } faa_jitter_t;
int faa_color_jitter(const uint8_t* d_in, uint8_t* d_out, int batch, int h, int w,
                     const faa_jitter_t* d_recs, void* stream);

/* Lighting (augmentations.py:197-215) sits between ToTensor and Normalize (data.py:70-72):
 * d_rgb [n][3] fp32 (device) = the per-image offsets eigvec . (alpha * eigval); subsequent faa_augment
 * launches over n images normalise with per-image tables ((u8/255 + rgb[c]) - mean[c]) / std[c] in torch's
 * fp32 operation order.  NULL switches it off again.  The array must stay valid until those launches ran. */
int faa_policy_set_lighting(faa_policy_t* p, const float* d_rgb, int n);

/* ---- EfficientNet crops + bicubic resize: the geometry of the ImageNet chains (data.py:61-62, 76-77, 267-345)
 * EfficientNetRandomCrop(img_size) / EfficientNetCenterCrop(img_size), then transforms.Resize((s, s), BICUBIC),
 * i.e. Pillow's Image.crop (box rounded half to even) and ImagingResample (8-bit, bicubic a = -0.5, 22-bit fixed
 * point, horizontal pass into a uint8 intermediate, then the vertical pass), bit-exact. */
typedef struct faa_crop_box { int32_t x0, y0, w, h; } faa_crop_box_t;   /* crop = rows [y0, y0+h) x columns [x0, x0+w) */

enum faa_crop_mode { FAA_CROP_RANDOM = 0, FAA_CROP_CENTER = 1 };

typedef struct faa_crop_cfg {
    int32_t   mode;                   /* enum faa_crop_mode                                            */
    int32_t   img_size;               /* EfficientNet*Crop(imgsize): the center crop is s/(s+32) of the short side */
    double    min_covered;            /* EfficientNetRandomCrop(min_covered=0.1,                          */
    double    aspect_lo, aspect_hi;   /*     aspect_ratio_range=(3/4, 4/3),                               */
    double    area_lo, area_hi;       /*     area_range=(0.08, 1.0),                                      */
    int32_t   max_attempts;           /*     max_attempts=10)                                             */
    int32_t   reserved;
    faa_rng_t rng;                    /* seed / first_index of the device crop sampler (other fields unused) */
} faa_crop_cfg_t;

/* host helper: the box EfficientNetCenterCrop(img_size) cuts from an h x w image */
int faa_center_crop_box(int h, int w, int img_size, faa_crop_box_t* out);

/* d_in : uint8 [batch][h][w][3] (device).  d_out: [batch][tail->out_h][tail->out_w][3] uint8 when tail->out_dtype is
 * FAA_U8_HWC (the train chain continues with faa_color_jitter), else [batch][3][out_h][out_w] with ToTensor + Normalize
 * (tail->mean / std) fused in: the same values faa_augment writes for the same uint8 image.  d_boxes: one box per image
 * (device memory; checked against the image on the host, which waits for the stream), or NULL: the kernel draws
 * them itself (cfg->mode; random boxes from Philox keyed by (cfg->rng.seed, cfg->rng.first_index + i): the reference's
 * distributions, not its stream).  An ordinary stream-ordered launch.  tail->use_zero_box and crop_pad are ignored. */
int faa_crop_resize(const uint8_t* d_in, void* d_out, int batch, int h, int w, const faa_tail_t* tail,
                    const faa_crop_box_t* d_boxes, const faa_crop_cfg_t* cfg, void* stream);

/* ---- the same crop + resize over a batch of differently sized images (data.py:61-62, 76-77, 267-345 run on one
 * PIL image at a time, so each image is cropped at its own size): image i is h_images[i].h x h_images[i].w uint8 HWC
 * at h_images[i].data (device memory, rows packed, any byte offset).  h_images is the host copy, used to validate and
 * plan without waiting for the device; d_images is a device copy with the same contents, which the kernel reads.
 * Boxes are drawn (or checked) against each image's own size, with the same Philox keys as faa_crop_resize, so a
 * batch of equal sizes gives the same bytes as faa_crop_resize.  One launch. */
typedef struct faa_image { const uint8_t* data; int32_t h, w; } faa_image_t;             /* 16 bytes */
int faa_crop_resize_ragged(const faa_image_t* h_images, const faa_image_t* d_images, int batch, void* d_out,
                           const faa_tail_t* tail, const faa_crop_box_t* d_boxes, const faa_crop_cfg_t* cfg,
                           void* stream);

/* ---- the policy over a batch of differently sized images (data.py:253-264 Augmentation, called on one PIL image of
 * any size at a time): image i (h_in[i].h x h_in[i].w uint8 HWC at h_in[i].data, device memory, rows packed, any byte
 * offset) is augmented at its own size into h_out[i] (same size, uint8 HWC).  h_in / h_out are host copies, used to
 * validate and plan without waiting for the device; d_in / d_out are device copies with the same contents, which the
 * kernels read.  Output i equals faa_augment on image i alone with a uint8 HWC tail of its size:
 *   d_samples == NULL: the decisions of global sample rng->first_index + i drawn for an h_i x w_i image (the records of
 *                      faa_sample_philox_at at position i); the rng has no crop_pad, hflip or zero_box_len;
 *   else             : d_samples[i] and d_boxes[i][n_op], drawn for image i's own size.
 * op_base selects the FAA_MAX_FUSED_OPS-wide window as in faa_augment; every window writes uint8.  One resolve launch and
 * one pixel launch per cluster size present (at most four), plus one copy launch when some image with w % 4 == 0 starts
 * off a 4-byte boundary (the library re-aligns those inputs).  Output alignment: h_out[i].data 4-byte aligned when
 * w % 4 == 0, else FAA_ERR_UNSUPPORTED.  batch <= 65535. */
int faa_augment_ragged(faa_policy_t* p, const faa_image_t* h_in, const faa_image_t* d_in, int batch,
                       const faa_image_t* h_out, const faa_image_t* d_out, const faa_sample_t* d_samples,
                       const faa_box_t* d_boxes, const faa_rng_t* rng, int op_base, void* stream);

/* ---- baseline JPEG decode: replaces torchvision's default_loader (imagenet.py:80, `Image.open(f).convert('RGB')`, Pillow
 * on libjpeg-turbo with its default islow IDCT, fancy upsampling and fixed-point YCbCr->RGB) for a batch of files, bit-exact.
 * Supported: SOF0 / SOF1 Huffman, 8-bit, one interleaved scan, 1 component (written R = G = B) or 3 in YCbCr (JFIF, or no
 * Adobe transform 0) with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1, any restart interval, up to FAA_MAX_DIM a side.
 * Headers are parsed once on the host (when a dataset is built); the tables they use go into a caller-owned pool of
 * faa_jpeg_table_t (deduplicated by the caller), which the headers index. */
typedef struct faa_jpeg_header {
    int64_t offset;           /* the file is bytes [offset, offset + len) of the decode call's d_src (parse: 0)       */
    int64_t len;
    int64_t scan_off;         /* entropy-coded data: bytes [scan_off, scan_off + scan_len) of the file               */
    int64_t scan_len;
    int32_t h, w;             /* image size                                                                          */
    int32_t ncomp;            /* 1 (grayscale) or 3 (YCbCr)                                                          */
    int32_t hs, vs;           /* luma sampling factors (chroma 1x1); 1, 1 for grayscale                              */
    int32_t restart;          /* restart interval in MCUs, 0 = none                                                  */
    int32_t mcu_x, mcu_y;     /* MCUs per row / per column                                                           */
    int32_t table_at[9];      /* file offsets of the tables of components 0..2: quantisation [0..2], DC Huffman
                                 [3..5], AC Huffman [6..8]; -1 for absent components; -2 - k for a Huffman table
                                 no DHT defines, which is standard table k of ITU T.81 K.3 (DC 0, DC 1, AC 0, AC 1)  */
    int32_t pool[9];          /* the same tables as indices into the caller's faa_jpeg_table_t pool (parse: -1)      */
    int32_t qprec;            /* bit c: component c's quantisation table has 16-bit entries                          */
    int32_t reserved;
} faa_jpeg_header_t;          /* 144 bytes */

typedef struct faa_jpeg_table {
    uint16_t q[64];           /* quantisation table, natural (row-major) order; zero in a Huffman entry             */
    uint8_t  bits[16];        /* Huffman table: number of codes of each length 1..16; zero in a quantisation entry  */
    uint8_t  vals[256];       /*                symbols in code order                                                */
} faa_jpeg_table_t;           /* 400 bytes */

/* per-image status bits of faa_jpeg_decode (0 = the scan decoded completely) */
enum faa_jpeg_status {
    FAA_JPEG_TRUNCATED = 1,    /* the scan ended, or met a marker, before its last MCU; the rest of the image is zeros */
    FAA_JPEG_BAD_CODE = 2,     /* a bit pattern that is no Huffman code                                              */
    FAA_JPEG_BAD_COEF = 4,     /* a run past coefficient 63                                                          */
    FAA_JPEG_BAD_RESTART = 8   /* not one restart marker per interval boundary                                       */
};

/* host only: parse one file's markers.  FAA_OK, FAA_ERR_UNSUPPORTED (progressive, arithmetic, lossless, 12-bit, Adobe
 * RGB / CMYK / YCCK, other sampling, multi-scan; reason in faa_last_error()) or FAA_ERR_VALUE (malformed header). */
int faa_jpeg_parse(const uint8_t* bytes, size_t len, faa_jpeg_header_t* out);
/* host only: the 9 tables a parsed header refers to (table_at), in pool form; slots of absent components are zeroed */
int faa_jpeg_tables(const uint8_t* bytes, size_t len, const faa_jpeg_header_t* hdr, faa_jpeg_table_t out[9]);

/* a decoder handle owns the scratch of its calls (coefficients, restart-segment starts, per-call table), grown on demand
 * in stream order; it is bound to the device current at its first decode, like a policy handle */
typedef struct faa_jpeg_decoder faa_jpeg_decoder_t;
int faa_jpeg_decoder_create(faa_jpeg_decoder_t** out);
int faa_jpeg_decoder_destroy(faa_jpeg_decoder_t* dec);

/* ---- scan index: lets a file without restart markers be decoded by many threads.  One serial pass (faa_jpeg_index_build)
 * records the decoder's state at up to 127 MCU boundaries; every later decode of the file starts one thread at each of
 * them.  Placement: a scan of scan_len bytes with no restart interval is cut into P = min(128, scan_len / 1024) parts
 * of about equal bytes; point k (1 <= k < P) is the first MCU boundary whose start byte is >= k * scan_len / P, and
 * points that coincide are dropped.  Below 2 parts (scans under 2 KiB), or with a restart interval, a file has no
 * points.  The file itself is not changed. */
typedef struct faa_jpeg_sync {
    int32_t mcu;              /* the next MCU to decode                                                              */
    int32_t byte;             /* scan offset of the data byte that holds its first bit (a stuffed 0xFF 0x00 is one data
                                 byte, at the 0xFF's offset)                                                         */
    int16_t bit;              /* bits of that byte already consumed, 0..7                                            */
    int16_t pred[3];          /* DC predictors of the components (0 for absent ones)                                 */
} faa_jpeg_sync_t;            /* 16 bytes */

/* host only: the most points faa_jpeg_index_build records for a file with this header (P - 1, or 0) */
int faa_jpeg_index_capacity(const faa_jpeg_header_t* hdr);

/* Records the scan index of `batch` files (inputs as faa_jpeg_decode).  h_first / d_first: host and device copies of
 * int64 [batch + 1] offsets into d_points, planned by the caller (image i may get first[i + 1] - first[i] points, at most
 * faa_jpeg_index_capacity of its header); d_count: [batch] int32, the points written at d_points + first[i]; d_status:
 * [batch] int32, the status of that serial decode (a file whose decode has a status gets no points; 0 for files that
 * get none by the placement rule).  FAA_ERR_VALUE for offsets that decrease or are negative.  One launch, no host wait. */
int faa_jpeg_index_build(const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                         const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                         const int64_t* h_first, const int64_t* d_first, faa_jpeg_sync_t* d_points, int32_t* d_count,
                         int32_t* d_status, void* stream);

/* Finds the scan index of `batch` files in parallel, without a serial decode (inputs, offsets and points as
 * faa_jpeg_index_build, no status).  One CTA per file: thread k parses from a little before part k's threshold until its
 * parse meets an MCU boundary (Huffman streams self-synchronise), then decodes from there to the next part's threshold,
 * and each such link is checked against the next part's start; a few rounds repair the links that disagree.  d_count[i]
 * is the number of verified points: always the first d_count[i] of faa_jpeg_index_build's points for a file whose serial
 * decode is clean, and all of them when the chain converged (DESIGN §4.8 measures how often).  A file the placement rule
 * gives no points gets 0.  FAA_ERR_VALUE for offsets that decrease or are negative and for progressive headers.  One
 * launch, no host wait. */
int faa_jpeg_index_find(const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                        const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                        const int64_t* h_first, const int64_t* d_first, faa_jpeg_sync_t* d_points, int32_t* d_count,
                        void* stream);

/* decodes `batch` baseline files into uint8 HWC images.  h_headers / d_headers: host and device copies of the same
 * headers (the host copy validates and plans without waiting for the device); d_tables: the pool of n_tables entries;
 * d_src: the device bytes the headers' offsets point into; h_out / d_out: host and device copies of the destinations,
 * each of its header's size (rows packed, any byte offset); d_status: [batch] int32 (device), enum faa_jpeg_status bits.
 * A corrupt scan never faults: its image gets a status and defined pixels.  Two launches (entropy decode, reconstruct),
 * one cudaMemcpyAsync of the per-call table, no host wait.
 *
 * Two optional groups of arguments, each all null or given; a group that is given is validated on the host as
 * faa_jpeg_index_build's offsets and points are (FAA_ERR_VALUE for a missing array or bad offsets):
 *   - scan index in (d_points, h_first, d_first): image i's points are d_points[first[i], first[i + 1]), host and device
 *     copies of int64 [batch + 1] offsets; d_points may be null when the offsets give no image a point.  The points are
 *     checked on the device before use, and every segment's end state against the next point; a file whose index is
 *     invalid, stale or from another file is decoded serially.  Points of files with a restart interval are ignored.
 *   - recording out (h_cap_first, d_cap_first, d_points_out, d_count): the decode also records the scan index of every
 *     file it decodes serially as a whole (a file without points, or whose points failed their checks) into d_points_out,
 *     laid out as faa_jpeg_index_build's: image i may get cap_first[i + 1] - cap_first[i] points, at most
 *     faa_jpeg_index_capacity of its header; d_points_out may be null when every capacity is 0.  d_count: [batch] int32,
 *     the points written at d_points_out + cap_first[i]; 0 for a file with a restart interval, a scan the placement rule
 *     gives no points, a non-zero status, or points that were used as they stood.  So count[i] > 0 means these are
 *     file i's points now.
 * find != 0 needs the recording group (FAA_ERR_VALUE without it): the files without input points first get their scan
 * index found in parallel (faa_jpeg_index_find, into d_points_out), so that a restart-free file decodes on many threads
 * without a saved index; files with input points keep them.  count[i] > 0 still means these are file i's points now:
 * the found index when its chain converged and was used, or the serial decode's recording when the file's points (given
 * or found) could not be used.  A found prefix that did not converge is used for the decode and gets count 0.  Three
 * launches (find, entropy decode, reconstruct), no host wait.
 *
 * Whatever the index holds, given or found, pixels and status equal those of the decode without one. */
int faa_jpeg_decode(faa_jpeg_decoder_t* dec, const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                    const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                    const faa_image_t* h_out, const faa_image_t* d_out, int32_t* d_status,
                    const faa_jpeg_sync_t* d_points, const int64_t* h_first, const int64_t* d_first,
                    const int64_t* h_cap_first, const int64_t* d_cap_first, faa_jpeg_sync_t* d_points_out,
                    int32_t* d_count, int find, void* stream);

/* ---- progressive JPEG decode (SOF2 Huffman), for callers that opt in: the files faa_jpeg_parse takes, coded
 * progressively, bit-exact with Pillow as above.  The parse accepts a file only when every coefficient of every component
 * ends at bit 0 (libjpeg smooths the blocks of an incomplete progression, which is not modelled), with at most
 * FAA_JPEG_MAX_SCANS scans; multi-scan sequential, arithmetic coding and the rest stay refused.  Its header has
 * reserved = FAA_JPEG_PROGRESSIVE, restart = 0 and no scan_off / scan_len, and its quantisation tables are those in force at
 * each component's first scan.  faa_jpeg_decode, faa_jpeg_index_build and faa_jpeg_index_find refuse such a header
 * with FAA_ERR_VALUE, and faa_jpeg_index_capacity gives it 0: progressive files have no scan index. */
#define FAA_JPEG_PROGRESSIVE 1
#define FAA_JPEG_MAX_SCANS 64
typedef struct faa_jpeg_scan {
    int64_t off;              /* entropy-coded data: bytes [off, off + len) of the file                              */
    int64_t len;
    int32_t restart;          /* restart interval in force at its SOS, in units (MCUs, or blocks of a one-component scan) */
    int32_t ns;               /* components in the scan: comp[0, ns), frame indices in frame order (-1 past ns)      */
    int32_t comp[3];
    int32_t ss, se, ah, al;   /* spectral band [ss, se] and successive approximation bits (ITU T.81 G.1.1.1)          */
    int32_t wave;             /* 1 + the largest wave of an earlier scan that shares a component and a coefficient
                                 (DC counts as coefficient 0): the scans of one wave are decoded concurrently         */
    int32_t dc_at[3];         /* file offsets of the DC tables of comp[k] (DC first scans) and of the AC table (ac_at[0],
                                 AC scans) as defined at its SOS; -2 - k for standard table k; -1 when unused          */
    int32_t ac_at[3];
    int32_t pool[6];          /* the same tables as pool indices: DC of comp[k] at k, AC at 3; -1 when unused        */
    int32_t reserved[2];
} faa_jpeg_scan_t;            /* 112 bytes */

/* host only: parse a progressive file into its header and scans[0, *n_scans) (room for max_scans).  FAA_OK,
 * FAA_ERR_UNSUPPORTED (not progressive, an incomplete progression, more scans than max_scans or FAA_JPEG_MAX_SCANS, or
 * what faa_jpeg_parse refuses; reason in faa_last_error()) or FAA_ERR_VALUE (malformed header or progression). */
int faa_jpeg_parse_progressive(const uint8_t* bytes, size_t len, faa_jpeg_header_t* out, faa_jpeg_scan_t* scans,
                               int max_scans, int* n_scans);
/* host only: the tables of a progressive file in pool form: out[c] (c < 3) the quantisation table of component c, and
 * out[3 + 6 s + k] the Huffman tables of scan s (slot k as in faa_jpeg_scan_t::pool); unused slots zeroed.  out has
 * 3 + 6 n_scans entries. */
int faa_jpeg_scan_tables(const uint8_t* bytes, size_t len, const faa_jpeg_header_t* hdr, const faa_jpeg_scan_t* scans,
                         int n_scans, faa_jpeg_table_t* out);
/* decodes `batch` progressive files (inputs as faa_jpeg_decode; the headers' pool[0, ncomp) index the quantisation
 * tables).  h_scans / d_scans: host and device copies of the scans, whose pool slots index d_tables; h_scan_first /
 * d_scan_first: int64 [batch + 1] offsets, image i's scans being scans[first[i], first[i + 1]) (1 to FAA_JPEG_MAX_SCANS
 * of them).  Everything, the waves included, is validated on the host before any device work.  d_status as
 * faa_jpeg_decode's (a segment that fails stops there; the image still gets defined pixels).  Two launches (progressive
 * entropy decode, the reconstruct kernel of faa_jpeg_decode), no host wait; the handle's scratch is shared with the
 * other decode calls. */
int faa_jpeg_decode_progressive(faa_jpeg_decoder_t* dec, const faa_jpeg_header_t* h_headers,
                                const faa_jpeg_header_t* d_headers, const faa_jpeg_table_t* d_tables, int n_tables,
                                const uint8_t* d_src, int batch, const faa_image_t* h_out, const faa_image_t* d_out,
                                int32_t* d_status, const faa_jpeg_scan_t* h_scans, const faa_jpeg_scan_t* d_scans,
                                const int64_t* h_scan_first, const int64_t* d_scan_first, void* stream);

/* number of kernels this library has launched since load (bench bookkeeping) */
uint64_t faa_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FAA_B200_H */
