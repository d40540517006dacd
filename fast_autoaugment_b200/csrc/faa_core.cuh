// faa_core.cuh - per-pixel arithmetic of the augmentation hot path, shared by the
// sm_90a kernels (faa_kernels.cu) and by the host-side emulation used in the CPU
// tests (tests/emu).  Every function states the reference call it reproduces
// (file:line relative to kakaobrain/fast-autoaugment @ 2424224) and the Pillow /
// torchvision arithmetic behind that call (SURVEY.md 8a).
//
// Design: the raw uint8 HWC image is READ-ONLY.  A sub-policy is evaluated lazily
// from the output pixel back to the raw image:
//     value<2>(x,y) = op2( value<1>(.) ),  value<1>(x,y) = op1( value<0>(.) ),  value<0> = raw
// Geometric ops remap the coordinate, per-channel ops go through a 3x256 byte LUT built
// once per image (static LUTs, AutoContrast/Equalize from the histogram, Brightness /
// Contrast blends), Color and Cutout are evaluated in registers, Sharpness evaluates its
// 3x3 neighbourhood one level down.  The chain needs no second image buffer in global memory
// and no barrier between ops; the kernels only materialise an intermediate image (in shared
// memory) where lazy evaluation would repeat work (Sharpness or a statistics op behind another
// op), and the ops that need whole-image statistics cost one extra pass over the row band.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#if defined(__CUDACC__)
#define FAA_HD __host__ __device__ __forceinline__
#else
#define FAA_HD inline
#endif

namespace faa {

// ------------------------------------------------------------------ records --
enum Kind : int32_t {
    K_NONE = 0,          // identity (gate not passed, Rotate by 0, Cutout with v<=0 ...)
    K_AFFINE = 1,        // a[0..5]: Pillow affine_fixed 16.16 coefficients
    K_SHIFT = 2,         // a[0]=dx, a[1]=dy, a[2]=bx, a[3]=by : out[y][x] = in[y+dy+(y>=by)][x+dx+(x>=bx)]
                         //   (bx/by: index from which Pillow's accumulated float offset has rounded
                         //    up to the next integer - at most one such break per axis)
    K_LUT = 3,           // a[0]=solarize threshold (0..256), a[1]=AND mask : static per-channel LUT
    K_AUTOCONTRAST = 4,  // histogram -> fp64 LUT
    K_EQUALIZE = 5,      // histogram -> integer prefix LUT
    K_BRIGHTNESS = 6,    // a[0]=fp32 bits of alpha, a[1]=clip flag ; blend with 0
    K_COLOR = 7,         //   "   blend with luma
    K_CONTRAST = 8,      //   "   blend with int(mean luma + .5) of the whole image
    K_SHARPNESS = 9,     //   "   blend with 3x3 SMOOTH
    K_CUTOUT = 10        // a[0..1]=fp64 bits of the side length in pixels; box comes per sample
};

struct alignas(16) OpRec {  // 32 bytes, one per (sub-policy, op slot, sign variant)
    int32_t kind;
    int32_t a[6];
    int32_t draw;        // enum faa_draw of the *named* op (kept even when kind==K_NONE)
};

struct Box { int16_t x0, y0, x1, y1; };       // inclusive, unclipped (== faa_box_t)

struct Sample {                               // == faa_sample_t
    uint16_t sub; uint8_t gate; uint8_t sign;
    int8_t crop_dy; int8_t crop_dx; uint8_t flip; uint8_t reserved;
    int16_t zero_box[4];
};

constexpr uint32_t kCutoutRGB = 125u | (123u << 8) | (114u << 16);   // augmentations.py:140

// kind classes
FAA_HD bool kind_uses_lut(int k)   { return k == K_LUT || k == K_AUTOCONTRAST || k == K_EQUALIZE ||
                                            k == K_BRIGHTNESS || k == K_CONTRAST; }
FAA_HD bool kind_needs_hist(int k) { return k == K_AUTOCONTRAST || k == K_EQUALIZE; }
FAA_HD bool kind_needs_mean(int k) { return k == K_CONTRAST; }
FAA_HD bool kind_is_pointwise(int k) { return k == K_NONE || kind_uses_lut(k) || k == K_COLOR || k == K_CUTOUT; }

// ------------------------------------------------------------ float helpers --
// Non-contracted fp32 / fp64 steps (Pillow is compiled for x86-64 SSE2: no FMA).
FAA_HD float f_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b; return r;
#endif
}
FAA_HD float f_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b; return r;
#endif
}
FAA_HD double d_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double r = a * b; return r;
#endif
}
FAA_HD double d_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    volatile double r = a + b; return r;
#endif
}
FAA_HD float bits_to_float(int32_t b) {
#if defined(__CUDA_ARCH__)
    return __int_as_float(b);
#else
    union { int32_t i; float f; } u; u.i = b; return u.f;
#endif
}
FAA_HD uint32_t umulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

// Pillow Image.blend (Blend.c), one byte: fp32, truncation; clip only when alpha is
// outside [0,1].  Serves ImageEnhance.*.enhance -> augmentations.py:99,104,109,114.
FAA_HD uint32_t blend_u8(uint32_t deg, uint32_t px, float alpha, bool clip) {
    float d = (float)(int)deg;
    float t = f_add(d, f_mul(alpha, (float)((int)px - (int)deg)));
    // Saturating truncation serves both cases: for alpha in [0,1] (no clip in Pillow) t already lies
    // between deg and px - the product is no larger than px-deg and both ends are representable.
    (void)clip;
#if defined(__CUDA_ARCH__)
    return min(__float2uint_rz(t), 255u);
#else
    if (t <= 0.0f) return 0u;
    if (t >= 255.0f) return 255u;
    return (uint32_t)(int)t;
#endif
}

// Pillow RGB->L (Convert.c rgb2l): ImageEnhance.Color / Contrast degenerate images.
FAA_HD uint32_t luma_of(uint32_t p) {
    return (19595u * (p & 255u) + 38470u * ((p >> 8) & 255u) + 7471u * ((p >> 16) & 255u) + 0x8000u) >> 16;
}

FAA_HD uint32_t apply_lut(const uint8_t* lut, uint32_t p) {
    return (uint32_t)lut[p & 255u] | ((uint32_t)lut[256 + ((p >> 8) & 255u)] << 8) |
           ((uint32_t)lut[512 + ((p >> 16) & 255u)] << 16);
}

FAA_HD uint32_t color_px(uint32_t p, float alpha, bool clip) {      // augmentations.py:102-104
    uint32_t l = luma_of(p);
    return blend_u8(l, p & 255u, alpha, clip) | (blend_u8(l, (p >> 8) & 255u, alpha, clip) << 8) |
           (blend_u8(l, (p >> 16) & 255u, alpha, clip) << 16);
}

// ------------------------------------------------------------ image context --
struct Ctx {
    const uint8_t* raw;      // this image, uint8 HWC (global memory)
    const uint8_t* sraw;     // TMA-staged copy of bytes [s_lo, s_lo + s_len) of the image (shared memory)
    uint32_t s_lo, s_len2;   // s_len2 = staged length - 2 (0 when nothing is staged)
    uint32_t rcp_w, rcp_wq;  // fastdiv reciprocals of W and W/4 (device loops)
    int H, W;
    OpRec op[2];             // the two fused op slots (K_NONE when not applied)
    Box box[2];              // clipped inclusive Cutout boxes (valid when op[j].kind==K_CUTOUT)
    const uint8_t* lut[2];   // 3x256 per slot (valid when kind_uses_lut)
};

FAA_HD uint32_t load_raw(const Ctx& c, int x, int y) {
    const uint32_t off = (uint32_t)(y * c.W + x) * 3u;            // H, W <= 8192: fits 32 bits
    const uint32_t rel = off - c.s_lo;
    if (rel < c.s_len2) {                                         // inside the staged row band
        const uint8_t* p = c.sraw + rel;
        return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
    }
    const uint8_t* p = c.raw + off;
#if defined(__CUDA_ARCH__)
    return (uint32_t)__ldg(p) | ((uint32_t)__ldg(p + 1) << 8) | ((uint32_t)__ldg(p + 2) << 16);
#else
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
#endif
}

// pointwise part of op slot j applied to an already fetched pixel at frame coords (x,y)
FAA_HD uint32_t apply_pointwise(const Ctx& c, int j, uint32_t p, int x, int y) {
    const OpRec& o = c.op[j];
    switch (o.kind) {
    case K_LUT: case K_AUTOCONTRAST: case K_EQUALIZE: case K_BRIGHTNESS: case K_CONTRAST:
        return apply_lut(c.lut[j], p);
    case K_COLOR:
        return color_px(p, bits_to_float(o.a[0]), o.a[1] != 0);
    case K_CUTOUT: {                                          // augmentations.py:142-143
        const Box& b = c.box[j];
        return (x >= b.x0 && x <= b.x1 && y >= b.y0 && y <= b.y1) ? kCutoutRGB : p;
    }
    default:
        return p;
    }
}

template <int L> struct Level;

template <> struct Level<0> {
    static FAA_HD uint32_t at(const Ctx& c, int x, int y) { return load_raw(c, x, y); }
};

// value of the image after the first L op slots, at (x, y) of that image.
// One call site per level for the centre tap (keeps the inlined code small).
template <int L> struct Level {
    static FAA_HD uint32_t at(const Ctx& c, int x, int y) {
        const OpRec& o = c.op[L - 1];
        const int k = o.kind;
        if (k == K_AFFINE) {          // Pillow affine_fixed: augmentations.py:17,24,61 (NEAREST, zero fill)
            int xin = (o.a[2] + o.a[0] * x + o.a[1] * y) >> 16;
            int yin = (o.a[5] + o.a[3] * x + o.a[4] * y) >> 16;
            if ((unsigned)xin >= (unsigned)c.W || (unsigned)yin >= (unsigned)c.H) return 0u;
            x = xin; y = yin;
        } else if (k == K_SHIFT) {    // Pillow ImagingScaleAffine, unit scale: augmentations.py:32,40,47,54
            int xin = x + o.a[0] + (x >= o.a[2]), yin = y + o.a[1] + (y >= o.a[3]);
            if ((unsigned)xin >= (unsigned)c.W || (unsigned)yin >= (unsigned)c.H) return 0u;
            x = xin; y = yin;
        }
        uint32_t p = Level<L - 1>::at(c, x, y);
        if (k <= K_SHIFT) return p;                                  // NONE / AFFINE / SHIFT
        if (k != K_SHARPNESS) return apply_pointwise(c, L - 1, p, x, y);
        // augmentations.py:112-114: blend(SMOOTH(img), img, v); 1-px border copied
        if (x == 0 || y == 0 || x == c.W - 1 || y == c.H - 1) return p;
        uint32_t s0 = 4u * (p & 255u), s1 = 4u * ((p >> 8) & 255u), s2 = 4u * ((p >> 16) & 255u);
        for (int t = 0; t < 9; ++t) {
            int dx = t % 3 - 1, dy = t / 3 - 1;
            uint32_t q = (t == 4) ? p : Level<L - 1>::at(c, x + dx, y + dy);
            s0 += q & 255u; s1 += (q >> 8) & 255u; s2 += (q >> 16) & 255u;
        }
        // [1 1 1;1 5 1;1 1 1]/13 rounded half up == (2S+13)/26
        s0 = (2u * s0 + 13u) / 26u; s1 = (2u * s1 + 13u) / 26u; s2 = (2u * s2 + 13u) / 26u;
        float al = bits_to_float(o.a[0]); bool clip = o.a[1] != 0;
        return blend_u8(s0, p & 255u, al, clip) | (blend_u8(s1, (p >> 8) & 255u, al, clip) << 8) |
               (blend_u8(s2, (p >> 16) & 255u, al, clip) << 16);
    }
};

// ------------------------------------------------------------------- LUTs --
// static / blend LUT entries: one (channel-independent) byte function
FAA_HD uint32_t lut_entry_static(const OpRec& o, uint32_t i, uint32_t mean) {
    switch (o.kind) {
    case K_LUT: {            // solarize (augmentations.py:80-82), posterize (:85-94), invert (:68-69)
        uint32_t v = ((int)i < o.a[0]) ? i : 255u - i;
        return v & (uint32_t)o.a[1];
    }
    case K_BRIGHTNESS:       // augmentations.py:107-109
        return blend_u8(0u, i, bits_to_float(o.a[0]), o.a[1] != 0);
    case K_CONTRAST:         // augmentations.py:97-99
        return blend_u8(mean, i, bits_to_float(o.a[0]), o.a[1] != 0);
    default:
        return i;
    }
}

// ImageEnhance.Contrast: int(ImageStat.mean + 0.5) == (2*sum + N) / (2*N)
FAA_HD uint32_t contrast_mean(uint64_t sum_l, uint32_t n) {
    return (uint32_t)((2ull * sum_l + n) / (2ull * n));
}

// Per-channel partial summary of 8 histogram bins [8*lane, 8*lane+8): phase A of the
// two-phase (no shuffle, host-emulatable) histogram LUT build.
struct HistPart { uint32_t sum; int16_t lo; int16_t hi; uint32_t nnz; };

FAA_HD HistPart hist_part(const uint32_t* h256, int lane) {
    HistPart p; p.sum = 0; p.lo = 256; p.hi = -1; p.nnz = 0;
    for (int j = 0; j < 8; ++j) {
        int i = lane * 8 + j;
        uint32_t v = h256[i];
        p.sum += v;
        if (v) { if (i < p.lo) p.lo = (int16_t)i; p.hi = (int16_t)i; ++p.nnz; }
    }
    return p;
}

// phase B: lane writes its 8 LUT entries of one channel.
//  AutoContrast: PIL ImageOps.autocontrast(cutoff=0)  (augmentations.py:64-65)
//  Equalize    : PIL ImageOps.equalize                (augmentations.py:72-73)
FAA_HD void hist_lut_lane(int kind, const uint32_t* h256, const HistPart* parts32, int lane,
                          uint32_t n_pixels, uint8_t* lut256) {
    int lo = 256, hi = -1; uint32_t nnz = 0, before = 0;
    for (int k = 0; k < 32; ++k) {
        const HistPart& q = parts32[k];
        if (q.lo < lo) lo = q.lo;
        if (q.hi > hi) hi = q.hi;
        nnz += q.nnz;
        if (k < lane) before += q.sum;
    }
    if (kind == K_AUTOCONTRAST) {
        if (hi <= lo) { for (int j = 0; j < 8; ++j) lut256[lane * 8 + j] = (uint8_t)(lane * 8 + j); return; }
        double scale = 255.0 / (double)(hi - lo);
        double offset = d_mul(-(double)lo, scale);
        for (int j = 0; j < 8; ++j) {
            int ix = lane * 8 + j;
            int t = (int)d_add(d_mul((double)ix, scale), offset);       // Python int(): toward zero
            lut256[ix] = (uint8_t)(t < 0 ? 0 : t > 255 ? 255 : t);
        }
    } else {   // K_EQUALIZE
        uint32_t step = 0;
        if (nnz > 1) step = (n_pixels - h256[hi]) / 255u;
        if (step == 0) { for (int j = 0; j < 8; ++j) lut256[lane * 8 + j] = (uint8_t)(lane * 8 + j); return; }
        uint32_t n = step / 2u + before;
        for (int j = 0; j < 8; ++j) {
            int ix = lane * 8 + j;
            uint32_t v = n / step;
            lut256[ix] = (uint8_t)(v > 255u ? 255u : v);                // Image.point clips
            n += h256[ix];
        }
    }
}

// ------------------------------------------------------------------- tail --
// RandomCrop(+pad) / HFlip / CutoutDefault index logic of data.py:40-41,235-250 for one
// output pixel.  Returns false when the output is the zero box (caller writes 0), and sets
// `inside` false when the source falls in the zero padding (pixel value 0,0,0).
FAA_HD bool tail_source(const Sample& s, bool use_zero_box, int out_w, int H, int W,
                        int ox, int oy, int& ax, int& ay, bool& inside) {
    if (use_zero_box && oy >= s.zero_box[0] && oy < s.zero_box[1] && ox >= s.zero_box[2] && ox < s.zero_box[3])
        return false;
    int cx = s.flip ? (out_w - 1 - ox) : ox;
    ax = cx + s.crop_dx;
    ay = oy + s.crop_dy;
    inside = (unsigned)ax < (unsigned)W && (unsigned)ay < (unsigned)H;
    return true;
}

// ----------------------------------------------------------------- Philox --
// Philox4x32-10 (Salmon et al. 2011) - the device-side sampler's generator.
struct U4 { uint32_t x, y, z, w; };

FAA_HD U4 philox4x32_10(U4 ctr, uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = umulhi32(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = umulhi32(M1, ctr.z), lo1 = M1 * ctr.z;
        U4 n; n.x = hi1 ^ ctr.y ^ k0; n.y = lo1; n.z = hi0 ^ ctr.w ^ k1; n.w = lo0;
        ctr = n; k0 += W0; k1 += W1;
    }
    return ctr;
}

// CutoutAbs rectangle from two uniforms (augmentations.py:130-137; numpy's legacy
// uniform(low=w, high=1.0) = w + (1.0 - w) * u).  v_px is the side in pixels.
FAA_HD Box cutout_box(int W, int H, double v_px, double ux, double uy) {
    double cx = d_add((double)W, d_mul(1.0 - (double)W, ux));
    double cy = d_add((double)H, d_mul(1.0 - (double)H, uy));
    double half = v_px / 2.0;
    double l = d_add(cx, -half), t = d_add(cy, -half);
    int x0 = (int)(l > 0.0 ? l : 0.0);
    int y0 = (int)(t > 0.0 ? t : 0.0);
    double r = d_add((double)x0, v_px), b = d_add((double)y0, v_px);
    if (r > (double)W) r = (double)W;
    if (b > (double)H) b = (double)H;
    Box o; o.x0 = (int16_t)x0; o.y0 = (int16_t)y0; o.x1 = (int16_t)(int)r; o.y1 = (int16_t)(int)b;
    return o;
}

struct RngCfg { uint64_t seed; uint64_t first_index; int32_t crop_pad; int32_t hflip; int32_t zero_box_len; int32_t reserved; };

// Device-side sampler: one sample's decisions from counter-based draws.  Same
// distributions as the reference's draws (data.py:259-261, augmentations.py mirror /
// Cutout draws, torchvision RandomCrop/HFlip, data.py:239-240), different stream.
// `ops` = compiled table [n_sub][n_op][2], `probs` = [n_sub][n_op].
FAA_HD void philox_sample(const RngCfg& r, uint64_t index, const OpRec* ops, const double* probs,
                          int n_sub, int n_op, int H, int W, int out_h, int out_w,
                          Sample& s, Box* boxes /* n_op */) {
    uint32_t k0 = (uint32_t)r.seed, k1 = (uint32_t)(r.seed >> 32);
    U4 c; c.x = (uint32_t)index; c.y = (uint32_t)(index >> 32); c.z = 0; c.w = 0;
    U4 b0 = philox4x32_10(c, k0, k1);
    s.sub = (uint16_t)umulhi32(b0.x, (uint32_t)n_sub);
    s.flip = (uint8_t)(r.hflip ? (b0.y >> 31) : 0u);                     // torch.rand(1) < 0.5
    // torchvision RandomCrop.get_params: top in [0, H + 2p - out_h], left in [0, W + 2p - out_w] (data.py:40);
    // offsets are stored relative to the unpadded image.  (The host rejects ranges that do not fit int8.)
    const bool do_crop = r.crop_pad > 0 || out_h != H || out_w != W;
    const int span_y = H + 2 * r.crop_pad - out_h + 1, span_x = W + 2 * r.crop_pad - out_w + 1;
    s.crop_dy = (int8_t)(do_crop && span_y > 1 ? (int)umulhi32(b0.z, (uint32_t)span_y) - r.crop_pad : (do_crop ? -r.crop_pad : 0));
    s.crop_dx = (int8_t)(do_crop && span_x > 1 ? (int)umulhi32(b0.w, (uint32_t)span_x) - r.crop_pad : (do_crop ? -r.crop_pad : 0));
    s.reserved = 0;
    s.zero_box[0] = s.zero_box[1] = s.zero_box[2] = s.zero_box[3] = 0;
    if (r.zero_box_len > 0) {                                             // data.py:239-246
        c.z = 1; U4 b1 = philox4x32_10(c, k0, k1);
        int cy = (int)umulhi32(b1.x, (uint32_t)out_h), cx = (int)umulhi32(b1.y, (uint32_t)out_w);
        int half = r.zero_box_len / 2;
        int ya = cy - half, yb = cy + half, xa = cx - half, xb = cx + half;
        s.zero_box[0] = (int16_t)(ya < 0 ? 0 : ya > out_h ? out_h : ya);
        s.zero_box[1] = (int16_t)(yb < 0 ? 0 : yb > out_h ? out_h : yb);
        s.zero_box[2] = (int16_t)(xa < 0 ? 0 : xa > out_w ? out_w : xa);
        s.zero_box[3] = (int16_t)(xb < 0 ? 0 : xb > out_w ? out_w : xb);
    }
    uint32_t gate = 0, sign = 0;
    for (int j = 0; j < n_op; ++j) {
        c.z = 2 + j; U4 bj = philox4x32_10(c, k0, k1);
        const OpRec* o = ops + ((size_t)s.sub * n_op + j) * 2;
        double u = (double)bj.x * (1.0 / 4294967296.0);
        boxes[j].x0 = boxes[j].y0 = 0; boxes[j].x1 = boxes[j].y1 = -1;
        if (u > probs[(size_t)s.sub * n_op + j]) continue;               // data.py:261
        gate |= 1u << j;
        if (o->draw == 1) {                                               // mirror: random() > 0.5
            if (bj.y >> 31) sign |= 1u << j;
        } else if (o->draw == 2 && o->kind == K_CUTOUT) {
            double v; { union { int32_t i[2]; double d; } cv; cv.i[0] = o->a[0]; cv.i[1] = o->a[1]; v = cv.d; }
            boxes[j] = cutout_box(W, H, v, (double)bj.z * (1.0 / 4294967296.0), (double)bj.w * (1.0 / 4294967296.0));
        }
    }
    s.gate = (uint8_t)gate; s.sign = (uint8_t)sign;
}

// One candidate policy of a multi-policy TTA call (faa_augment_tta_policies, faa_augment_ragged_policies): its compiled
// table at the launch's size (the ragged resolve takes each image's table from its RaggedImg instead), probabilities and
// sub-policy count.  Candidates share n_op; only the table, the probabilities and n_sub the decisions are drawn from
// differ per entry, never the Philox keys.
struct PolicyRef { const OpRec* ops; const double* probs; int32_t n_sub; int32_t reserved; };

// schedule entry v of a uniform multi-policy TTA call, v = (t * K + r) * B + i, belongs to candidate t = v / (K * B)
FAA_HD int tta_candidate(int v, int per_candidate) { return v / per_candidate; }

// fast exact division of q by d via a 32-bit reciprocal (valid while q*d < 2^32)
FAA_HD uint32_t recip32(uint32_t d) { return (uint32_t)((0x100000000ull + d - 1) / d); }
FAA_HD uint32_t fastdiv(uint32_t q, uint32_t rcp) { return umulhi32(q, rcp); }

// ------------------------------------------------ vectorised 3x3 Sharpness --
// Four consecutive output pixels (x0 % 4 == 0) of Sharpness (augmentations.py:112-114) from
// three source rows.  rm/r0/rp point at pixel x0 of rows y-1, y, y+1 (any address space, 4-byte
// aligned); has_l / has_r tell whether columns x0-1 / x0+4 exist; edge bits mark pixels of the
// quad that lie on the image border (copied unchanged, like Pillow's filter).  The 3x3 sums are
// built from per-column sums with R|B packed in one register (16-bit lanes) and G in another.
FAA_HD uint32_t ld32(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const uint32_t*>(p);
#else
    uint32_t v; __builtin_memcpy(&v, p, 4); return v;
#endif
}
FAA_HD void row6(const uint8_t* r, bool has_l, bool has_r, uint32_t px[6]) {
    uint32_t w0 = ld32(r), w1 = ld32(r + 4), w2 = ld32(r + 8);
    px[0] = has_l ? (ld32(r - 4) >> 8) : 0u;
    px[1] = w0 & 0xFFFFFFu;
    px[2] = (w0 >> 24) | ((w1 & 0xFFFFu) << 8);
    px[3] = (w1 >> 16) | ((w2 & 0xFFu) << 16);
    px[4] = w2 >> 8;
    px[5] = has_r ? (ld32(r + 12) & 0xFFFFFFu) : 0u;
}
FAA_HD void sharp_quad(const uint8_t* rm, const uint8_t* r0, const uint8_t* rp, bool has_l, bool has_r,
                       bool row_is_border, bool left_is_border, bool right_is_border, float alpha, bool clip,
                       uint32_t out[4]) {
    uint32_t c[6];
    row6(r0, has_l, has_r, c);
    if (row_is_border) { out[0] = c[1]; out[1] = c[2]; out[2] = c[3]; out[3] = c[4]; return; }
    uint32_t a[6], b[6];
    row6(rm, has_l, has_r, a);
    row6(rp, has_l, has_r, b);
    uint32_t rb[6], g[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        rb[i] = (a[i] & 0xFF00FFu) + (c[i] & 0xFF00FFu) + (b[i] & 0xFF00FFu);
        g[i] = ((a[i] >> 8) & 0xFFu) + ((c[i] >> 8) & 0xFFu) + ((b[i] >> 8) & 0xFFu);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t ctr = c[k + 1];
        if ((k == 0 && left_is_border) || (k == 3 && right_is_border)) { out[k] = ctr; continue; }
        uint32_t srb = rb[k] + rb[k + 1] + rb[k + 2] + 4u * (ctr & 0xFF00FFu);
        uint32_t sg = g[k] + g[k + 1] + g[k + 2] + 4u * ((ctr >> 8) & 0xFFu);
        uint32_t dr = (2u * (srb & 0xFFFFu) + 13u) / 26u, db = (2u * (srb >> 16) + 13u) / 26u;
        uint32_t dg = (2u * sg + 13u) / 26u;                       // [1 1 1;1 5 1;1 1 1]/13, round half up
        out[k] = blend_u8(dr, ctr & 255u, alpha, clip) | (blend_u8(dg, (ctr >> 8) & 255u, alpha, clip) << 8) |
                 (blend_u8(db, (ctr >> 16) & 255u, alpha, clip) << 16);
    }
}

// ------------------------------------------------------- per-image program --
// What the resolve step hands to the pixel kernel for one image: the two applied op records,
// clipped Cutout boxes, the tail decisions and the evaluation class of the final pass.
enum ProgClass : uint8_t {
    C_PLAIN = 0,     // no op applied, aligned: 12-byte vector loads straight to the store
    C_LUT = 1,       // every applied op is a per-channel LUT (static / hist / blend-with-const), aligned
    C_POINT = 2,     // pointwise incl. Color / Cutout, aligned
    C_GENERIC = 3,   // geometric ops, unaligned rows, ...: per-pixel lazy evaluation of the chain
    C_SHARP = 4,     // Sharpness on the raw image then a pointwise op, aligned: vectorised 3x3
    C_GEOM = 6,      // one geometric op + pointwise ops: incremental fixed-point source coordinates
    C_SG = 7,        // Sharpness then a geometric op: the sharpened image goes through a global scratch
                     // image (L2-resident), then the gather reads it - no 9-tap re-evaluation per gather
    C_MAT = 5,       // op0 then (Sharpness | statistics op): op0's output is materialised chunk-wise in
                     // shared memory and op1 runs on it as a single-op program of class `cls2`
    C_GEOM2 = 8      // two geometric ops (launches with the lean gather paths only): the two nearest-neighbour
                     // coordinate maps compose per pixel - no intermediate image
};

struct alignas(16) Prog {   // 96 bytes (moved with 128-bit loads / stores)
    OpRec op[2];
    Box box[2];
    int16_t zero_box[4];
    int8_t crop_dy, crop_dx; uint8_t flip; uint8_t cls;
    uint8_t stat_mask;           // bit j: slot j needs whole-image statistics
    uint8_t lut_mask;            // bit j: slot j is evaluated through a 3x256 LUT
    uint8_t bucket;              // scheduling cost bucket (0 = most expensive)
    uint8_t cls2;                // C_MAT: class of the op1-only program run on the materialised chunk
};

FAA_HD bool kind_is_lutlike(int k) { return k == K_NONE || kind_uses_lut(k); }

// Sample + boxes -> Prog.  ops: compiled table [n_sub][n_op][2]; boxes: this sample's n_op boxes.
// allow: bit 0 = the launch has a materialisation chunk of at least 3 rows, bit 1 = it has a global
// scratch image (both only for single-source launches), bit 2 = split launch with the lean gather paths
// (float planes of the image's own size, W % 8 == 0, no crop), bit 3 = the light kernel is its lean variant
// (octet paths only: prog_is_light; split launches, so only the resolve kernel's programs - see lean_order).
FAA_HD void build_prog(const Sample& s_in, const Box* boxes, const OpRec* ops, int n_op, int op_base,
                       int apply_tail, int H, int W, int out_w, int allow, Prog& g) {
    const bool allow_mat = (allow & 1) != 0, allow_scratch = (allow & 2) != 0;
    Sample s = s_in;
    if (!apply_tail) { s.crop_dx = s.crop_dy = 0; s.flip = 0; s.zero_box[0] = s.zero_box[1] = s.zero_box[2] = s.zero_box[3] = 0; }
    g.crop_dy = s.crop_dy; g.crop_dx = s.crop_dx; g.flip = s.flip;
    for (int i = 0; i < 4; ++i) g.zero_box[i] = s.zero_box[i];
    g.stat_mask = 0; g.lut_mask = 0; g.bucket = 0; g.cls2 = C_GENERIC;
    int n = 0;
    for (int j = 0; j < 2; ++j) {
        int jj = op_base + j;
        OpRec o; o.kind = K_NONE; o.a[0] = o.a[1] = o.a[2] = o.a[3] = o.a[4] = o.a[5] = 0; o.draw = 0;
        if (jj < n_op && ((s.gate >> jj) & 1u)) o = ops[((size_t)s.sub * n_op + jj) * 2 + ((s.sign >> jj) & 1u)];
        Box b; b.x0 = b.y0 = 0; b.x1 = b.y1 = -1;
        if (o.kind == K_CUTOUT) {                 // ImageDraw.rectangle clips to the image
            b = boxes[jj];
            if (b.x0 < 0) b.x0 = 0;
            if (b.y0 < 0) b.y0 = 0;
            if (b.x1 > W - 1) b.x1 = (int16_t)(W - 1);
            if (b.y1 > H - 1) b.y1 = (int16_t)(H - 1);
            if (b.x1 < b.x0 || b.y1 < b.y0) o.kind = K_NONE;
        }
        if (o.kind != K_NONE) { g.op[n] = o; g.box[n] = b; ++n; }   // applied ops are compacted to the front
    }
    for (int j = n; j < 2; ++j) {
        g.op[j].kind = K_NONE; g.op[j].a[0] = g.op[j].a[1] = g.op[j].a[2] = g.op[j].a[3] = g.op[j].a[4] = g.op[j].a[5] = 0;
        g.op[j].draw = 0;
        g.box[j].x0 = g.box[j].y0 = 0; g.box[j].x1 = g.box[j].y1 = -1;
    }
    bool all_point = true, all_lut = true;
    for (int j = 0; j < 2; ++j) {
        const int k = g.op[j].kind;
        if (kind_needs_hist(k) || kind_needs_mean(k)) g.stat_mask |= (uint8_t)(1u << j);
        if (kind_uses_lut(k)) g.lut_mask |= (uint8_t)(1u << j);
        all_point = all_point && kind_is_pointwise(k);
        all_lut = all_lut && kind_is_lutlike(k);
    }
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    const bool aligned = ((W & 3) == 0) && ((out_w & 3) == 0) && ((s.crop_dx & 3) == 0);
    const bool k1_stat = kind_needs_hist(k1) || kind_needs_mean(k1);
    // a histogram op behind per-channel LUT ops needs no second pass: its histogram is the raw
    // histogram pushed forward through the first LUT
    const bool push = k0 != K_NONE && kind_is_lutlike(k0) && kind_needs_hist(k1);
    if (allow_mat && k0 != K_NONE && (k1 == K_SHARPNESS || (k1_stat && !push))) {
        g.cls = C_MAT;
        g.cls2 = !aligned ? C_GENERIC : (k1 == K_SHARPNESS ? C_SHARP : C_LUT);
    } else if (allow_scratch && k0 == K_SHARPNESS && (k1 == K_AFFINE || k1 == K_SHIFT) && (W & 3) == 0) {
        g.cls = C_SG;
    } else if (((k0 == K_AFFINE || k0 == K_SHIFT) && kind_is_pointwise(k1)) ||
               ((k1 == K_AFFINE || k1 == K_SHIFT) && kind_is_pointwise(k0))) g.cls = C_GEOM;
    else if ((allow & 4) && (k0 == K_AFFINE || k0 == K_SHIFT) && (k1 == K_AFFINE || k1 == K_SHIFT)) g.cls = C_GEOM2;
    else if (!aligned) g.cls = C_GENERIC;
    else if (all_point) g.cls = n == 0 ? C_PLAIN : all_lut ? C_LUT : C_POINT;
    else if (k0 == K_SHARPNESS && kind_is_pointwise(k1)) g.cls = C_SHARP;
    else g.cls = C_GENERIC;
}

// Programs of lean light launches (allow bit 3), after build_prog: Color, then a gather == the gather, then Color (Color
// is per pixel and maps the gather's zero fill to zero).  The lean light kernel has no path for Color in front of a
// gather; the mid kernel runs gather -> Color (prog_two_stage).  Both slots are C_GEOM's, neither has a mask bit.
FAA_HD void lean_order(Prog& g, int allow) {
    if ((allow & 8) && g.op[0].kind == K_COLOR && (g.op[1].kind == K_AFFINE || g.op[1].kind == K_SHIFT)) {
        const OpRec o = g.op[0]; g.op[0] = g.op[1]; g.op[1] = o;
        const Box b = g.box[0]; g.box[0] = g.box[1]; g.box[1] = b;
    }
}

// "Light" programs need no whole-image statistics and no neighbourhood: they run in the small
// streaming kernel (no cluster, few registers); everything else runs in the cluster kernel.
// allow bit 3: the light kernel is its lean variant, which has the octet paths only.  Its Color / Cutout programs are the
// ones a float table can finish (alone, or followed by a static LUT) and Cutout followed by a gather; the other pairs with
// Color or Cutout run in the mid kernel (prog_two_stage).
FAA_HD bool prog_is_light(const Prog& g, int allow = 0) {
    if (g.stat_mask != 0 || !(g.cls == C_PLAIN || g.cls == C_LUT || g.cls == C_POINT || g.cls == C_GEOM || g.cls == C_GEOM2))
        return false;
    if (!(allow & 8)) return true;
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    if (g.cls == C_POINT) return k1 == K_NONE || kind_uses_lut(k1);
    if (g.cls == C_GEOM) {
        const bool g0 = k0 == K_AFFINE || k0 == K_SHIFT;
        const int pk = g0 ? k1 : k0;                  // the pointwise partner
        return pk == K_NONE || kind_uses_lut(pk) || (!g0 && pk == K_CUTOUT);
    }
    return true;
}

// "Mid" programs: whole-image statistics feeding per-channel LUTs, or Sharpness (+ a static LUT) - they need a
// cluster (statistics exchange) or only halo rows, but none of the cluster kernel's materialisation / generic
// machinery: they run in their own lean kernel when the launch geometry allows it (three-way split).
// Two-stage programs of the mid kernel: stage A materialises op0 in the band buffer (per-channel LUT / Color / Cutout in
// place, a gather from global memory, Sharpness through the global scratch image), stage B runs op1 on the band.
FAA_HD bool prog_two_stage(const Prog& g, int allow) {
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    const bool scratch = (allow & 2) != 0;
    if (g.cls == C_MAT) {
        const bool op0 = kind_uses_lut(k0) || k0 == K_COLOR || k0 == K_CUTOUT || k0 == K_AFFINE || k0 == K_SHIFT ||
                         (k0 == K_SHARPNESS && scratch);
        const bool op1 = (k1 == K_SHARPNESS && g.cls2 == C_SHARP) ||
                         ((k1 == K_AUTOCONTRAST || k1 == K_EQUALIZE || k1 == K_CONTRAST) && g.cls2 == C_LUT);
        return op0 && op1;
    }
    // lean light launches: a static LUT, Color, Cutout or a gather, then Color / Cutout (stage A in place or a gather)
    if ((allow & 8) && g.stat_mask == 0 && (g.cls == C_POINT || g.cls == C_GEOM)) return k1 == K_COLOR || k1 == K_CUTOUT;
    if (g.cls == C_SG) return true;                                                   // Sharpness, then a gather (scratch exists)
    if (g.cls == C_SHARP) return scratch && (k1 == K_COLOR || k1 == K_CUTOUT);        // Sharpness, then Color / Cutout
    if (g.cls == C_POINT) return g.stat_mask == 1 && (k1 == K_COLOR || k1 == K_CUTOUT);   // statistics LUT, then Color / Cutout
    return false;
}

FAA_HD bool prog_is_mid(const Prog& g, int allow) {
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    if (g.cls == C_LUT) return g.stat_mask != 0;
    // statistics LUT, then a gather: the table rides through the lean gather paths (fill colour = plain zero)
    if (g.cls == C_GEOM && g.stat_mask != 0)
        return (allow & 4) && g.stat_mask == 1 && (k0 == K_AUTOCONTRAST || k0 == K_EQUALIZE || k0 == K_CONTRAST) &&
               (k1 == K_AFFINE || k1 == K_SHIFT);
    if (g.cls == C_SHARP && (k1 == K_NONE || k1 == K_LUT || k1 == K_BRIGHTNESS)) return true;
    return prog_two_stage(g, allow);
}

// Rough relative cost of an image (per-pixel work units) - only used to schedule the
// expensive images first (longest-processing-time order); never affects results.
FAA_HD uint32_t op_unit_cost(int k) {
    return k == K_NONE ? 0u : k == K_SHARPNESS ? 12u : (k == K_AFFINE || k == K_SHIFT) ? 4u : k == K_COLOR ? 3u : 1u;
}
FAA_HD uint32_t prog_cost(const Prog& g) {
    const int k0 = g.op[0].kind, k1 = g.op[1].kind;
    uint32_t c0 = op_unit_cost(k0), c1 = op_unit_cost(k1);
    if (g.cls == C_SHARP || g.cls == C_SG) c0 = 5u;
    if (g.cls == C_MAT && g.cls2 == C_SHARP) c1 = 5u;
    uint32_t chain = (k1 == K_SHARPNESS && g.cls != C_MAT) ? c1 + 9u * c0 : c0 + c1;   // lazy Sharpness: 9 taps below it
    if (k0 == K_SHARPNESS && (k1 == K_AFFINE || k1 == K_SHIFT) && g.cls != C_SG) chain = c1 + 9u * 4u;
    uint32_t cost = 2u + chain + (g.cls == C_GENERIC ? 2u : 0u);
    if (g.stat_mask & 1u) cost += 2u;                                    // extra pass over the raw band
    if (g.stat_mask & 2u) cost += 2u + c0;                               // extra pass evaluating op 0
    return cost;
}

// ------------------------------------------------------- crop + bicubic resize --
// EfficientNetRandomCrop / EfficientNetCenterCrop (data.py:267-345) followed by
// transforms.Resize((s, s), BICUBIC) (data.py:61-62, 76-77), i.e. Pillow's ImagingResample
// for 8-bit RGB: per axis an fp64 coefficient table, converted to 22-bit fixed point; a
// horizontal pass into a uint8 intermediate, then a vertical pass.  A pass whose axis keeps
// its size is the identity (Pillow skips it; the bicubic weights would be exactly 1, 0, 0 ...).
struct CropBox { int32_t x0, y0, w, h; };                 // == faa_crop_box_t

constexpr int kResPrecisionBits = 22;

FAA_HD double d_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    volatile double r = a / b; return r;
#endif
}
FAA_HD double d_sqrt(double a) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(a);
#else
    volatile double r = __builtin_sqrt(a); return r;
#endif
}
FAA_HD double d_rint(double a) {                           // Python round() of a float: half to even
#if defined(__CUDA_ARCH__)
    return rint(a);
#else
    return __builtin_rint(a);
#endif
}

// Pillow bicubic_filter, a = -0.5 (support 2)
FAA_HD double bicubic_w(double x) {
    if (x < 0.0) x = -x;
    if (x < 1.0) return d_add(d_mul(d_mul(d_add(d_mul(1.5, x), -2.5), x), x), 1.0);
    if (x < 2.0) return d_mul(d_add(d_mul(d_add(d_mul(d_add(x, -5.0), x), 8.0), x), -4.0), -0.5);
    return 0.0;
}

// Taps of one axis: ksize of precompute_coeffs (an upper bound on the taps of any output index).
FAA_HD int resize_ksize(int in, int out) {
    const double scale = d_div((double)in, (double)out);
    const double fs = scale > 1.0 ? scale : 1.0;
    const double support = d_mul(2.0, fs);
    const double c = (double)(int)support;
    return 2 * (int)(c < support ? c + 1.0 : c) + 1;
}

// precompute_coeffs + normalize_coeffs_8bpc for output index xx: first input index and tap count, then the
// int32 weights k[0..n).  Identity axes (in == out) give one tap of weight 1 << 22.
FAA_HD int resize_coeffs(int in, int out, int xx, int* xmin_out, int32_t* k) {
    if (in == out) { *xmin_out = xx; k[0] = 1 << kResPrecisionBits; return 1; }
    const double scale = d_div((double)in, (double)out);
    const double fs = scale > 1.0 ? scale : 1.0;
    const double support = d_mul(2.0, fs);
    const double ss = d_div(1.0, fs);
    const double center = d_mul(d_add((double)xx, 0.5), scale);
    int xmin = (int)d_add(d_add(center, -support), 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)d_add(d_add(center, support), 0.5);
    if (xmax > in) xmax = in;
    const int n = xmax - xmin;
    double ww = 0.0;
    for (int x = 0; x < n; ++x) ww = d_add(ww, bicubic_w(d_mul(d_add(d_add((double)(x + xmin), -center), 0.5), ss)));
    for (int x = 0; x < n; ++x) {
        double w = bicubic_w(d_mul(d_add(d_add((double)(x + xmin), -center), 0.5), ss));
        if (ww != 0.0) w = d_div(w, ww);
        const double f = d_mul(w, (double)(1 << kResPrecisionBits));
        k[x] = (int32_t)(w < 0.0 ? d_add(f, -0.5) : d_add(f, 0.5));
    }
    *xmin_out = xmin;
    return n;
}

// (1 << 21) + sum, shifted and clipped to a byte (Pillow clip8)
FAA_HD uint32_t resize_clip8(int32_t ss) {
    if (ss <= 0) return 0u;
    if (ss >= (1 << (kResPrecisionBits + 8))) return 255u;
    return (uint32_t)(ss >> kResPrecisionBits);
}

// EfficientNetCenterCrop (data.py:337-345) through Image.crop's int(round()) of the box
FAA_HD CropBox center_crop_box(int H, int W, int img_size) {
    const int short_side = W < H ? W : H;
    const double c = d_mul(d_div((double)img_size, (double)(img_size + 32)), (double)short_side);
    const double top = d_rint(d_div(d_add((double)H, -c), 2.0));
    const double left = d_rint(d_div(d_add((double)W, -c), 2.0));
    CropBox b;
    b.x0 = (int32_t)left; b.y0 = (int32_t)top;
    b.w = (int32_t)d_rint(d_add(left, c)) - b.x0;
    b.h = (int32_t)d_rint(d_add(top, c)) - b.y0;
    return b;
}

struct CropCfg {                                           // == faa_crop_cfg_t
    int32_t mode;                                          // 0 random, 1 center
    int32_t img_size;
    double min_covered, aspect_lo, aspect_hi, area_lo, area_hi;
    int32_t max_attempts, reserved;
    RngCfg rng;
};

// One attempt of EfficientNetRandomCrop.__call__ (data.py:280-317) from its two uniforms (u_ar: the aspect
// ratio's random(), u_h: the height's).  Returns 0 = rejected, 1 = box size accepted (w, h set; the caller then
// draws x, y), 2 = the crop is the whole image (center-crop fallback).
FAA_HD int crop_attempt(const CropCfg& c, int W, int H, double u_ar, double u_h, int& w_out, int& h_out) {
    const double area = (double)((long long)W * H);
    const double min_area = d_mul(c.area_lo, area), max_area = d_mul(c.area_hi, area);
    const double ar = d_add(c.aspect_lo, d_mul(d_add(c.aspect_hi, -c.aspect_lo), u_ar));     // random.uniform
    int height = (int)d_rint(d_sqrt(d_div(min_area, ar)));
    int max_height = (int)d_rint(d_sqrt(d_div(max_area, ar)));
    if (d_mul((double)max_height, ar) > (double)W) {
        max_height = (int)d_div(d_add(d_add((double)W, 0.5), -1e-7), ar);
        if (d_mul((double)max_height, ar) > (double)W) max_height -= 1;
    }
    if (max_height > H) max_height = H;
    if (height >= max_height) height = max_height;
    height = (int)d_rint(d_add((double)height, d_mul((double)(max_height - height), u_h)));
    const int width = (int)d_rint(d_mul((double)height, ar));
    const double a = (double)((long long)width * height);
    if (a < min_area || a > max_area) return 0;
    if (width > W || height > H) return 0;
    if (a < d_mul(c.min_covered, area)) return 0;
    if (width == W && height == H) return 2;
    w_out = width; h_out = height;
    return 1;
}

// Device-side crop sampler: same distributions as EfficientNetRandomCrop, drawn from Philox keyed like
// philox_sample (seed, global sample index) in a counter subspace philox_sample never uses: w = 1, z = attempt
// number for the two uniforms of an attempt, z = 0xFFFFFFFF for the offsets x, y.
FAA_HD CropBox philox_crop_box(const CropCfg& c, uint64_t index, int H, int W) {
    if (c.mode != 0) return center_crop_box(H, W, c.img_size);
    const uint32_t k0 = (uint32_t)c.rng.seed, k1 = (uint32_t)(c.rng.seed >> 32);
    U4 ctr; ctr.x = (uint32_t)index; ctr.y = (uint32_t)(index >> 32); ctr.w = 1u;
    for (int t = 0; t < c.max_attempts; ++t) {
        ctr.z = (uint32_t)t;
        const U4 b = philox4x32_10(ctr, k0, k1);
        int w = 0, h = 0;
        const int r = crop_attempt(c, W, H, (double)b.x * (1.0 / 4294967296.0), (double)b.y * (1.0 / 4294967296.0), w, h);
        if (r == 0) continue;
        if (r == 2) break;
        ctr.z = 0xFFFFFFFFu;
        const U4 o = philox4x32_10(ctr, k0, k1);
        CropBox bx;
        bx.x0 = (int32_t)umulhi32(o.x, (uint32_t)(W - w + 1));      // random.randint(0, W - w)
        bx.y0 = (int32_t)umulhi32(o.y, (uint32_t)(H - h + 1));
        bx.w = w; bx.h = h;
        return bx;
    }
    return center_crop_box(H, W, c.img_size);
}

// ------------------------------------------------- launch planner (host only) --
// Which code each kernel of a policy launch runs, decided from the launch's sizes and buffer addresses alone - no
// device, no allocation.  faa_cabi.cu launches what plan_launch returns; the host build (tests/emu) exports the same
// function, so the CPU tests check the launch-geometry case table against the planner itself.

// row-band geometry of a pixel launch, precomputed on the host (no divisions in the kernels)
struct BandGeom {
    int32_t bands;              // CTAs per image
    int32_t band_cap;           // bytes of dynamic shared memory per staged band (0: staging off)
    int32_t y[9];               // band b owns image rows [y[b], y[b+1]) for whole-image statistics
    int32_t oy[9];              // ... and output rows [oy[b], oy[b+1])
    uint32_t lo[8], len[8];     // staged byte range of the raw image per band (len 0: nothing staged)
};

// the byte range of image rows a CTA may touch through the band-local paths
inline void band_range(int band, int bands, int H, int W, int out_h, int crop_pad, uint32_t img_bytes, uint32_t& lo,
                       uint32_t& len) {
    const int y0 = (int)((uint32_t)(band * H) / (uint32_t)bands), y1 = (int)((uint32_t)((band + 1) * H) / (uint32_t)bands);
    const int oy0 = (int)((uint32_t)(band * out_h) / (uint32_t)bands), oy1 = (int)((uint32_t)((band + 1) * out_h) / (uint32_t)bands);
    int r0 = (y0 < oy0 - crop_pad ? y0 : oy0 - crop_pad) - 1;
    int r1 = (y1 > oy1 + crop_pad ? y1 : oy1 + crop_pad) + 1;
    if (r0 < 0) r0 = 0;
    if (r1 > H) r1 = H;
    if (r1 <= r0) { lo = 0; len = 0; return; }
    const uint32_t row = (uint32_t)W * 3u;
    lo = ((uint32_t)r0 * row) & ~15u;
    uint32_t hi = ((uint32_t)r1 * row + 15u) & ~15u;
    if (hi > img_bytes) hi = img_bytes;
    len = hi - lo;
}

inline int pick_bands(int H, int out_h, int out_w) {
    // aim for >= ~1024 output quads per CTA; cluster size must be a power of two <= 8
    long long quads = (long long)out_h * ((out_w + 3) / 4);
    int b = 1;
    while (b < 8 && quads / (b * 2) >= 1024 && b * 2 <= H && b * 2 <= out_h) b *= 2;
    return b;
}

inline void fill_geom(BandGeom& g, int bands, int H, int W, int out_h, int crop_pad, bool stage) {
    g = BandGeom{}; g.bands = bands;
    uint32_t cap = 0;
    for (int b = 0; b <= bands; ++b) {
        g.y[b] = (int32_t)((uint32_t)(b * H) / (uint32_t)bands);
        g.oy[b] = (int32_t)((uint32_t)(b * out_h) / (uint32_t)bands);
    }
    for (int b = 0; b < bands && stage; ++b) {
        band_range(b, bands, H, W, out_h, crop_pad, (uint32_t)H * (uint32_t)W * 3u, g.lo[b], g.len[b]);
        if (g.len[b] > cap) cap = g.len[b];
    }
    g.band_cap = (int32_t)((cap + 127u) & ~127u);
}

// the largest band of `bands`, rounded up to 128 bytes
inline uint32_t band_capacity(int bands, int H, int W, int out_h, int crop_pad) {
    BandGeom g;
    fill_geom(g, bands, H, W, out_h, crop_pad, true);
    return (uint32_t)g.band_cap;
}

// the mid kernel runs enough threads for its band: 512 for the tall bands of large images, 256 otherwise
inline int mid_kernel_threads(uint32_t band_cap) { return band_cap > 48 * 1024 ? 512 : 256; }

constexpr uint64_t kSplitMin = (uint64_t)4 << 20;     // pixels per launch from which two pixel kernels pay off

struct PlanInput {
    int32_t H, W, out_h, out_w, batch;
    int32_t crop_pad;               // the larger of the tail's and the rng's, clamped to H
    bool out_u8;                    // uint8 HWC output (else fp32 / fp16 / bf16 planes)
    uint32_t in_mod16, out_mod16;   // the input's and the output's base address mod 16
    // fused Mixup (a partner image per output); the final window of the policy; some program is Sharpness -> gather
    bool two_src, apply_tail, has_sg;
    uint64_t split_min;             // pixels per launch from which the light (+ mid) kernels take part of the work
    // decisions drawn on the device (else resolved samples); the caller lets the next batch be resolved ahead
    bool philox, allow_ahead;
};

struct LaunchPlan {
    BandGeom geo[2];            // [0] cluster kernel (band_cap 0: no TMA staging), [1] light streaming kernel
    BandGeom mid;               // the mid kernel's own (taller) bands, when use_mid
    int32_t mid_threads;        // ... and its threads per CTA
    bool stage;                 // TMA-stage the cluster kernel's band
    bool octets;                // the 8-pixel fast paths
    int32_t mat_cap;            // bytes of the materialisation chunk (0: none)
    bool use_order;             // the resolve kernel writes a cost-sorted schedule (order / n_heavy)
    bool use_split;             // the light streaming kernel (and the mid kernel) take the programs they cover
    bool use_mid;               // three-way split: statistics-LUT and Sharpness programs run in the mid kernel
    int32_t split;              // ResolveParams::split
    int32_t allow;              // ResolveParams::allow: bit 0 chunk, bit 1 scratch image, bit 2 lean gathers, bit 3 lean_light
    bool lean_light;            // the light kernel runs its lean variant (octet paths only, 4 CTAs / SM)
    bool scratch;               // a scratch image per image (Sharpness -> gather)
    bool no_heavy;              // every program is light or mid: the cluster kernel is not launched
    bool self_resolving;        // one kernel that draws and builds its programs itself
    bool use_chain;             // chained schedule (else the event schedule), unless self-resolving
    bool speculate;             // resolve the next call's batch ahead (resolve-ahead)
};

inline LaunchPlan plan_launch(const PlanInput& in) {
    LaunchPlan L = {};
    const int h = in.H, w = in.W;
    const bool same_size = in.out_w == w && in.out_h == h;
    // TMA band staging needs 16-byte aligned image bases and a band that fits shared memory
    // (crop_pad only sizes the staged band; rows outside it are read from global memory)
    const int bands = pick_bands(h, in.out_h, in.out_w);
    const uint32_t cap = band_capacity(bands, h, w, in.out_h, in.crop_pad);
    L.stage = ((size_t)h * w * 3) % 16 == 0 && in.in_mod16 == 0 && (size_t)cap * (in.two_src ? 2 : 1) <= 150 * 1024;
    fill_geom(L.geo[0], bands, h, w, in.out_h, in.crop_pad, L.stage);
    int lb = bands;
    if (bands == 8) {
        // the light kernel needs no cluster, so any band count works: take the one in 5..8 whose
        // quads-per-CTA fills whole 256-thread iterations best (224x224: 7 bands = exactly 7 iterations)
        const int qpr = (in.out_w + 3) / 4;
        double best = -1.0;
        for (int b = 8; b >= 5; --b) {
            const int rows = (in.out_h + b - 1) / b;
            const int quads = rows * qpr, iters = (quads + 255) / 256;
            const double eff = (double)quads / (iters * 256.0) * ((double)in.out_h / (rows * b));
            if (eff > best + 0.02) { best = eff; lb = b; }
        }
    }
    fill_geom(L.geo[1], lb, h, w, in.out_h, in.crop_pad, L.stage && band_capacity(lb, h, w, in.out_h, in.crop_pad) <= 100 * 1024);
    L.octets = (w & 7) == 0 && same_size && in.out_mod16 == 0 && L.stage;    // (uint8 HWC included: 24-byte octets)
    // materialisation chunk: a whole band (+ halo, + crop slack) when that is <= 24 KB, else ~16 KB; >= 3 rows
    const int pitch = w * 3;
    const int band_rows = (h + bands - 1) / bands + 2 + 2 * in.crop_pad;
    int mat_rows = band_rows * pitch <= 24576 ? band_rows : 16384 / pitch;
    if (mat_rows > h + 2) mat_rows = h + 2;
    L.mat_cap = (!in.two_src && mat_rows >= 3) ? ((mat_rows * pitch + 32 + 15) & ~15) : 0;   // + 2 guard bands
    L.use_order = !in.two_src;
    // (small launches are launch-latency bound: one pixel kernel is faster there; uint8 HWC output - the Mixup exchange
    //  format - splits when the lean octet paths can write it)
    L.use_split = L.use_order && (!in.out_u8 || (L.octets && in.crop_pad == 0 && in.apply_tail)) &&
                  (uint64_t)in.batch * h * w >= in.split_min;
    // Three-way split: statistics-LUT and Sharpness programs run in the lean mid kernel.
    // Needs the geometry its paths assume: float planes of the image's own size, no crop, W % 4 == 0, staged bands.
    L.use_mid = L.use_split && L.stage && (w & 3) == 0 && same_size && in.crop_pad == 0 && in.out_mod16 == 0;
    L.split = L.use_mid ? 2 : L.use_split ? 1 : 0;
    if (L.use_mid) {            // halve the band count while a band (+ halo) stays <= 80 KB (2 CTAs / SM)
        int mb = bands;
        while (mb > 1 && band_capacity(mb / 2, h, w, in.out_h, 0) <= 80 * 1024) mb /= 2;
        fill_geom(L.mid, mb, h, w, in.out_h, 0, true);
        L.mid_threads = mid_kernel_threads((uint32_t)L.mid.band_cap);
    }
    // scratch images: Sharpness -> gather programs of the cluster kernel, every Sharpness-first two-op program of the mid
    // kernel
    L.scratch = (in.has_sg || L.use_mid) && !in.two_src && (w & 3) == 0;
    // allow bit 0: the chunk, bit 1: a scratch image, bit 2: the lean gather paths exist in this launch
    L.allow = (L.mat_cap > 0 ? 1 : 0) | (L.scratch ? 2 : 0) | (L.use_split && L.octets && in.crop_pad == 0 ? 4 : 0);
    // The lean light kernel has only the octet paths: every light entry must find its band staged and its output the
    // (possibly mirrored) image itself.  Philox draws no crop offset without crop padding at the image's own size;
    // resolved records carry whatever offsets their caller drew, so those launches keep the kernel with the generic paths.
    L.lean_light = (L.allow & 4) && L.geo[1].band_cap > 0 && in.philox;
    if (L.lean_light) L.allow |= 8;
    // With the lean gathers (allow bit 2) and a scratch image (bit 1) every program of a three-way split is light or mid
    // (prog_is_light / prog_is_mid cover all class combinations; tests/test_gpu_fastpaths.py runs every ordered op pair
    // through this schedule): the cluster kernel has nothing to do and is not launched.
    L.no_heavy = L.use_mid && (L.allow & 6) == 6 && L.mat_cap > 0;
    const bool ahead = in.philox && !in.two_src;
    // Only for tiny images (CIFAR): there the one-block resolve kernel is as long as the pixel kernel; for larger images
    // every band CTA would repeat the whole serial resolve work.
    L.self_resolving = !L.use_split && ahead && (size_t)h * w <= 4096;
    // Chained steps need the Philox sampler on the device and a caller that allows the next batch to be resolved ahead.
    // Launches too small to split are chained as well (resolve(N+1), cluster(N)): their step is bound by kernel latencies,
    // which only overlap across steps on one stream; uint8 output of one pixel kernel stays on the event schedule.
    L.use_chain = (L.use_split || !in.out_u8) && in.allow_ahead && ahead;
    L.speculate = in.allow_ahead && ahead;
    return L;
}

// ---- ragged policy launches: one launch over images of many sizes, uint8 HWC out at each image's own size ----------
// Each image runs the cluster kernel with the geometry plan_launch gives a uniform uint8 launch of that size alone (its
// bands, staged band, chunk, octets, allow bits).  The cluster size is a launch attribute, so the images are grouped
// into one pixel launch per band count present (1, 2, 4 or 8 CTAs per image).
struct RaggedImageIn { int32_t H, W; uint32_t in_mod16, out_mod16; };   // an image's size and its buffers' bases mod 16

struct RaggedGeom {                 // one distinct (size, staging, octets) of the batch
    int32_t H, W;
    LaunchPlan plan;                // plan_launch of a uniform uint8 launch of this size at these bases (unsplit)
    uint32_t rcp_out_qpr, rcp_w, rcp_wq, rcp_opr;    // fastdiv reciprocals (AugParams)
};

struct RaggedLaunch { int32_t bands, first, count; uint32_t smem; };   // images order[first, first + count)

struct RaggedPlan {
    std::vector<RaggedGeom> geoms;
    std::vector<int32_t> geom_of;   // [n] image -> geoms index
    std::vector<int32_t> order;     // [n] image indices, launch by launch; each launch's images largest first
    std::vector<RaggedLaunch> launches;   // largest first (by their first image): the large images start first
};

inline uint32_t fastdiv_rcp(uint32_t d) { return d <= 1 ? 0u : (uint32_t)((0x100000000ull + d - 1) / d); }

inline RaggedPlan plan_ragged(const RaggedImageIn* imgs, int n, bool has_sg) {
    RaggedPlan R;
    R.geom_of.resize((size_t)n);
    for (int i = 0; i < n; ++i) {
        const RaggedImageIn& m = imgs[i];
        PlanInput in = {};
        in.H = m.H; in.W = m.W; in.out_h = m.H; in.out_w = m.W; in.batch = 1; in.out_u8 = true;
        in.in_mod16 = m.in_mod16; in.out_mod16 = m.out_mod16; in.apply_tail = true; in.has_sg = has_sg;
        in.split_min = UINT64_MAX;                        // the cluster kernel alone
        const LaunchPlan L = plan_launch(in);
        int k = 0;
        while (k < (int)R.geoms.size() && !(R.geoms[k].H == m.H && R.geoms[k].W == m.W && R.geoms[k].plan.stage == L.stage &&
                                            R.geoms[k].plan.octets == L.octets)) ++k;
        if (k == (int)R.geoms.size()) {
            RaggedGeom g;
            g.H = m.H; g.W = m.W; g.plan = L;
            g.rcp_out_qpr = fastdiv_rcp((uint32_t)(m.W + 3) / 4); g.rcp_w = fastdiv_rcp((uint32_t)m.W);
            g.rcp_wq = fastdiv_rcp((uint32_t)m.W / 4); g.rcp_opr = (m.W & 7) ? 0u : fastdiv_rcp((uint32_t)m.W / 8);
            R.geoms.push_back(g);
        }
        R.geom_of[(size_t)i] = k;
    }
    // largest first (pixels, then batch position): the order of the launches and of the images inside each
    std::vector<int32_t> by_size((size_t)n);
    for (int i = 0; i < n; ++i) by_size[(size_t)i] = i;
    std::stable_sort(by_size.begin(), by_size.end(), [&](int32_t a, int32_t b) {
        return (int64_t)imgs[a].H * imgs[a].W > (int64_t)imgs[b].H * imgs[b].W;
    });
    for (int32_t i : by_size) {
        const RaggedGeom& g = R.geoms[(size_t)R.geom_of[(size_t)i]];
        const int32_t bands = g.plan.geo[0].bands;
        size_t l = 0;
        while (l < R.launches.size() && R.launches[l].bands != bands) ++l;
        if (l == R.launches.size()) R.launches.push_back({bands, 0, 0, 0u});
        RaggedLaunch& L = R.launches[l];
        ++L.count;
        const uint32_t smem = (uint32_t)g.plan.geo[0].band_cap + (uint32_t)g.plan.mat_cap;
        if (smem > L.smem) L.smem = smem;
    }
    int32_t at = 0;
    for (RaggedLaunch& L : R.launches) { L.first = at; at += L.count; L.count = 0; }
    R.order.resize((size_t)n);
    for (int32_t i : by_size) {
        size_t l = 0;
        while (R.launches[l].bands != R.geoms[(size_t)R.geom_of[(size_t)i]].plan.geo[0].bands) ++l;
        R.order[(size_t)(R.launches[l].first + R.launches[l].count++)] = i;
    }
    return R;
}

}  // namespace faa
