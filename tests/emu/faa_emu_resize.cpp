// faa_emu_resize.cpp - HOST build of the crop + bicubic resize arithmetic, TEST INFRASTRUCTURE ONLY.
//
// Compiles the coefficient builder, the crop-box functions and the Philox crop sampler of
// fast_autoaugment_b200/csrc/faa_core.cuh with g++ and drives them with faa_crop_resize_kernel's
// control flow (horizontal pass into a uint8 intermediate, then the vertical pass), one whole
// image at a time, so the CPU tests can check the kernel's arithmetic against the NumPy model of
// Pillow's resample.  The package never loads it.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

using namespace faa;

extern "C" {

int faa_emu_resize_ksize(int in, int out) { return resize_ksize(in, out); }

// bounds [out][2] = (xmin, n), k [out][ksize] (zero padded)
int faa_emu_resize_coeffs(int in, int out, int32_t* bounds, int32_t* k, int ksize) {
    for (int xx = 0; xx < out; ++xx) {
        int32_t* kk = k + (size_t)xx * ksize;
        memset(kk, 0, sizeof(int32_t) * ksize);
        int xmin = 0;
        const int n = resize_coeffs(in, out, xx, &xmin, kk);
        bounds[2 * xx] = xmin; bounds[2 * xx + 1] = n;
    }
    return 0;
}

// crop `box` of the uint8 [H][W][3] image, resized to out_h x out_w (uint8 [out_h][out_w][3])
int faa_emu_crop_resize(const uint8_t* in, int H, int W, const void* box_v, int out_h, int out_w, uint8_t* out) {
    (void)H;
    CropBox b; memcpy(&b, box_v, sizeof b);
    std::vector<int32_t> k((size_t)(b.w > b.h ? b.w : b.h) + 1);
    std::vector<uint8_t> mid((size_t)b.h * out_w * 3);
    for (int x = 0; x < out_w; ++x) {
        int xmin = 0;
        const int n = resize_coeffs(b.w, out_w, x, &xmin, k.data());
        for (int y = 0; y < b.h; ++y) {
            const uint8_t* src = in + ((size_t)(b.y0 + y) * W + b.x0 + xmin) * 3;
            for (int ch = 0; ch < 3; ++ch) {
                int32_t s = 1 << (kResPrecisionBits - 1);
                for (int t = 0; t < n; ++t) s += (int32_t)src[3 * t + ch] * k[t];
                mid[((size_t)y * out_w + x) * 3 + ch] = (uint8_t)resize_clip8(s);
            }
        }
    }
    for (int y = 0; y < out_h; ++y) {
        int ymin = 0;
        const int n = resize_coeffs(b.h, out_h, y, &ymin, k.data());
        for (int x = 0; x < out_w; ++x)
            for (int ch = 0; ch < 3; ++ch) {
                int32_t s = 1 << (kResPrecisionBits - 1);
                for (int t = 0; t < n; ++t) s += (int32_t)mid[((size_t)(ymin + t) * out_w + x) * 3 + ch] * k[t];
                out[((size_t)y * out_w + x) * 3 + ch] = (uint8_t)resize_clip8(s);
            }
    }
    return 0;
}

int faa_emu_center_crop_box(int H, int W, int img_size, void* box_out) {
    CropBox b = center_crop_box(H, W, img_size);
    memcpy(box_out, &b, sizeof b);
    return 0;
}

// one attempt of EfficientNetRandomCrop from its two uniforms: returns 0 / 1 / 2 like crop_attempt
int faa_emu_crop_attempt(const void* cfg_v, int H, int W, double u_ar, double u_h, int32_t* wh) {
    CropCfg c; memcpy(&c, cfg_v, sizeof c);
    int w = 0, h = 0;
    const int r = crop_attempt(c, W, H, u_ar, u_h, w, h);
    wh[0] = w; wh[1] = h;
    return r;
}

// boxes of samples first_index + i, i < n, as the kernel draws them
int faa_emu_philox_crop_boxes(const void* cfg_v, int n, int H, int W, void* boxes_out) {
    CropCfg c; memcpy(&c, cfg_v, sizeof c);
    CropBox* o = (CropBox*)boxes_out;
    for (int i = 0; i < n; ++i) o[i] = philox_crop_box(c, c.rng.first_index + (uint64_t)i, H, W);
    return 0;
}

}  // extern "C"
