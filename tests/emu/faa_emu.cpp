// faa_emu.cpp - HOST emulation of the CUDA kernels' control flow, TEST INFRASTRUCTURE ONLY.
//
// There is no GPU in the build container, so the CPU test-suite cannot run the kernels.
// This file compiles the very same per-pixel arithmetic header the kernels use
// (fast_autoaugment_b200/csrc/faa_core.cuh: program builder and classes, lazy op-chain
// evaluation, LUT builders, blend, Philox sampler) with g++ and drives it with the kernels'
// control flow (resolve -> statistics -> LUTs -> class-specialised final pass) for ONE band
// per image (cluster size 1), so the arithmetic the GPU will execute is checked against the
// oracle on the CPU first.  It is not part of the product: the package never loads it, and
// the product has no CPU fallback.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

using namespace faa;

namespace {

struct State {
    Prog prog;
    uint32_t hist[2][768];
    uint32_t tot[768];
    uint8_t lut[2][768];
    uint8_t lutc[768];
    HistPart parts[3][32];
    unsigned long long suml[2];
};

Ctx make_ctx(const uint8_t* raw, int H, int W, const State& st) {
    Ctx c; c.raw = raw; c.sraw = nullptr; c.s_lo = 0; c.s_len2 = 0; c.H = H; c.W = W;   // no staged band on the host
    c.op[0] = st.prog.op[0]; c.op[1] = st.prog.op[1]; c.box[0] = st.prog.box[0]; c.box[1] = st.prog.box[1];
    c.lut[0] = st.lut[0]; c.lut[1] = st.lut[1];
    return c;
}

template <int L>
void accumulate(const Ctx& c, int kind, uint32_t* hist, unsigned long long* suml) {
    for (int y = 0; y < c.H; ++y)
        for (int x = 0; x < c.W; ++x) {
            uint32_t p = Level<L>::at(c, x, y);
            if (kind == K_CONTRAST) *suml += luma_of(p);
            else { hist[p & 255u]++; hist[256 + ((p >> 8) & 255u)]++; hist[512 + (p >> 16)]++; }
        }
}

void build_lut(State& st, int j, int H, int W) {
    const OpRec o = st.prog.op[j];
    const int kind = o.kind;
    uint32_t mean = 0;
    if (kind_needs_hist(kind)) memcpy(st.tot, st.hist[j], sizeof st.tot);
    if (kind_needs_mean(kind)) mean = contrast_mean(st.suml[j], (uint32_t)H * (uint32_t)W);
    if (kind_needs_hist(kind)) {
        for (int t = 0; t < 96; ++t) st.parts[t >> 5][t & 31] = hist_part(&st.tot[(t >> 5) * 256], t & 31);
        for (int t = 0; t < 96; ++t)
            hist_lut_lane(kind, &st.tot[(t >> 5) * 256], st.parts[t >> 5], t & 31, (uint32_t)H * (uint32_t)W,
                          &st.lut[j][(t >> 5) * 256]);
    } else {
        for (int i = 0; i < 768; ++i) st.lut[j][i] = (uint8_t)lut_entry_static(o, (uint32_t)(i & 255), mean);
    }
}

void prepare(const uint8_t* raw, int H, int W, State& st) {
    const uint32_t stat_mask = st.prog.stat_mask, lut_mask = st.prog.lut_mask;
    if (lut_mask == 0) return;
    memset(st.hist, 0, sizeof st.hist);
    st.suml[0] = st.suml[1] = 0;
    const int k0 = st.prog.op[0].kind, k1 = st.prog.op[1].kind;
    const bool push = k0 != K_NONE && kind_is_lutlike(k0) && kind_needs_hist(k1);      // like the kernel
    Ctx c = make_ctx(raw, H, W, st);
    if (lut_mask & 1u) {
        if (kind_needs_hist(k0) || push) accumulate<0>(c, K_EQUALIZE, st.hist[0], &st.suml[0]);
        if (kind_needs_mean(k0)) accumulate<0>(c, K_CONTRAST, st.hist[0], &st.suml[0]);
        build_lut(st, 0, H, W);
    }
    if (lut_mask & 2u) {
        if (push) {
            // raw histogram pushed forward through the first LUT
            memset(st.hist[1], 0, sizeof st.hist[1]);
            for (int i = 0; i < 768; ++i) st.hist[1][(i & ~255) + st.lut[0][i]] += st.hist[0][i];
        } else if ((stat_mask >> 1) & 1u) {
            accumulate<1>(c, k1, st.hist[1], &st.suml[1]);
        }
        build_lut(st, 1, H, W);
    }
    if (st.prog.cls == C_LUT) {
        for (int i = 0; i < 768; ++i) {
            uint32_t v = (uint32_t)(i & 255), base = (uint32_t)(i & ~255);
            if (lut_mask & 1u) v = st.lut[0][base + v];
            if (lut_mask & 2u) v = st.lut[1][base + v];
            st.lutc[i] = (uint8_t)v;
        }
    }
}

struct TailInfo { int crop_dy, crop_dx, flip, zb0, zb1, zb2, zb3; };

TailInfo make_tail(const Prog& g, bool use_zero_box) {
    TailInfo t; t.crop_dy = g.crop_dy; t.crop_dx = g.crop_dx; t.flip = g.flip;
    t.zb0 = use_zero_box ? g.zero_box[0] : 0; t.zb1 = use_zero_box ? g.zero_box[1] : 0;
    t.zb2 = use_zero_box ? g.zero_box[2] : 0; t.zb3 = use_zero_box ? g.zero_box[3] : 0;
    return t;
}

uint32_t zero_mask(const TailInfo& t, int ox0, int oy) {
    if (oy < t.zb0 || oy >= t.zb1) return 0u;
    uint32_t m = 0;
    for (int k = 0; k < 4; ++k) m |= (uint32_t)(ox0 + k >= t.zb2 && ox0 + k < t.zb3) << k;
    return m;
}

void quad_vec(int cls, const Ctx& c, const uint8_t* lutc, const TailInfo& t, int out_w, int ox0, int oy, uint32_t px[4]) {
    const int sx0 = (t.flip ? (out_w - 4 - ox0) : ox0) + t.crop_dx;
    const int ay = oy + t.crop_dy;
    uint32_t q[4] = {0, 0, 0, 0};
    if ((unsigned)sx0 < (unsigned)c.W && (unsigned)ay < (unsigned)c.H) {
        const uint8_t* b = c.raw + (uint32_t)(ay * c.W + sx0) * 3u;
        if (cls == C_SHARP) {
            const uint32_t pitch = (uint32_t)c.W * 3u;
            const bool rowb = ay == 0 || ay == c.H - 1;
            sharp_quad(rowb ? b : b - pitch, b, rowb ? b : b + pitch, sx0 > 0, sx0 + 4 < c.W, rowb, sx0 == 0,
                       sx0 + 4 == c.W, bits_to_float(c.op[0].a[0]), c.op[0].a[1] != 0, q);
            for (int k = 0; k < 4; ++k) q[k] = apply_pointwise(c, 1, q[k], sx0 + k, ay);
        } else {
            uint32_t w[3]; memcpy(w, b, 12);
            q[0] = w[0] & 0xFFFFFFu;
            q[1] = (w[0] >> 24) | ((w[1] & 0xFFFFu) << 8);
            q[2] = (w[1] >> 16) | ((w[2] & 0xFFu) << 16);
            q[3] = w[2] >> 8;
            for (int k = 0; k < 4; ++k) {
                if (cls == C_LUT) q[k] = apply_lut(lutc, q[k]);
                else if (cls == C_POINT) q[k] = apply_pointwise(c, 1, apply_pointwise(c, 0, q[k], sx0 + k, ay), sx0 + k, ay);
            }
        }
    }
    for (int k = 0; k < 4; ++k) px[k] = t.flip ? q[3 - k] : q[k];
}

void quad_generic(const Ctx& c, const TailInfo& t, int out_w, int ox0, int oy, uint32_t px[4]) {
    const int ay = oy + t.crop_dy;
    for (int k = 0; k < 4; ++k) {
        const int ox = ox0 + k;
        px[k] = 0u;
        const int ax = (t.flip ? (out_w - 1 - ox) : ox) + t.crop_dx;
        if (ox < out_w && (unsigned)ax < (unsigned)c.W && (unsigned)ay < (unsigned)c.H) px[k] = Level<2>::at(c, ax, ay);
    }
}

}  // namespace

extern "C" {

// ops: compiled table [n_sub][n_op][2] (32-byte records); samples/boxes indexed like the kernel's.
// norm_tab == NULL -> uint8 HWC output, else fp32 NCHW through the exact table.
// force_generic != 0 evaluates every image through the generic class (to test both paths).
int faa_emu_augment(const uint8_t* in, int n_all, int first, int B, int H, int W, const void* ops_v, int n_sub,
                    int n_op, const void* samples_v, const void* boxes_v, int op_base, int apply_tail, int out_h,
                    int out_w, int use_zero_box, const float* norm_tab, void* out, const int32_t* partner,
                    float lam, float oml, int force_generic) {
    (void)n_sub; (void)n_all;
    const OpRec* ops = (const OpRec*)ops_v;
    const Sample* samples = (const Sample*)samples_v;
    const Box* boxes = (const Box*)boxes_v;
    const int nsrc = partner ? 2 : 1;
    std::vector<State> st(2);
    std::vector<std::vector<uint8_t>> l1(2);
    const size_t img_bytes = (size_t)H * W * 3;
    const bool zb = use_zero_box && apply_tail;
    for (int img = 0; img < B; ++img) {
        int src[2] = {first + img, partner ? partner[img] : 0};
        Ctx c[2]; TailInfo t[2]; int cls[2];
        for (int k = 0; k < nsrc; ++k) {
            // force_generic: no materialisation / vector classes (the kernel's mixup launches and fallbacks)
            build_prog(samples[src[k]], boxes + (size_t)src[k] * n_op, ops, n_op, op_base, apply_tail, H, W, out_w,
                       (force_generic || partner) ? 0 : 3, st[k].prog);
            if (force_generic) st[k].prog.cls = C_GENERIC;
            const uint8_t* raw = in + img_bytes * src[k];
            t[k] = make_tail(st[k].prog, zb);
            if (st[k].prog.cls == C_MAT) {
                // like run_materialised(): op0's LUT, op0's output as an image, op1 as a single-op program on it
                State& S = st[k];
                memset(S.hist, 0, sizeof S.hist); S.suml[0] = S.suml[1] = 0;
                Ctx c0 = make_ctx(raw, H, W, S);
                if (S.prog.lut_mask & 1u) {
                    if (S.prog.stat_mask & 1u) accumulate<0>(c0, S.prog.op[0].kind, S.hist[0], &S.suml[0]);
                    build_lut(S, 0, H, W);
                }
                l1[k].resize(img_bytes);
                for (int y = 0; y < H; ++y)
                    for (int x = 0; x < W; ++x) {
                        uint32_t p = Level<1>::at(c0, x, y);
                        uint8_t* o = &l1[k][((size_t)y * W + x) * 3];
                        o[0] = (uint8_t)p; o[1] = (uint8_t)(p >> 8); o[2] = (uint8_t)(p >> 16);
                    }
                Ctx c2 = make_ctx(l1[k].data(), H, W, S);
                c2.op[0] = S.prog.op[1]; c2.box[0] = S.prog.box[1]; c2.op[1].kind = K_NONE;
                c2.lut[0] = S.lut[1]; c2.lut[1] = S.lut[1];
                const int k1 = S.prog.op[1].kind;
                if (kind_needs_hist(k1) || kind_needs_mean(k1)) {
                    accumulate<0>(c2, k1, S.hist[1], &S.suml[1]);
                    build_lut(S, 1, H, W);
                    memcpy(S.lutc, S.lut[1], 768);
                }
                c[k] = c2;
                cls[k] = S.prog.cls2;
            } else {
                prepare(raw, H, W, st[k]);
                c[k] = make_ctx(raw, H, W, st[k]);
                cls[k] = st[k].prog.cls;
            }
        }
        for (int oy = 0; oy < out_h; ++oy)
            for (int ox0 = 0; ox0 < out_w; ox0 += 4) {
                uint32_t px[2][4], zm[2] = {0, 0};
                for (int k = 0; k < nsrc; ++k) {
                    if (cls[k] == C_GENERIC || cls[k] == C_GEOM || cls[k] == C_SG) quad_generic(c[k], t[k], out_w, ox0, oy, px[k]);
                    else quad_vec(cls[k], c[k], st[k].lutc, t[k], out_w, ox0, oy, px[k]);
                    zm[k] = zero_mask(t[k], ox0, oy);
                }
                const int nvalid = (out_w - ox0) < 4 ? (out_w - ox0) : 4;
                for (int k = 0; k < nvalid; ++k) {
                    if (!norm_tab) {
                        uint32_t p = ((zm[0] >> k) & 1u) ? 0u : px[0][k];
                        uint8_t* o = (uint8_t*)out + (((size_t)img * out_h + oy) * out_w + ox0 + k) * 3;
                        o[0] = (uint8_t)p; o[1] = (uint8_t)(p >> 8); o[2] = (uint8_t)(p >> 16);
                    } else {
                        for (int ch = 0; ch < 3; ++ch) {
                            float a = ((zm[0] >> k) & 1u) ? 0.0f : norm_tab[ch * 256 + ((px[0][k] >> (8 * ch)) & 255u)];
                            if (nsrc == 2) {
                                float b = ((zm[1] >> k) & 1u) ? 0.0f : norm_tab[ch * 256 + ((px[1][k] >> (8 * ch)) & 255u)];
                                a = f_add(f_mul(a, lam), f_mul(b, oml));
                            }
                            ((float*)out)[(((size_t)img * 3 + ch) * out_h + oy) * out_w + ox0 + k] = a;
                        }
                    }
                }
            }
    }
    return 0;
}

// class histogram of a batch (which final-pass specialisation each image takes)
int faa_emu_classes(const void* ops_v, int n_op, const void* samples_v, const void* boxes_v, int B, int H, int W,
                    int out_w, int apply_tail, uint8_t* cls_out) {
    const OpRec* ops = (const OpRec*)ops_v;
    const Sample* samples = (const Sample*)samples_v;
    const Box* boxes = (const Box*)boxes_v;
    for (int i = 0; i < B; ++i) {
        Prog g;
        build_prog(samples[i], boxes + (size_t)i * n_op, ops, n_op, 0, apply_tail, H, W, out_w, 3, g);
        cls_out[i] = g.cls;
    }
    return 0;
}

// weight class of every image's program in a three-way split launch (faa_resolve_kernel): 2 light, 1 mid, 0 heavy.
// `allow`: bit 0 materialisation chunk, bit 1 scratch image, bit 2 lean octet gathers (plan_launch sets 7 for the
// headline geometry and then does NOT launch the cluster kernel: no program may be heavy)
int faa_emu_weight_classes(const void* ops_v, int n_op, const void* samples_v, const void* boxes_v, int B, int H, int W,
                           int out_w, int apply_tail, int allow, uint8_t* wc_out, uint8_t* cls_out) {
    const OpRec* ops = (const OpRec*)ops_v;
    const Sample* samples = (const Sample*)samples_v;
    const Box* boxes = (const Box*)boxes_v;
    for (int i = 0; i < B; ++i) {
        Prog g;
        build_prog(samples[i], boxes + (size_t)i * n_op, ops, n_op, 0, apply_tail, H, W, out_w, allow, g);
        wc_out[i] = prog_is_light(g) ? 2 : prog_is_mid(g, allow) ? 1 : 0;
        if (cls_out) cls_out[i] = g.cls;
    }
    return 0;
}

int faa_emu_philox(const void* ops_v, const double* probs, int n_sub, int n_op, const void* rng_v, int B, int H,
                   int W, int out_h, int out_w, void* samples_v, void* boxes_v) {
    const OpRec* ops = (const OpRec*)ops_v;
    RngCfg r; memcpy(&r, rng_v, sizeof r);
    Sample* samples = (Sample*)samples_v;
    Box* boxes = (Box*)boxes_v;
    for (int i = 0; i < B; ++i) {
        Box bx[8];
        philox_sample(r, r.first_index + (uint64_t)i, ops, probs, n_sub, n_op, H, W, out_h, out_w, samples[i], bx);
        for (int j = 0; j < n_op; ++j) boxes[(size_t)i * n_op + j] = bx[j];
    }
    return 0;
}

// The launch planner's decisions (plan_launch) as int32 values, in the order faa_emu_plan_fields names them; returns
// their count.  split_min < 0: the library's default.
const char* faa_emu_plan_fields() {
    return "bands band_cap stage light_bands light_staged octets mat_cap use_order use_split use_mid split mid_bands "
           "mid_threads allow scratch no_heavy self_resolving use_chain speculate light_cap";
}

int faa_emu_plan(int H, int W, int out_h, int out_w, int batch, int crop_pad, int out_u8, int in_mod16, int out_mod16,
                 int two_src, int apply_tail, int has_sg, long long split_min, int philox, int allow_ahead, int32_t* out) {
    const LaunchPlan L = plan_launch({H, W, out_h, out_w, batch, crop_pad, out_u8 != 0, (uint32_t)in_mod16,
                                      (uint32_t)out_mod16, two_src != 0, apply_tail != 0, has_sg != 0,
                                      split_min < 0 ? kSplitMin : (uint64_t)split_min, philox != 0, allow_ahead != 0});
    const int32_t v[] = {L.geo[0].bands, L.geo[0].band_cap, L.stage, L.geo[1].bands, L.geo[1].band_cap > 0, L.octets,
                         L.mat_cap, L.use_order, L.use_split, L.use_mid, L.split, L.mid.bands, L.mid_threads, L.allow,
                         L.scratch, L.no_heavy, L.self_resolving, L.use_chain, L.speculate, L.geo[1].band_cap};
    memcpy(out, v, sizeof v);
    return (int)(sizeof v / sizeof v[0]);
}

// raw Philox4x32-10 block, for the known-answer test
void faa_emu_philox_block(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    U4 c; c.x = ctr[0]; c.y = ctr[1]; c.z = ctr[2]; c.w = ctr[3];
    U4 r = philox4x32_10(c, key[0], key[1]);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

}  // extern "C"
