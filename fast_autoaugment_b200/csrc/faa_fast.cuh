// faa_fast.cuh - lean final passes of the light (streaming) kernel for the common launch geometry:
// W % 8 == 0, output size == image size, no crop (P.octets, TailInfo without crop).  Included by
// faa_kernels.cu behind the generic evaluators; every routine here has a generic counterpart there that
// is used whenever its preconditions do not hold, and the GPU parity tests run both.
//
//   row-shift gathers   TranslateX/Y(+Abs) and ShearX move whole rows: an output octet (8 pixels) is 24
//                       contiguous source bytes at an arbitrary byte offset -> seven aligned words and six
//                       funnel shifts, then the same 16-byte plane stores as the streaming loop
//                       (augmentations.py:13-17,27-54 through Pillow's affine_fixed / ImagingScaleAffine)
//   lean affine gather  ShearY / Rotate (augmentations.py:20-24,57-61): four source pixels per thread from
//                       global memory (L1), no staged-copy test, no branches between the loads
//   Color               ImageEnhance.Color (augmentations.py:102-104) with the fp32 blend kept on the FMA
//                       pipe: byte -> float through the 1.5*2^23 bias trick, truncation through a
//                       round-toward-zero add, no I2F / F2I (the conversion unit runs at a fraction of the FMA rate)
//   Cutout              the streaming loop plus a box test per octet (augmentations.py:126-144)
// A per-channel LUT in the program's other slot rides for free: the float table already composes
// LUT o ToTensor o Normalize; only the fill colour depends on the order of the two ops.
#pragma once

namespace faa {

// (kBias15 = 1.5 * 2^23 and kBias15Bits: faa_kernels.cu, next to the uint8 output helpers)

// byte j (0..3) of w as the float (kBias15 + byte): one PRMT, no conversion instruction
__device__ __forceinline__ float biased_byte(uint32_t w, int j) {
    return __uint_as_float(__byte_perm(w, kBias15Bits, 0x7650 + j));      // selector: [7][6][5][j] -> 0x4B40 00 bb
}

// ---------------------------------------------------------------------------------------------------
// masked emit: pixels whose bit in `valid` is clear take the fill value pad[ch] (already normalised)
template <int OUT, bool USE_TAB>
__device__ __forceinline__ void emit_oct_masked(const AugParams& P, const float* tab, typename OutElem<OUT>::T* o,
                                                uint32_t plane, const uint32_t px[8], uint32_t valid, const float pad[3]) {
    if constexpr (OUT == OUT_U8_HWC) {
        uint32_t ob[24];
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const uint32_t u = (px[k] >> (8 * ch)) & 255u;
                const uint32_t b = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
                ob[3 * k + ch] = ((valid >> k) & 1u) ? b : f2b(pad[ch]);
            }
        store_oct_u8(o, ob);
        return;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        uint32_t u[8]; float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) u[k] = (px[k] >> (8 * ch)) & 255u;
        norm8<USE_TAB>(P, tab, ch, u, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = ((valid >> k) & 1u) ? v[k] : pad[ch];
        store_plane8<OUT>(o + ch * plane, v);
    }
}

template <int OUT>
__device__ __forceinline__ void fill_oct(typename OutElem<OUT>::T* o, uint32_t plane, const float pad[3]) {
    if constexpr (OUT == OUT_U8_HWC) {
        uint32_t ob[24];
#pragma unroll
        for (int k = 0; k < 24; ++k) ob[k] = f2b(pad[k % 3]);
        store_oct_u8(o, ob);
        return;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float v[8] = {pad[ch], pad[ch], pad[ch], pad[ch], pad[ch], pad[ch], pad[ch], pad[ch]};
        store_plane8<OUT>(o + ch * plane, v);
    }
}

// ---------------------------------------------------------------------------------------------------
// Row-shift geometric ops.  K_SHIFT: source = (x + dx + (x >= bx), y + dy + (y >= by)); K_AFFINE with
// a0 == a4 == 1.0 and a3 == 0 (ShearX): source = (x + ((a2 + a1*y) >> 16), y) - exact, because the x term
// of Pillow's fixed-point sum has no fractional bits.
struct RowShift {
    int dx, bx, dy, by;       // K_SHIFT
    int a1, a2;               // ShearX
    int shear;
};

__device__ __forceinline__ bool rowshift_of(const OpRec& r, RowShift& rs) {
    rs.dx = rs.dy = 0; rs.bx = rs.by = 0x7fffffff; rs.a1 = rs.a2 = 0; rs.shear = 0;
    if (r.kind == K_SHIFT) { rs.dx = r.a[0]; rs.dy = r.a[1]; rs.bx = r.a[2]; rs.by = r.a[3]; return true; }
    if (r.kind == K_AFFINE && r.a[0] == 65536 && r.a[3] == 0 && r.a[4] == 65536) {
        rs.shear = 1; rs.a1 = r.a[1]; rs.a2 = r.a[2]; return true;
    }
    return false;
}

// USE_TAB: value = tab[ch][byte] (LUT partner composed with the normalisation, or the exact table);
// pad[ch]: the normalised fill value for pixels whose source is outside the image
template <int OUT, bool USE_TAB, bool FLIP>
__device__ __forceinline__ void final_rows_rowshift(const AugParams& P, const float* tab, const float pad[3], const Ctx& c,
                                                    const RowShift rs, void* out_img, int oy0, int oy1) {
    constexpr int flip = FLIP ? 1 : 0;
    using T = typename OutElem<OUT>::T;
    const int W = P.W, H = P.H;
    const uint32_t opr = (uint32_t)W >> 3;
    const uint32_t n8 = (uint32_t)(oy1 - oy0) * opr;
    const uint32_t plane = (uint32_t)H * (uint32_t)W, pitch = (uint32_t)W * 3u;
    const uint32_t s_len = c.s_len2 ? c.s_len2 + 2u : 0u;
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)W;
    FastDiv dq; dq.init(opr, P.rcp_opr);
    uint32_t r = dq.div(threadIdx.x), ox = threadIdx.x - r * opr;
    const uint32_t dr = dq.div(blockDim.x), dxo = blockDim.x - dr * opr;
    for (uint32_t i = threadIdx.x; i < n8; i += blockDim.x) {
        const int y = oy0 + (int)r;
        const int ax0 = flip ? W - 8 - (int)ox * 8 : (int)ox * 8;        // first column of the octet in the augmented image
        const int ys = rs.shear ? y : y + rs.dy + (y >= rs.by);
        const int s0 = rs.shear ? (rs.a2 + rs.a1 * y) >> 16 : rs.dx + (ax0 >= rs.bx);
        const int s7 = rs.shear ? s0 : rs.dx + (ax0 + 7 >= rs.bx);
        const int sx0 = ax0 + s0;
        T* o = dst + PS * 8u * i;
        if ((unsigned)ys >= (unsigned)H || sx0 + 7 + (s7 - s0) < 0 || sx0 >= W) {
            fill_oct<OUT>(o, plane, pad);                                 // nothing of the octet has a source
        } else if (s0 == s7) {
            // One shift for the whole octet: its sources are 24 contiguous bytes from byte B0 of the image.  At a
            // row edge only pixels [lo, hi) of the octet have a source; the aligned words are always clamped into the
            // source row (valid memory, ignored bytes), and warps that hold an edge octet patch the missing pixels
            // with the fill value after the normalisation - full and edge octets share one instruction stream.
            const int lo = max(0, -sx0), hi = min(8, W - sx0);
            uint32_t vmask = (0xFFu >> (8 - hi)) & (0xFFu << lo) & 0xFFu;
            if (flip) vmask = __brev(vmask) >> 24;
            const int row_lo = ys * (int)pitch, row_hi = row_lo + (int)pitch - 4;
            const int B0 = row_lo + sx0 * 3, A = B0 & ~3;
            const uint32_t k = (uint32_t)B0 & 3u;
            const bool staged = (uint32_t)row_lo - c.s_lo <= s_len - pitch && s_len >= pitch;      // the whole source row
            uint32_t v[7];
            if (staged) {
#pragma unroll
                for (int j = 0; j < 7; ++j)
                    v[j] = *reinterpret_cast<const uint32_t*>(c.sraw + ((uint32_t)min(max(A + 4 * j, row_lo), row_hi) - c.s_lo));
            } else {
#pragma unroll
                for (int j = 0; j < 7; ++j) v[j] = __ldg(reinterpret_cast<const uint32_t*>(c.raw + min(max(A + 4 * j, row_lo), row_hi)));
            }
            uint32_t w[6];
#pragma unroll
            for (int j = 0; j < 6; ++j) w[j] = __funnelshift_r(v[j], v[j + 1], 8u * k);
            const bool patch = __any_sync(__activemask(), vmask != 0xFFu);
            if constexpr (OUT == OUT_U8_HWC) {
                uint32_t ob[24];
#pragma unroll
                for (int kk = 0; kk < 8; ++kk)                           // output pixel kk = source pixel (FLIP ? 7 - kk : kk)
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        const int bi = 3 * (FLIP ? 7 - kk : kk) + ch;
                        const uint32_t u = (w[bi >> 2] >> (8 * (bi & 3))) & 255u;
                        const uint32_t b = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
                        ob[3 * kk + ch] = ((vmask >> kk) & 1u) ? b : f2b(pad[ch]);
                    }
                store_oct_u8(o, ob);
            } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                uint32_t u[8]; float nv[8];
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) {
                    const int bi = 3 * kk + ch;                          // byte of source pixel kk
                    u[kk] = (w[bi >> 2] >> (8 * (bi & 3))) & 255u;
                }
                float fv[8];
                norm8<USE_TAB>(P, tab, ch, u, fv);
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) nv[kk] = fv[FLIP ? 7 - kk : kk];
                if (patch) {
#pragma unroll
                    for (int kk = 0; kk < 8; ++kk) nv[kk] = ((vmask >> kk) & 1u) ? nv[kk] : pad[ch];
                }
                store_plane8<OUT>(o + ch * plane, nv);
            }
            }
        } else {
            // a shift break (Pillow's accumulated float offset) inside the octet: per pixel
            uint32_t px[8]; uint32_t valid = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int x = flip ? ax0 + 7 - j : ax0 + j;              // output pixel j of the octet
                const int xs = x + rs.dx + (x >= rs.bx);
                const bool ok = (unsigned)xs < (unsigned)W;
                px[j] = ok ? load_raw(c, xs, ys) : 0u;
                valid |= (uint32_t)ok << j;
            }
            emit_oct_masked<OUT, USE_TAB>(P, tab, o, plane, px, valid, pad);
        }
        ox += dxo; r += dr;
        if (ox >= opr) { ox -= opr; ++r; }
    }
}

// ---------------------------------------------------------------------------------------------------
// General gather (ShearY, Rotate; two geometric ops).  Sources come from global memory (L1): a rotated band has no compact
// source footprint.  To keep the gather coalesced each warp works on a tile of 128 consecutive output pixels in two
// phases: (1) lane l fetches pixels l, l+32, l+64, l+96 of the tile - neighbouring lanes read neighbouring source
// pixels, two aligned word loads and a funnel shift each - into a shared-memory tile; (2) lane l normalises pixels
// 4l..4l+3 and writes 8-byte plane quads.  `tile`: 128 words per warp.
// one nearest-neighbour coordinate map (Pillow affine_fixed / unit-scale ImagingScaleAffine, faa_core.cuh Level::at)
// with its six parameters in registers: K_AFFINE 16.16 coefficients, or K_SHIFT dx, dy, bx, by in a0..a3
struct MapRegs { int aff, a0, a1, a2, a3, a4, a5; };
__device__ __forceinline__ MapRegs map_regs(const OpRec& o) {
    MapRegs m; m.aff = o.kind == K_AFFINE; m.a0 = o.a[0]; m.a1 = o.a[1]; m.a2 = o.a[2]; m.a3 = o.a[3]; m.a4 = o.a[4]; m.a5 = o.a[5];
    return m;
}
__device__ __forceinline__ bool map_xy(const MapRegs& m, int& x, int& y, int W, int H) {
    int xin, yin;
    if (m.aff) { xin = (m.a2 + m.a0 * x + m.a1 * y) >> 16; yin = (m.a5 + m.a3 * x + m.a4 * y) >> 16; }
    else { xin = x + m.a0 + (x >= m.a2); yin = y + m.a1 + (y >= m.a3); }
    x = xin; y = yin;
    return (unsigned)xin < (unsigned)W && (unsigned)yin < (unsigned)H;
}

// one source pixel (24 bits) of the gather, bit 24 set when it exists.  mA maps the output pixel into the image in
// front of the last op; opB (shared memory, may be null: CTA-uniform) maps that position into the image in front of it.
// cut (shared memory, may be null: CTA-uniform): the clipped box of a Cutout in front of the gather.
template <bool COH = false>   // COH: the source image was written by this kernel (scratch, behind a cluster barrier): loads bypass L1
__device__ __forceinline__ uint32_t gather_fetch(const uint8_t* raw, int W, int H, const MapRegs& mA, const OpRec* opB, int x, int y,
                                                 const Box* cut = nullptr) {
    bool ok = map_xy(mA, x, y, W, H);
    if (opB != nullptr) { const MapRegs mB = map_regs(*opB); const bool ok2 = map_xy(mB, x, y, W, H); ok = ok && ok2; }
    const uint32_t off = ok ? (uint32_t)(y * W + x) * 3u : 0u;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(raw + (off & ~3u));
    const uint32_t lo = COH ? __ldcg(wp) : __ldg(wp);
    const uint32_t hi = (off & 2u) ? (COH ? __ldcg(wp + 1) : __ldg(wp + 1)) : 0u;     // bytes 2,3 of the word: the pixel spills into the next one
    uint32_t px = __funnelshift_r(lo, hi, 8u * (off & 3u)) & 0xFFFFFFu;
    if (cut != nullptr && x >= cut->x0 && x <= cut->x1 && y >= cut->y0 && y <= cut->y1) px = kCutoutRGB;
    return ok ? (px | 0x01000000u) : 0u;
}

template <int OUT, bool USE_TAB, bool FULL, bool COH = false>
__device__ __forceinline__ void final_rows_gather_t(const AugParams& P, const float* tab, const float pad[3], const Ctx& c,
                                                    const OpRec* opA, const OpRec* opB, int flip, void* out_img, int oy0, int oy1,
                                                    uint32_t* tile, const Box* cut) {
    using T = typename OutElem<OUT>::T;
    const int W = P.W, H = P.H;
    const uint32_t npx = (uint32_t)(oy1 - oy0) * (uint32_t)W;
    const uint32_t plane = (uint32_t)H * (uint32_t)W;
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)W;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    uint32_t* my = tile + warp * 128u;
    const uint8_t* raw = c.raw;
    const MapRegs mA = map_regs(*opA);
    FastDiv dw; dw.init((uint32_t)W, P.rcp_w);
    for (uint32_t base = warp * 128u; base < npx; base += nwarp * 128u) {
        if (W >= 32) {                                                   // one division per tile, then x += 32 with at most one wrap
            const uint32_t p = base + lane;
            const uint32_t r = dw.div(p);
            int x = (int)(p - r * (uint32_t)W), y = oy0 + (int)r;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                uint32_t v = 0u;
                if (FULL || p + 32u * (uint32_t)i < npx) v = gather_fetch<COH>(raw, W, H, mA, opB, flip ? W - 1 - x : x, y, cut);
                my[lane + 32u * (uint32_t)i] = v;
                x += 32;
                if (x >= W) { x -= W; ++y; }
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t p = base + lane + 32u * (uint32_t)i;
                uint32_t v = 0u;
                if (p < npx) {
                    const uint32_t r = dw.div(p);
                    const int x = (int)(p - r * (uint32_t)W);
                    v = gather_fetch<COH>(raw, W, H, mA, opB, flip ? W - 1 - x : x, oy0 + (int)r, cut);
                }
                my[lane + 32u * (uint32_t)i] = v;
            }
        }
        __syncwarp();
        const uint32_t p0 = base + 4u * lane;
        if (FULL || p0 < npx) {
            const uint4 q4 = reinterpret_cast<const uint4*>(my)[lane];
            const uint32_t px[4] = {q4.x, q4.y, q4.z, q4.w};
            const bool patch = __any_sync(__activemask(), ((q4.x & q4.y & q4.z & q4.w) >> 24) == 0u);
            T* o = dst + PS * p0;
            if constexpr (OUT == OUT_U8_HWC) {
                uint32_t ob[12];
#pragma unroll
                for (int k = 0; k < 4; ++k)
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        const uint32_t u = (px[k] >> (8 * ch)) & 255u;
                        const uint32_t b = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
                        ob[3 * k + ch] = (px[k] >> 24) ? b : f2b(pad[ch]);
                    }
                store_quad_u8(o, ob);
            } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float v[4];
                if (USE_TAB) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) v[k] = tab[ch * 256 + ((px[k] >> (8 * ch)) & 255u)];
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k) v[k] = __fmaf_rn((float)((px[k] >> (8 * ch)) & 255u), P.scale[ch], P.bias[ch]);
                }
                if (patch) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) v[k] = (px[k] >> 24) ? v[k] : pad[ch];
                }
                store_plane4<OUT>(o + ch * plane, v, true, 4);
            }
            }
        }
        __syncwarp();
    }
}

// rows [ra, rb) of a gathered image, materialised as uint8 HWC at `dst` (shared memory, byte 0 = pixel (0, ra)):
// the same two-phase tile walk as the final pass, the quads are packed back into 12 bytes
__device__ __forceinline__ void gather_rows_to_band(const AugParams& P, const uint8_t* raw, const OpRec* opA, uint8_t* dst,
                                                    int ra, int rb, uint32_t* tile) {
    const int W = P.W, H = P.H;
    const uint32_t npx = (uint32_t)(rb - ra) * (uint32_t)W;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    uint32_t* my = tile + warp * 128u;
    const MapRegs mA = map_regs(*opA);
    FastDiv dw; dw.init((uint32_t)W, P.rcp_w);
    for (uint32_t base = warp * 128u; base < npx; base += nwarp * 128u) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t p = base + lane + 32u * (uint32_t)i;
            uint32_t v = 0u;
            if (p < npx) {
                const uint32_t r = dw.div(p);
                v = gather_fetch(raw, W, H, mA, nullptr, (int)(p - r * (uint32_t)W), ra + (int)r) & 0xFFFFFFu;
            }
            my[lane + 32u * (uint32_t)i] = v;
        }
        __syncwarp();
        const uint32_t p0 = base + 4u * lane;
        if (p0 < npx) {
            const uint4 q = reinterpret_cast<const uint4*>(my)[lane];
            uint32_t* w = reinterpret_cast<uint32_t*>(dst + 3u * p0);
            w[0] = q.x | (q.y << 24);
            w[1] = (q.y >> 8) | (q.z << 16);
            w[2] = (q.z >> 16) | (q.w << 8);
        }
        __syncwarp();
    }
}

template <int OUT, bool USE_TAB>
__device__ __forceinline__ void final_rows_gather(const AugParams& P, const float* tab, const float pad[3], const Ctx& c,
                                                  const OpRec* opA, const OpRec* opB, int flip, void* out_img, int oy0, int oy1,
                                                  uint32_t* tile, const Box* cut = nullptr) {
    const uint32_t npx = (uint32_t)(oy1 - oy0) * (uint32_t)P.W;
    if ((npx & 127u) == 0u) final_rows_gather_t<OUT, USE_TAB, true>(P, tab, pad, c, opA, opB, flip, out_img, oy0, oy1, tile, cut);
    else final_rows_gather_t<OUT, USE_TAB, false>(P, tab, pad, c, opA, opB, flip, out_img, oy0, oy1, tile, cut);
}

// the gather reads an image this kernel wrote (c.raw = scratch): coherent loads
template <int OUT, bool USE_TAB>
__device__ __forceinline__ void final_rows_gather_coh(const AugParams& P, const float* tab, const float pad[3], const Ctx& c,
                                                      const OpRec* opA, int flip, void* out_img, int oy0, int oy1, uint32_t* tile) {
    final_rows_gather_t<OUT, USE_TAB, false, true>(P, tab, pad, c, opA, nullptr, flip, out_img, oy0, oy1, tile, nullptr);
}

// ---------------------------------------------------------------------------------------------------
// ImageEnhance.Color alone: out = blend(luma, px, alpha) per channel, then ToTensor + Normalize.
// The blend (Pillow Blend.c: fp32, separate multiply and add, truncation, clip when alpha is outside
// [0,1]) is evaluated on biased floats: fb = kBias15 + byte (exact), px - luma = fb_px - fb_l (exact),
// t = l + alpha * (px - l) with the reference's two roundings, trunc(t) = (t +rz kBias15) - kBias15 for
// t >= 0 and anything below zero clamps to zero either way.
template <int OUT, bool TAB, bool CLIP>
__device__ __forceinline__ void final_rows_color(const AugParams& P, const float* s_norm, const Ctx& c, float alpha, int flip,
                                                 void* out_img, int oy0, int oy1) {
    using T = typename OutElem<OUT>::T;
    const int W = P.W;
    const uint32_t opr = (uint32_t)W >> 3;
    const uint32_t n8 = (uint32_t)(oy1 - oy0) * opr;
    const uint32_t plane = (uint32_t)P.H * (uint32_t)W;
    const uint8_t* src = c.sraw + ((uint32_t)oy0 * (uint32_t)W * 3u - c.s_lo);
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)W;
    FastDiv dq; dq.init(opr, P.rcp_opr);
    uint32_t r = dq.div(threadIdx.x), ox = threadIdx.x - r * opr;
    const uint32_t dr = dq.div(blockDim.x), dxo = blockDim.x - dr * opr;
    for (uint32_t i = threadIdx.x; i < n8; i += blockDim.x) {
        const uint32_t sox = flip ? opr - 1u - ox : ox;
        const uint2* s8 = reinterpret_cast<const uint2*>(src + 24u * (r * opr + sox));
        const uint2 wa = s8[0], wb = s8[1], wc = s8[2];
        const uint32_t w[6] = {wa.x, wa.y, wb.x, wb.y, wc.x, wc.y};
        float v[3][8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int sk = flip ? 7 - k : k;                              // source pixel of output pixel k
            float fb[3]; uint32_t u[3];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const int bidx = 3 * sk + ch;
                fb[ch] = biased_byte(w[bidx >> 2], bidx & 3);
                u[ch] = (w[bidx >> 2] >> (8 * (bidx & 3))) & 255u;
            }
            const uint32_t l = (19595u * u[0] + 38470u * u[1] + 7471u * u[2] + 0x8000u) >> 16;      // Pillow rgb2l
            const float fl = __uint_as_float(kBias15Bits + l);           // kBias15 + l
            const float lf = __fadd_rn(fl, -kBias15);                    // (float)l
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float d = __fadd_rn(fb[ch], -fl);                  // (float)(px - l), exact
                const float t = __fadd_rn(lf, __fmul_rn(alpha, d));      // Blend.c, no contraction
                float z = __fadd_rz(t, kBias15);                         // kBias15 + floor(t)
                if (CLIP) z = fminf(fmaxf(z, kBias15), kBias15 + 255.0f);
                v[ch][k] = __fadd_rn(z, -kBias15);                       // the byte value as a float, exact
            }
        }
        T* o = dst + PS * 8u * i;
        if constexpr (OUT == OUT_U8_HWC) {
            uint32_t ob[24];
#pragma unroll
            for (int k = 0; k < 8; ++k)
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) ob[3 * k + ch] = TAB ? f2b(s_norm[ch * 256 + (int)v[ch][k]]) : f2b(v[ch][k]);
            store_oct_u8(o, ob);
        } else {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float nv[8];
            if (TAB) {
#pragma unroll
                for (int k = 0; k < 8; ++k) nv[k] = s_norm[ch * 256 + (int)v[ch][k]];
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) nv[k] = __fmaf_rn(v[ch][k], P.scale[ch], P.bias[ch]);
            }
            store_plane8<OUT>(o + ch * plane, nv);
        }
        }
        ox += dxo; r += dr;
        if (ox >= opr) { ox -= opr; ++r; }
    }
}

// ---------------------------------------------------------------------------------------------------
// Cutout alone: the streaming loop, except for octets that touch the (clipped, inclusive) box
template <int OUT, bool TAB>
__device__ __forceinline__ void final_rows_cutout(const AugParams& P, const float* s_norm, const Ctx& c, const Box bx, int flip,
                                                  void* out_img, int oy0, int oy1) {
    using T = typename OutElem<OUT>::T;
    const int W = P.W;
    const uint32_t opr = (uint32_t)W >> 3;
    const uint32_t n8 = (uint32_t)(oy1 - oy0) * opr;
    const uint32_t plane = (uint32_t)P.H * (uint32_t)W;
    const uint8_t* src = c.sraw + ((uint32_t)oy0 * (uint32_t)W * 3u - c.s_lo);
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)W;
    FastDiv dq; dq.init(opr, P.rcp_opr);
    uint32_t r = dq.div(threadIdx.x), ox = threadIdx.x - r * opr;
    const uint32_t dr = dq.div(blockDim.x), dxo = blockDim.x - dr * opr;
    for (uint32_t i = threadIdx.x; i < n8; i += blockDim.x) {
        const int y = oy0 + (int)r;
        const uint32_t sox = flip ? opr - 1u - ox : ox;
        const int sx0 = (int)sox * 8;                                     // first source column of the octet
        const uint2* s8 = reinterpret_cast<const uint2*>(src + 24u * (r * opr + sox));
        const uint2 wa = s8[0], wb = s8[1], wc = s8[2];
        const uint32_t w[6] = {wa.x, wa.y, wb.x, wb.y, wc.x, wc.y};
        T* o = dst + PS * 8u * i;
        if (y < bx.y0 || y > bx.y1 || sx0 + 7 < bx.x0 || sx0 > bx.x1) {
            if (flip) stream_oct<OUT, TAB, true>(P, w, s_norm, o, plane);
            else stream_oct<OUT, TAB, false>(P, w, s_norm, o, plane);
        } else {
            uint32_t q[8], px[8];
            unpack12(w[0], w[1], w[2], q); unpack12(w[3], w[4], w[5], q + 4);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int sk = flip ? 7 - k : k;
                const int x = sx0 + sk;
                px[k] = (x >= bx.x0 && x <= bx.x1) ? kCutoutRGB : q[sk];
            }
            emit_oct<OUT, TAB>(P, s_norm, o, plane, px);
        }
        ox += dxo; r += dr;
        if (ox >= opr) { ox -= opr; ++r; }
    }
}

// ---------------------------------------------------------------------------------------------------
// Sharpness (ImageEnhance.Sharpness = blend(img.filter(SMOOTH), img, alpha), augmentations.py:112-114) as a
// filter on the BYTE STREAM: with interleaved RGB the horizontal neighbours of byte k are bytes k-3 and k+3, so
// the 3x3 SMOOTH sum needs no channel bookkeeping:
//     col[k] = a[k] + b[k] + c[k]                    (rows y-1, y, y+1)
//     S[k]   = col[k-3] + col[k] + col[k+3] + 4 b[k]   ([1 1 1; 1 5 1; 1 1 1])
//     deg[k] = (2 S[k] + 13) / 26                     (/13, rounded half up)
// Bytes travel as 16-bit lanes, two per register, in stream order: a 3-byte shift of the stream is ONE PRMT.
// The division and the fp32 blend run on the FMA pipe (biased floats, see final_rows_color); no I2F / F2I.
// One quad (12 output bytes) per thread and iteration; `tab` as in the streaming loop.
__device__ __forceinline__ uint32_t pair_lo(uint32_t w) { return __byte_perm(w, 0u, 0x4140); }   // (b0, b1) as 16-bit lanes
__device__ __forceinline__ uint32_t pair_hi(uint32_t w) { return __byte_perm(w, 0u, 0x4342); }   // (b2, b3)

// zb[12]: kBias15 + byte of the quad in source order -> normalised plane quads (FLIP: mirrored)
// zb[12] -> 12 bytes of a uint8 HWC image (scratch images of Sharpness-first programs)
__device__ __forceinline__ void sharp_emit_u8(const float zb[12], uint32_t* w) {
    uint32_t b[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) b[k] = __float_as_uint(zb[k]) & 255u;
    w[0] = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
    w[1] = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
    w[2] = b[8] | (b[9] << 8) | (b[10] << 16) | (b[11] << 24);
}

template <int OUT, bool USE_TAB, bool FLIP>
__device__ __forceinline__ void sharp_emit(const AugParams& P, const float* tab, const float zb[12], typename OutElem<OUT>::T* o,
                                           uint32_t plane) {
    if constexpr (OUT == OUT_U8_HWC) {
        uint32_t ob[12];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const uint32_t u = __float_as_uint(zb[3 * (FLIP ? 3 - k : k) + ch]) & 255u;
                ob[3 * k + ch] = USE_TAB ? f2b(tab[ch * 256 + u]) : u;
            }
        store_quad_u8(o, ob);
        return;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float v[4];
        if (USE_TAB) {
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = tab[ch * 256 + (__float_as_uint(zb[3 * (FLIP ? 3 - k : k) + ch]) & 255u)];
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                v[k] = __fmaf_rn(__fadd_rn(zb[3 * (FLIP ? 3 - k : k) + ch], -kBias15), P.scale[ch], P.bias[ch]);
        }
        store_plane4<OUT>(o + ch * plane, v, true, 4);
    }
}

// u8_dst != nullptr: the result goes, un-normalised and un-mirrored, to a uint8 HWC image (row 0 = image row 0)
template <int OUT, bool USE_TAB, bool CLIP>
__device__ __forceinline__ void final_rows_sharp4(const AugParams& P, const float* tab, const Ctx& c, float alpha, int flip,
                                                  void* out_img, int oy0, int oy1, uint8_t* u8_dst = nullptr) {
    using T = typename OutElem<OUT>::T;
    const int W = P.W, H = P.H;
    const uint32_t qpr = (uint32_t)W >> 2;
    const uint32_t nq = (uint32_t)(oy1 - oy0) * qpr;
    const uint32_t plane = (uint32_t)H * (uint32_t)W, pitch = (uint32_t)W * 3u;
    constexpr uint32_t PS = PixStep<OUT>::v;
    T* dst = reinterpret_cast<T*>(out_img) + PS * (uint32_t)oy0 * (uint32_t)W;
    FastDiv dq; dq.init(qpr, P.rcp_wq);
    uint32_t r = dq.div(threadIdx.x), qx = threadIdx.x - r * qpr;
    const uint32_t dr = dq.div(blockDim.x), dxq = blockDim.x - dr * qpr;
    const float k26 = 1.0f / 26.0f, h26 = 0.5f / 26.0f;
    for (uint32_t q = threadIdx.x; q < nq; q += blockDim.x) {
        const int y = oy0 + (int)r;
        const uint32_t sqx = flip ? qpr - 1u - qx : qx;                   // source quad of this output quad
        const uint32_t* rb = reinterpret_cast<const uint32_t*>(c.sraw + ((uint32_t)y * pitch + 12u * sqx - c.s_lo));
        float zb[12];                                                    // kBias15 + output byte, source order
        if (y == 0 || y == H - 1) {                                      // border rows are copied (Pillow filter)
#pragma unroll
            for (int k = 0; k < 12; ++k) zb[k] = biased_byte(rb[k >> 2], k & 3);
        } else {
            const uint32_t* ra = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(rb) - pitch);
            const uint32_t* rc = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(rb) + pitch);
            const bool has_l = sqx > 0u, has_r = sqx + 1u < qpr;
            // words [-1 .. 3] of the three rows: bytes -4 .. 15 relative to the quad's first byte
            uint32_t wb[5], colp[10], ctr[10];
            {
                uint32_t wa[5], wc[5];
                wa[0] = has_l ? ra[-1] : 0u; wb[0] = has_l ? rb[-1] : 0u; wc[0] = has_l ? rc[-1] : 0u;
#pragma unroll
                for (int j = 1; j < 4; ++j) { wa[j] = ra[j - 1]; wb[j] = rb[j - 1]; wc[j] = rc[j - 1]; }
                wa[4] = has_r ? ra[3] : 0u; wb[4] = has_r ? rb[3] : 0u; wc[4] = has_r ? rc[3] : 0u;
#pragma unroll
                for (int j = 0; j < 5; ++j) {                             // pair m covers bytes 2m, 2m+1 (from byte -4)
                    ctr[2 * j] = pair_lo(wb[j]); ctr[2 * j + 1] = pair_hi(wb[j]);
                    colp[2 * j] = pair_lo(wa[j]) + ctr[2 * j] + pair_lo(wc[j]);
                    colp[2 * j + 1] = pair_hi(wa[j]) + ctr[2 * j + 1] + pair_hi(wc[j]);
                }
            }
            uint32_t sh[9];                                              // sh[m] = stream shifted by 3 bytes: (col[2m-3], col[2m-2])
#pragma unroll
            for (int m = 2; m <= 10; ++m) sh[m - 2] = m < 10 ? __byte_perm(colp[m - 2], colp[m - 1], 0x5432)
                                                             : __byte_perm(colp[8], colp[9], 0x5432);
#pragma unroll
            for (int m = 2; m < 8; ++m) {                                 // output bytes 2m-4, 2m-3
                const uint32_t t = sh[m - 2] + colp[m] + sh[m + 1];      // col[k-3] + col[k] + col[k+3]
                const uint32_t x2 = 2u * t + 8u * ctr[m] + 0x000D000Du;  // 2 S + 13 per lane (< 6644)
#pragma unroll
                for (int l = 0; l < 2; ++l) {                            // the two bytes of the pair
                    const int k = 2 * m + l;                             // byte index from byte -4
                    const float fx = __uint_as_float(__byte_perm(x2, kBias15Bits, l ? 0x7632 : 0x7610));   // kBias15 + (2S+13)
                    const float u = __fmaf_rn(__fadd_rn(fx, -kBias15), k26, h26);                         // (2S+13+.5)/26
                    const float fdeg = __fadd_rz(u, kBias15);                                              // kBias15 + floor(u)
                    const float d = __fmaf_rn(fdeg, -1.0f, biased_byte(wb[k >> 2], k & 3));               // (float)(px - deg), exact
                    // Blend.c: product and sum are rounded SEPARATELY (__fmul_rn / __fadd_rn are never contracted into an fma)
                    float z = __fadd_rz(__fadd_rn(__fadd_rn(fdeg, -kBias15), __fmul_rn(alpha, d)), kBias15);
                    if (CLIP) z = fminf(fmaxf(z, kBias15), kBias15 + 255.0f);
                    zb[k - 4] = z;
                }
            }
            // first / last pixel of the row are image border: copied
            if (!has_l) {
#pragma unroll
                for (int k = 0; k < 3; ++k) zb[k] = biased_byte(wb[1], k);
            }
            if (!has_r) {
#pragma unroll
                for (int k = 9; k < 12; ++k) zb[k] = biased_byte(wb[3], k - 8);
            }
        }
        if (u8_dst != nullptr) {
            sharp_emit_u8(zb, reinterpret_cast<uint32_t*>(u8_dst + (uint32_t)y * pitch + 12u * sqx));
        } else {
            T* o = dst + PS * 4u * q;
            if (flip) sharp_emit<OUT, USE_TAB, true>(P, tab, zb, o, plane);
            else sharp_emit<OUT, USE_TAB, false>(P, tab, zb, o, plane);
        }
        qx += dxq; r += dr;
        if (qx >= qpr) { qx -= qpr; ++r; }
    }
}

}  // namespace faa
