// faa_cabi.cu - host side of the C ABI declared in include/faa_b200.h:
// policy compilation (level -> magnitude -> Pillow fixed-point / LUT / blend parameters),
// the MT19937 parity sampler, normalisation tables, device-table management and launches.
// There is NO CPU implementation of the pixel path in this library: every compute entry
// point fails with FAA_ERR_NO_DEVICE when no CUDA device is usable.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/faa_b200.h"
#include "faa_kernels.cuh"

using namespace faa;

static_assert(sizeof(faa_sample_t) == 16 && sizeof(Sample) == 16, "sample record is 16 bytes");
static_assert(sizeof(faa_box_t) == 8 && sizeof(Box) == 8, "box record is 8 bytes");
static_assert(sizeof(OpRec) == 32, "op record is 32 bytes");
static_assert(sizeof(faa_rng_t) == sizeof(RngCfg), "rng config layout");

// ------------------------------------------------------------------ errors --
static thread_local std::string g_err;
static std::atomic<uint64_t> g_launches{0};

static int fail(int code, const std::string& msg) { g_err = msg; return code; }
static int cuda_fail(cudaError_t e, const char* what) {
    return fail(FAA_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
#define CK(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return cuda_fail(e__, #call); } while (0)

// --------------------------------------------------------------- op table --
struct OpInfo { const char* name; double low, high; int draw; };
// augment_list(for_autoaug=True): augmentations.py:156-182
static const OpInfo kOps[FAA_NUM_OPS] = {
    {"ShearX", -0.3, 0.3, FAA_DRAW_MIRROR},      {"ShearY", -0.3, 0.3, FAA_DRAW_MIRROR},
    {"TranslateX", -0.45, 0.45, FAA_DRAW_MIRROR}, {"TranslateY", -0.45, 0.45, FAA_DRAW_MIRROR},
    {"Rotate", -30, 30, FAA_DRAW_MIRROR},        {"AutoContrast", 0, 1, FAA_DRAW_NONE},
    {"Invert", 0, 1, FAA_DRAW_NONE},             {"Equalize", 0, 1, FAA_DRAW_NONE},
    {"Solarize", 0, 256, FAA_DRAW_NONE},         {"Posterize", 4, 8, FAA_DRAW_NONE},
    {"Contrast", 0.1, 1.9, FAA_DRAW_NONE},       {"Color", 0.1, 1.9, FAA_DRAW_NONE},
    {"Brightness", 0.1, 1.9, FAA_DRAW_NONE},     {"Sharpness", 0.1, 1.9, FAA_DRAW_NONE},
    {"Cutout", 0, 0.2, FAA_DRAW_BOX},            {"CutoutAbs", 0, 20, FAA_DRAW_BOX},
    {"Posterize2", 0, 4, FAA_DRAW_NONE},         {"TranslateXAbs", 0, 10, FAA_DRAW_MIRROR},
    {"TranslateYAbs", 0, 10, FAA_DRAW_MIRROR},
};

// ---------------------------------------------------------- compile helpers --
static inline int32_t fix16(double z) { return (int32_t)std::floor(z * 65536.0 + 0.5); }   // Pillow FIX()

// Python's round(x, 15): correctly rounded decimal round trip
static double py_round15(double x) {
    char buf[64];
    snprintf(buf, sizeof buf, "%.15f", x);
    return strtod(buf, nullptr);
}
// Python float %: result takes the sign of the divisor
static double py_fmod(double a, double b) {
    double r = std::fmod(a, b);
    if (r != 0.0 && ((r < 0.0) != (b < 0.0))) r += b;
    return r;
}
// ImagingScaleAffine axis table (Geometry.c): o = offset + scale*0.5, then o += scale per
// pixel, COORD(o) = o < 0 ? -1 : (int)o.  With unit scale the table is "i + shift", except
// that the repeatedly rounded accumulator may snap up to the next integer once (when
// offset+0.5 sits a few ulp below an integer): from index `brk` on the shift is shift+1.
// Returns false when the table is anything else.
static bool unit_scale_shift(int n, double offset, int32_t* shift, int32_t* brk) {
    double o = offset + 0.5;
    bool have = false; int32_t sh = 0, bk = INT32_MAX;
    std::vector<int32_t> tab(n);
    for (int i = 0; i < n; ++i) { tab[i] = (o < 0.0) ? INT32_MIN : (int32_t)o; o += 1.0; }
    for (int i = 0; i < n; ++i) {
        if (tab[i] == INT32_MIN) continue;
        int32_t d = tab[i] - i;
        if (!have) { sh = d; have = true; }
        else if (d == sh + 1 && bk == INT32_MAX) bk = i;
        else if (d != sh + (bk != INT32_MAX ? 1 : 0)) return false;
    }
    if (!have) { *shift = -2 * (int32_t)FAA_MAX_DIM; *brk = INT32_MAX; return true; }   // everything is fill
    for (int i = 0; i < n; ++i) {            // negative accumulator => Pillow skips the pixel
        if (tab[i] != INT32_MIN) continue;
        int32_t c = i + sh + (i >= bk ? 1 : 0);
        if (c >= 0 && c < n) return false;
    }
    *shift = sh; *brk = bk;
    return true;
}

struct Compiled { OpRec rec; int err; };   // err: 0 ok, FAA_ERR_UNKNOWN_OP, FAA_ERR_MAGNITUDE, FAA_ERR_UNSUPPORTED

static void set_affine(OpRec& r, const double m[6], int H, int W, int& err) {
    if (m[1] == 0.0 && m[3] == 0.0) {                     // Pillow: pure scale -> ImagingScaleAffine
        if (m[0] != 1.0 || m[4] != 1.0) { err = FAA_ERR_UNSUPPORTED; return; }
        int32_t dx, dy, bx, by;
        if (!unit_scale_shift(W, m[2], &dx, &bx) || !unit_scale_shift(H, m[5], &dy, &by)) { err = FAA_ERR_UNSUPPORTED; return; }
        if (dx == 0 && dy == 0 && bx == INT32_MAX && by == INT32_MAX) { r.kind = K_NONE; return; }
        r.kind = K_SHIFT; r.a[0] = dx; r.a[1] = dy; r.a[2] = bx; r.a[3] = by;
        return;
    }
    r.kind = K_AFFINE;                                    // Pillow affine_fixed
    r.a[0] = fix16(m[0]); r.a[1] = fix16(m[1]); r.a[2] = fix16(m[2] + m[0] * 0.5 + m[1] * 0.5);
    r.a[3] = fix16(m[3]); r.a[4] = fix16(m[4]); r.a[5] = fix16(m[5] + m[3] * 0.5 + m[4] * 0.5);
}

static void set_blend(OpRec& r, int kind, double v) {
    float a = (float)v;                                   // _blend passes a C float to ImagingBlend
    r.kind = kind;
    memcpy(&r.a[0], &a, 4);
    r.a[1] = !(a >= 0.0f && a <= 1.0f);
}

// apply_augment (augmentations.py:192-194) + the op's own parameter handling, at compile time
static Compiled compile_op(int op_id, double level, int sign, int H, int W) {
    Compiled c; memset(&c, 0, sizeof c);
    OpRec& r = c.rec; r.kind = K_NONE;
    if (op_id < 0 || op_id >= FAA_NUM_OPS) { c.err = FAA_ERR_UNKNOWN_OP; return c; }
    const OpInfo& info = kOps[op_id];
    r.draw = info.draw;
    double v = level * (info.high - info.low) + info.low;
    // the reference's per-op asserts (CutoutAbs' is commented out, augmentations.py:127)
    bool has_assert = !(op_id == FAA_AUTOCONTRAST || op_id == FAA_INVERT || op_id == FAA_EQUALIZE || op_id == FAA_CUTOUT_ABS);
    if (has_assert && !(info.low <= v && v <= info.high)) { c.err = FAA_ERR_MAGNITUDE; return c; }
    if (info.draw == FAA_DRAW_MIRROR && sign) v = -v;
    double m[6] = {1, 0, 0, 0, 1, 0};
    switch (op_id) {
    case FAA_SHEAR_X: m[1] = v; set_affine(r, m, H, W, c.err); break;                        // :17
    case FAA_SHEAR_Y: m[3] = v; set_affine(r, m, H, W, c.err); break;                        // :24
    case FAA_TRANSLATE_X: m[2] = v * (double)W; set_affine(r, m, H, W, c.err); break;        // :31-32
    case FAA_TRANSLATE_Y: m[5] = v * (double)H; set_affine(r, m, H, W, c.err); break;        // :39-40
    case FAA_TRANSLATE_X_ABS: m[2] = v; set_affine(r, m, H, W, c.err); break;                // :47
    case FAA_TRANSLATE_Y_ABS: m[5] = v; set_affine(r, m, H, W, c.err); break;                // :54
    case FAA_ROTATE: {                                                                        // :61 + PIL Image.rotate
        double angle = py_fmod(v, 360.0);
        if (angle == 0.0) break;                                                              // copy fast path
        if (angle == 180.0 || ((angle == 90.0 || angle == 270.0) && W == H)) { c.err = FAA_ERR_UNSUPPORTED; break; }
        double cx = W / 2.0, cy = H / 2.0;
        double t = -(angle * (M_PI / 180.0));                                                 // -math.radians(angle)
        m[0] = py_round15(std::cos(t)); m[1] = py_round15(std::sin(t)); m[2] = 0.0;
        m[3] = py_round15(-std::sin(t)); m[4] = py_round15(std::cos(t)); m[5] = 0.0;
        double t2 = m[0] * (-cx) + m[1] * (-cy) + m[2];
        double t5 = m[3] * (-cx) + m[4] * (-cy) + m[5];
        m[2] = t2 + cx; m[5] = t5 + cy;
        set_affine(r, m, H, W, c.err);
        break;
    }
    case FAA_AUTOCONTRAST: r.kind = K_AUTOCONTRAST; break;                                    // :65
    case FAA_EQUALIZE: r.kind = K_EQUALIZE; break;                                            // :73
    case FAA_INVERT: r.kind = K_LUT; r.a[0] = 0; r.a[1] = 0xFF; break;                        // :69
    case FAA_SOLARIZE: {                                                                      // :82  (i < v with float v)
        double th = std::ceil(v);
        r.kind = K_LUT; r.a[0] = (int32_t)(th < 0 ? 0 : th > 256 ? 256 : th); r.a[1] = 0xFF;
        break;
    }
    case FAA_POSTERIZE: case FAA_POSTERIZE2: {                                                // :87-88, :93-94
        int bits = (int)v;
        int mask = ~((1 << (8 - bits)) - 1) & 0xFF;
        r.kind = K_LUT; r.a[0] = 256; r.a[1] = mask;
        break;
    }
    case FAA_CONTRAST: set_blend(r, K_CONTRAST, v); break;                                    // :99
    case FAA_COLOR: set_blend(r, K_COLOR, v); break;                                          // :104
    case FAA_BRIGHTNESS: set_blend(r, K_BRIGHTNESS, v); break;                                // :109
    case FAA_SHARPNESS: set_blend(r, K_SHARPNESS, v); break;                                  // :114
    case FAA_CUTOUT: {                                                                        // :117-123
        if (v <= 0.0) { r.draw = FAA_DRAW_NONE; break; }                                      // returns before any draw
        double px = v * (double)W;
        r.kind = K_CUTOUT; memcpy(&r.a[0], &px, 8);
        break;
    }
    case FAA_CUTOUT_ABS: {                                                                    // :126-144
        if (v < 0.0) { r.draw = FAA_DRAW_NONE; break; }
        r.kind = K_CUTOUT; memcpy(&r.a[0], &v, 8);
        break;
    }
    }
    if (c.err) r.kind = K_NONE;
    return c;
}

// ------------------------------------------------------------------ policy --
struct DeviceTable { OpRec* d_ops = nullptr; };

struct faa_policy {
    int n_sub = 0, n_op = 0;
    std::vector<int32_t> op_ids;
    std::vector<double> probs, levels;
    std::mutex mu;
    std::map<std::pair<int, int>, std::vector<Compiled>> host_tables;   // (H,W) -> [n_sub][n_op][2]
    std::map<std::pair<int, int>, DeviceTable> dev_tables;
    double* d_probs = nullptr;
    float* d_norm = nullptr;            // [3][256]
    float norm_mean[3] = {-1e30f, 0, 0}, norm_std[3] = {0, 0, 0};
    float norm_host[768];
    bool fma_known[2] = {false, false}, fma_ok[2] = {false, false};   // [fp16, bf16]: does fmaf(u, scale, bias) round like the table?
    // scratch of faa_augment_host
    void* d_progs = nullptr; size_t d_progs_bytes = 0;
    void* d_order = nullptr;             // int32 [capacity of d_progs in images] (+ counters), two slots like d_progs
    // resolve-ahead: the decisions of the NEXT batch are resolved on a side stream while this batch's
    // pixels are computed; a call whose (rng, shapes, ...) key matches the speculation skips its resolve launch
    struct AheadKey { uint64_t seed, first_index; int32_t v[16]; };
    AheadKey ahead_key{}; bool ahead_valid = false; int ahead_slot = 0, cur_slot = 0;
    bool have_last = false; AheadKey last_key{};
    cudaStream_t ahead_stream = nullptr; cudaEvent_t ev_ahead = nullptr;
    bool ahead_on_side = false;          // an event-schedule resolve-ahead on ahead_stream that no later launch waited for yet
    cudaStream_t last_stream = nullptr; bool have_last_stream = false;   // the stream of the previous call (follow_stream)
    cudaEvent_t ev_switch = nullptr;
    void* d_scratch = nullptr; size_t d_scratch_bytes = 0;   // Sharpness->gather scratch images
    bool overlap_calls = false;          // faa_policy_set_overlap: consecutive calls on one stream may overlap (see augment_common)
    uint32_t done_target[2] = {0, 0};    // persistent chained steps: CTAs that have been launched on each program slot so far
    int sm_count = 0;
    bool has_sg = false;                 // some sub-policy has Sharpness followed by a geometric op
    void* d_in = nullptr; size_t d_in_bytes = 0;
    void* d_out = nullptr; size_t d_out_bytes = 0;
    void* h_in_stage = nullptr; size_t h_in_bytes = 0;
    void* h_out_stage = nullptr; size_t h_out_bytes = 0;
    cudaStream_t side[2] = {nullptr, nullptr};
    cudaStream_t light_stream = nullptr; cudaEvent_t ev_res = nullptr, ev_light = nullptr;
    cudaStream_t mid_stream = nullptr; cudaEvent_t ev_mid = nullptr;   // the mid kernel of a three-way split co-runs on its own stream
    cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
    cudaEvent_t ev_host_done = nullptr; bool host_in_flight = false;   // faa_augment_host: last call's work (it owns d_in / stages)
    std::mutex call_mu;                  // launches of one policy are serialised (speculation state, slots, staging)
    const float* lighting_rgb = nullptr; int lighting_n = 0;       // Lighting offsets [n][3] (device) for the next launches, or null
    float* d_norm_img = nullptr; size_t d_norm_img_bytes = 0;      // per-image normalisation tables [n][3][256]
    int device = -1;                     // the device that owns every buffer / stream / event above (-1: none yet)
    int32_t ticket = 0;                  // chained steps: id of the last resolve launch
    int32_t ahead_ticket = 0;
    cudaStream_t chain_stream = nullptr; bool chain_live = false;   // the previous call was a chained step on this stream
    uintptr_t prev_out[2] = {0, 0}, prev_in[2] = {0, 0};            // byte ranges the previous chained step wrote / read
    // faa_augment_ragged: per-call tables (per-size AugParams, RaggedImg, launch lists, copy jobs), programs, scratch
    // images and re-aligned input copies (grown, never shrunk; stream-ordered reuse)
    void* d_rg_tab = nullptr; size_t d_rg_tab_bytes = 0;
    void* d_rg_progs = nullptr; size_t d_rg_progs_bytes = 0;
    void* d_rg_scratch = nullptr; size_t d_rg_scratch_bytes = 0;
    void* d_rg_copy = nullptr; size_t d_rg_copy_bytes = 0;
    // faa_augment_tta_policies: the candidates' PolicyRef array of the call (grown, never shrunk; stream-ordered reuse)
    void* d_cands = nullptr; size_t d_cands_bytes = 0;
};

// All device state of a policy handle lives on ONE device: the one current at its first device call.
static int bind_device(faa_policy* p) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return fail(FAA_ERR_NO_DEVICE, "no current CUDA device"); }
    std::lock_guard<std::mutex> lk(p->mu);
    if (p->device < 0) p->device = dev;
    if (p->device != dev)
        return fail(FAA_ERR_VALUE, "policy handle is bound to device " + std::to_string(p->device) + " but the current device is " +
                    std::to_string(dev) + ": create one policy handle per device");
    return FAA_OK;
}

static const std::vector<Compiled>& host_table(faa_policy* p, int H, int W) {
    std::lock_guard<std::mutex> lk(p->mu);
    auto key = std::make_pair(H, W);
    auto it = p->host_tables.find(key);
    if (it != p->host_tables.end()) return it->second;
    std::vector<Compiled> t((size_t)p->n_sub * p->n_op * 2);
    for (int s = 0; s < p->n_sub; ++s)
        for (int j = 0; j < p->n_op; ++j)
            for (int sg = 0; sg < 2; ++sg) {
                size_t k = (size_t)s * p->n_op + j;
                t[k * 2 + sg] = compile_op(p->op_ids[k], p->levels[k], sg, H, W);
            }
    return p->host_tables.emplace(key, std::move(t)).first->second;
}

static int first_table_error(const std::vector<Compiled>& t, std::string& what) {
    for (size_t i = 0; i < t.size(); ++i)
        if (t[i].err) {
            what = "sub-policy " + std::to_string(i / 2) + " (flattened op index)";
            return t[i].err;
        }
    return 0;
}

extern "C" {

int faa_abi_version(void) { return FAA_ABI_VERSION; }
const char* faa_last_error(void) { return g_err.c_str(); }
uint64_t faa_launch_count(void) { return g_launches.load(); }

int faa_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int faa_op_id_from_name(const char* name) {
    if (!name) return -1;
    for (int i = 0; i < FAA_NUM_OPS; ++i) if (strcmp(name, kOps[i].name) == 0) return i;
    return -1;
}
const char* faa_op_name(int op_id) { return (op_id >= 0 && op_id < FAA_NUM_OPS) ? kOps[op_id].name : nullptr; }
int faa_op_range(int op_id, double* low, double* high) {
    if (op_id < 0 || op_id >= FAA_NUM_OPS) return fail(FAA_ERR_UNKNOWN_OP, "unknown op id");
    if (low) *low = kOps[op_id].low;
    if (high) *high = kOps[op_id].high;
    return FAA_OK;
}

int faa_policy_create(const int32_t* op_ids, const double* probs, const double* levels, int n_sub, int n_op,
                      faa_policy_t** out) {
    if (!op_ids || !probs || !levels || !out) return fail(FAA_ERR_VALUE, "null argument");
    if (n_sub <= 0 || n_sub > 65535) return fail(FAA_ERR_VALUE, "n_sub must be in [1, 65535]");
    if (n_op <= 0 || n_op > FAA_MAX_POLICY_OPS) return fail(FAA_ERR_VALUE, "n_op must be in [1, 8]");
    faa_policy* p = new faa_policy();
    p->n_sub = n_sub; p->n_op = n_op;
    size_t n = (size_t)n_sub * n_op;
    p->op_ids.assign(op_ids, op_ids + n);
    p->probs.assign(probs, probs + n);
    p->levels.assign(levels, levels + n);
    auto is_geo = [](int id) { return id == FAA_SHEAR_X || id == FAA_SHEAR_Y || id == FAA_TRANSLATE_X || id == FAA_TRANSLATE_Y ||
                                      id == FAA_ROTATE || id == FAA_TRANSLATE_X_ABS || id == FAA_TRANSLATE_Y_ABS; };
    for (int s = 0; s < n_sub && !p->has_sg; ++s)
        for (int j = 0; j + 1 < n_op; ++j)
            if (op_ids[(size_t)s * n_op + j] == FAA_SHARPNESS && is_geo(op_ids[(size_t)s * n_op + j + 1])) p->has_sg = true;
    *out = p;
    return FAA_OK;
}

int faa_policy_destroy(faa_policy_t* p) {
    if (!p) return FAA_OK;
    for (auto& kv : p->dev_tables) if (kv.second.d_ops) cudaFree(kv.second.d_ops);
    if (p->d_probs) cudaFree(p->d_probs);
    if (p->d_norm) cudaFree(p->d_norm);
    if (p->d_progs) cudaFree(p->d_progs);
    if (p->d_order) cudaFree(p->d_order);
    if (p->d_scratch) cudaFree(p->d_scratch);
    if (p->d_norm_img) cudaFree(p->d_norm_img);
    if (p->d_in) cudaFree(p->d_in);
    if (p->d_out) cudaFree(p->d_out);
    for (void* b : {p->d_rg_tab, p->d_rg_progs, p->d_rg_scratch, p->d_rg_copy, p->d_cands}) if (b) cudaFree(b);
    if (p->h_in_stage) cudaFreeHost(p->h_in_stage);
    if (p->h_out_stage) cudaFreeHost(p->h_out_stage);
    for (int i = 0; i < 2; ++i) {
        if (p->side[i]) cudaStreamDestroy(p->side[i]);
        if (p->ev_join[i]) cudaEventDestroy(p->ev_join[i]);
    }
    if (p->ev_fork) cudaEventDestroy(p->ev_fork);
    if (p->ev_host_done) cudaEventDestroy(p->ev_host_done);
    if (p->light_stream) cudaStreamDestroy(p->light_stream);
    if (p->mid_stream) cudaStreamDestroy(p->mid_stream);
    if (p->ev_mid) cudaEventDestroy(p->ev_mid);
    if (p->ahead_stream) cudaStreamDestroy(p->ahead_stream);
    if (p->ev_ahead) cudaEventDestroy(p->ev_ahead);
    if (p->ev_switch) cudaEventDestroy(p->ev_switch);
    if (p->ev_res) cudaEventDestroy(p->ev_res);
    if (p->ev_light) cudaEventDestroy(p->ev_light);
    delete p;
    return FAA_OK;
}

int faa_policy_dims(const faa_policy_t* p, int* n_sub, int* n_op) {
    if (!p) return fail(FAA_ERR_VALUE, "null policy");
    if (n_sub) *n_sub = p->n_sub;
    if (n_op) *n_op = p->n_op;
    return FAA_OK;
}

static int check_shape(int h, int w) {
    if (h <= 0 || w <= 0 || h > FAA_MAX_DIM || w > FAA_MAX_DIM) return fail(FAA_ERR_VALUE, "image size out of range");
    return FAA_OK;
}

int faa_policy_compiled_op(faa_policy_t* p, int h, int w, int sub, int op, int sign, int32_t out8[8]) {
    if (!p || !out8) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_shape(h, w)) return e;
    if (sub < 0 || sub >= p->n_sub || op < 0 || op >= p->n_op) return fail(FAA_ERR_VALUE, "index out of range");
    const Compiled& c = host_table(p, h, w)[((size_t)sub * p->n_op + op) * 2 + (sign ? 1 : 0)];
    memcpy(out8, &c.rec, 32);
    if (c.err) return fail(c.err, "op cannot be compiled (unknown op / magnitude out of range)");
    return FAA_OK;
}

int faa_policy_draw_kind(const faa_policy_t* p, int sub, int op) {
    if (!p || sub < 0 || sub >= p->n_sub || op < 0 || op >= p->n_op) return -1;
    int id = p->op_ids[(size_t)sub * p->n_op + op];
    if (id < 0 || id >= FAA_NUM_OPS) return -1;
    if (id == FAA_CUTOUT) {
        double v = p->levels[(size_t)sub * p->n_op + op] * (kOps[id].high - kOps[id].low) + kOps[id].low;
        if (v <= 0.0) return FAA_DRAW_NONE;
    }
    return kOps[id].draw;
}

int faa_cutout_box(const faa_policy_t* pc, int h, int w, int sub, int op, double ux, double uy, faa_box_t* out) {
    faa_policy* p = const_cast<faa_policy*>(pc);
    if (!p || !out) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_shape(h, w)) return e;
    if (sub < 0 || sub >= p->n_sub || op < 0 || op >= p->n_op) return fail(FAA_ERR_VALUE, "index out of range");
    const Compiled& c = host_table(p, h, w)[((size_t)sub * p->n_op + op) * 2];
    if (c.err) return fail(c.err, "op cannot be compiled");
    if (c.rec.kind != K_CUTOUT) return fail(FAA_ERR_VALUE, "op draws no box");
    double v; memcpy(&v, &c.rec.a[0], 8);
    Box b = cutout_box(w, h, v, ux, uy);
    memcpy(out, &b, 8);
    return FAA_OK;
}

// ------------------------------------------------------------ MT19937 replay --
struct MT {
    uint32_t* s; uint32_t* pos;
    explicit MT(uint32_t st[625]) : s(st), pos(st + 624) {}
    void refill() {
        const uint32_t N = 624, M = 397, UP = 0x80000000u, LO = 0x7fffffffu, A = 0x9908b0dfu;
        uint32_t y; uint32_t kk;
        for (kk = 0; kk < N - M; ++kk) { y = (s[kk] & UP) | (s[kk + 1] & LO); s[kk] = s[kk + M] ^ (y >> 1) ^ ((y & 1u) ? A : 0u); }
        for (; kk < N - 1; ++kk) { y = (s[kk] & UP) | (s[kk + 1] & LO); s[kk] = s[kk + (M - N)] ^ (y >> 1) ^ ((y & 1u) ? A : 0u); }
        y = (s[N - 1] & UP) | (s[0] & LO); s[N - 1] = s[M - 1] ^ (y >> 1) ^ ((y & 1u) ? A : 0u);
        *pos = 0;
    }
    uint32_t u32() {
        if (*pos >= 624) refill();
        uint32_t y = s[(*pos)++];
        y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
        return y;
    }
    double real53() {   // CPython random.random() and numpy legacy random_sample(): same formula
        uint32_t a = u32() >> 5, b = u32() >> 6;
        return (a * 67108864.0 + b) * (1.0 / 9007199254740992.0);
    }
    uint32_t below(uint32_t n) {   // CPython _randbelow_with_getrandbits
        int k = 32 - __builtin_clz(n);
        uint32_t r;
        do { r = u32() >> (32 - k); } while (r >= n);
        return r;
    }
};

int faa_sample_policy_mt(const faa_policy_t* pc, int batch, int h, int w, uint32_t py_state[625],
                         uint32_t np_state[625], faa_sample_t* out_samples, faa_box_t* out_boxes) {
    faa_policy* p = const_cast<faa_policy*>(pc);
    if (!p || !py_state || !np_state || !out_samples || !out_boxes) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (int e = check_shape(h, w)) return e;
    if (py_state[624] > 624 || np_state[624] > 624) return fail(FAA_ERR_VALUE, "bad MT19937 position");
    const std::vector<Compiled>& tab = host_table(p, h, w);
    MT py(py_state), np(np_state);
    for (int i = 0; i < batch; ++i) {
        faa_sample_t s; memset(&s, 0, sizeof s);
        uint32_t sub = py.below((uint32_t)p->n_sub);                          // random.choice, data.py:259
        s.sub = (uint16_t)sub;
        for (int j = 0; j < p->n_op; ++j) {
            faa_box_t& bx = out_boxes[(size_t)i * p->n_op + j];
            bx.x0 = bx.y0 = 0; bx.x1 = bx.y1 = -1;
            size_t k = (size_t)sub * p->n_op + j;
            if (p->probs[k] < 0.0) continue;                                   // padding slot of a ragged sub-policy: no draw
            if (py.real53() > p->probs[k]) continue;                           // data.py:261
            const Compiled& c0 = tab[k * 2];
            if (c0.err) return fail(c0.err, std::string("applied op is invalid: ") +
                                    (c0.err == FAA_ERR_UNKNOWN_OP ? "unknown op" : "magnitude out of range / unsupported"));
            s.gate |= (uint8_t)(1u << j);
            if (c0.rec.draw == FAA_DRAW_MIRROR) {
                if (py.real53() > 0.5) s.sign |= (uint8_t)(1u << j);           // augmentations.py:15 ...
            } else if (c0.rec.draw == FAA_DRAW_BOX) {
                double ux = np.real53(), uy = np.real53();                     // augmentations.py:131-132
                double v; memcpy(&v, &c0.rec.a[0], 8);
                Box b = cutout_box(w, h, v, ux, uy);
                memcpy(&bx, &b, 8);
            }
        }
        out_samples[i] = s;
    }
    return FAA_OK;
}

// ------------------------------------------------------------ device tables --
static int ensure_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(FAA_ERR_NO_DEVICE, "no CUDA device available: fast_autoaugment_b200 has no CPU fallback");
    }
    return FAA_OK;
}

static int device_table(faa_policy* p, int H, int W, bool need_valid, const OpRec** d_ops) {
    const std::vector<Compiled>& t = host_table(p, H, W);
    if (need_valid) {
        std::string what;
        if (int e = first_table_error(t, what))
            return fail(e, "policy contains an op that cannot run (" + what + "): unknown op or magnitude out of range");
    }
    std::lock_guard<std::mutex> lk(p->mu);
    auto key = std::make_pair(H, W);
    auto it = p->dev_tables.find(key);
    if (it == p->dev_tables.end()) {
        std::vector<OpRec> flat(t.size());
        for (size_t i = 0; i < t.size(); ++i) flat[i] = t[i].rec;
        DeviceTable d;
        CK(cudaMalloc(&d.d_ops, flat.size() * sizeof(OpRec)));
        CK(cudaMemcpy(d.d_ops, flat.data(), flat.size() * sizeof(OpRec), cudaMemcpyHostToDevice));
        it = p->dev_tables.emplace(key, d).first;
    }
    if (!p->d_probs) {
        CK(cudaMalloc(&p->d_probs, p->probs.size() * sizeof(double)));
        CK(cudaMemcpy(p->d_probs, p->probs.data(), p->probs.size() * sizeof(double), cudaMemcpyHostToDevice));
    }
    *d_ops = it->second.d_ops;
    return FAA_OK;
}

// ToTensor + Normalize exactly as torch computes them in fp32 (data.py:42-43):
// x = u8 / 255 ; (x - mean) / std.  Also decides whether one fused multiply-add reproduces
// the rounded result for every byte value in the requested output dtype.
static uint16_t bits16(int dtype, float v) {
    if (dtype == FAA_F16) { __half h = __float2half_rn(v); return __half_as_ushort(h); }
    __nv_bfloat16 b = __float2bfloat16_rn(v); return __bfloat16_as_ushort(b);
}

static int normalisation(faa_policy* p, const faa_tail_t* tail, AugParams& P, bool& use_tab, cudaStream_t stream) {
    bool same = true;
    for (int c = 0; c < 3; ++c) same = same && p->norm_mean[c] == tail->mean[c] && p->norm_std[c] == tail->std[c];
    if (!p->d_norm) { CK(cudaMalloc(&p->d_norm, 768 * sizeof(float))); same = false; }
    if (!same) {
        for (int c = 0; c < 3; ++c) {
            if (!(tail->std[c] != 0.0f)) return fail(FAA_ERR_VALUE, "std must be non-zero");
            for (int u = 0; u < 256; ++u) {
                volatile float x = (float)u / 255.0f;
                volatile float y = x - tail->mean[c];
                volatile float z = y / tail->std[c];
                p->norm_host[c * 256 + u] = z;
            }
            p->norm_mean[c] = tail->mean[c]; p->norm_std[c] = tail->std[c];
        }
        CK(cudaMemcpyAsync(p->d_norm, p->norm_host, 768 * sizeof(float), cudaMemcpyHostToDevice, stream));
    }
    P.norm_tab = p->d_norm;
    if (!same) p->fma_known[0] = p->fma_known[1] = false;
    const bool half_out = tail->out_dtype == FAA_F16 || tail->out_dtype == FAA_BF16;
    const int slot = tail->out_dtype == FAA_BF16 ? 1 : 0;
    bool fma_ok = half_out;
    for (int c = 0; c < 3; ++c) {
        double sc = 1.0 / (255.0 * (double)tail->std[c]);
        double bi = -(double)tail->mean[c] / (double)tail->std[c];
        P.scale[c] = (float)sc; P.bias[c] = (float)bi;
    }
    if (half_out && p->fma_known[slot]) {
        fma_ok = p->fma_ok[slot];                           // (768 conversions per call are a visible part of a small step)
    } else if (half_out) {
        for (int c = 0; c < 3 && fma_ok; ++c)
            for (int u = 0; u < 256 && fma_ok; ++u) {
                float f = fmaf((float)u, P.scale[c], P.bias[c]);
                if (bits16(tail->out_dtype, f) != bits16(tail->out_dtype, p->norm_host[c * 256 + u])) fma_ok = false;
            }
        p->fma_known[slot] = true; p->fma_ok[slot] = fma_ok;
    }
    use_tab = !fma_ok;
    return FAA_OK;
}

static int out_elem_size(int dtype) { return dtype == FAA_F32 ? 4 : dtype == FAA_U8_HWC ? 1 : 2; }

// RandomCrop offsets travel as int8 (faa_sample_t): ranges that do not fit are refused, never silently changed
static int check_crop(int h, int w, const faa_tail_t* tail, int crop_pad) {
    const int span_y = h + 2 * crop_pad - tail->out_h, span_x = w + 2 * crop_pad - tail->out_w;
    if (span_y < 0 || span_x < 0)
        return fail(FAA_ERR_VALUE, "Required crop size is larger than the (padded) input image size");   // torchvision's message
    if (crop_pad > 127 || span_y - crop_pad > 127 || span_x - crop_pad > 127)
        return fail(FAA_ERR_UNSUPPORTED, "RandomCrop offsets beyond +-127 pixels are not supported (int8 records): crop on the host side");
    return FAA_OK;
}

static int check_tail(const faa_tail_t* tail) {
    if (!tail) return fail(FAA_ERR_VALUE, "null tail");
    if (tail->out_h <= 0 || tail->out_w <= 0 || tail->out_h > FAA_MAX_DIM || tail->out_w > FAA_MAX_DIM)
        return fail(FAA_ERR_VALUE, "output size out of range");
    if (tail->out_dtype < 0 || tail->out_dtype > FAA_U8_HWC) return fail(FAA_ERR_VALUE, "bad out_dtype");
    return FAA_OK;
}

// The policy kernels move whole quads of pixels as words whenever rows hold whole quads: the input as 32-bit words
// (load12, W % 4 == 0) and each output plane as one 16-byte (fp32), 8-byte (fp16 / bf16) or three 32-bit (uint8 HWC)
// stores (store_plane4, emit_quad, out_w % 4 == 0).  Image, plane and row offsets are multiples of those sizes then, so
// the buffers' bases decide.  (The 16-byte paths - TMA staging, octets, the mid kernel - test their own alignment and
// are simply not taken.)  A contiguous view at an offset into a larger allocation can miss these alignments.
static int check_alignment(const void* d_in, const void* d_out, int w, const faa_tail_t* tail) {
    if ((w & 3) == 0 && ((uintptr_t)d_in & 3))
        return fail(FAA_ERR_UNSUPPORTED, "the input must be 4-byte aligned when W % 4 == 0 (32-bit loads)");
    if ((tail->out_w & 3) == 0) {
        const uintptr_t need = tail->out_dtype == FAA_F32 ? 16 : tail->out_dtype == FAA_U8_HWC ? 4 : 8;
        if ((uintptr_t)d_out & (need - 1))
            return fail(FAA_ERR_UNSUPPORTED, "the output must be " + std::to_string(need) +
                                             "-byte aligned when its width is a multiple of 4 (vector stores)");
    }
    return FAA_OK;
}

int faa_sample_philox(faa_policy_t* p, int batch, int h, int w, const faa_tail_t* tail, const faa_rng_t* rng,
                      faa_sample_t* d_samples, faa_box_t* d_boxes, void* stream) {
    return faa_sample_philox_at(p, batch, h, w, tail, rng, nullptr, d_samples, d_boxes, stream);
}

int faa_policy_cached_tables(faa_policy_t* p, int* n_tables, uint64_t* bytes) {
    if (!p || !n_tables || !bytes) return fail(FAA_ERR_VALUE, "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    *n_tables = (int)p->dev_tables.size();
    *bytes = (uint64_t)p->dev_tables.size() * p->n_sub * p->n_op * 2u * sizeof(OpRec);
    return FAA_OK;
}

int faa_sample_philox_at(faa_policy_t* p, int batch, int h, int w, const faa_tail_t* tail, const faa_rng_t* rng,
                         const int32_t* d_pos, faa_sample_t* d_samples, faa_box_t* d_boxes, void* stream) {
    if (!p || !rng || !d_samples || !d_boxes) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_tail(tail)) return e;
    if (int e = check_crop(h, w, tail, rng->crop_pad > 0 ? rng->crop_pad : 0)) return e;
    if (int e = ensure_device()) return e;
    if (int e = bind_device(p)) return e;
    const OpRec* d_ops = nullptr;
    if (int e = device_table(p, h, w, true, &d_ops)) return e;
    ResolveParams R; memset(&R, 0, sizeof R);
    R.ops = d_ops; R.probs = p->d_probs; memcpy(&R.rng, rng, sizeof(RngCfg));
    R.samples_out = reinterpret_cast<Sample*>(d_samples); R.boxes_out = reinterpret_cast<Box*>(d_boxes);
    R.pos = d_pos; R.first = 0; R.n = batch; R.H = h; R.W = w; R.out_h = tail->out_h; R.out_w = tail->out_w;
    R.n_sub = p->n_sub; R.n_op = p->n_op; R.op_base = 0; R.apply_tail = 1;
    CK(launch_resolve(R, (cudaStream_t)stream));
    if (batch > 0) g_launches++;
    return FAA_OK;
}

// What augment_common decided for one call: the launch plan, and what this call adds to it.
struct Schedule : LaunchPlan {
    bool use_tab;               // exact normalisation table instead of one fma
    bool hit;                   // the previous call already resolved exactly this batch (resolve-ahead)
    size_t scratch_slot_bytes;  // scratch images per program slot
};

// Program / schedule buffers come in two slots; a slot = progs[cap] + order[cap] + counters[2 cap] + ready[cap] + done word.
// The segment counters of a split launch live behind the order array, indexed by `first` so that concurrent chunk launches
// do not share them (same for the ready word).  Chained steps also own a completion counter and a scratch image per slot.
static void bind_slot(const faa_policy* p, const Schedule& s, int first, int slot, ResolveParams& r, AugParams* a) {
    const size_t cap_imgs = p->d_progs_bytes / sizeof(Prog);
    Prog* progs = reinterpret_cast<Prog*>((uint8_t*)p->d_progs + (size_t)slot * p->d_progs_bytes);
    int32_t* order = reinterpret_cast<int32_t*>(p->d_order) + (size_t)slot * (4 * cap_imgs + 8);
    int32_t* counter = order + cap_imgs + 2 * (size_t)first;
    int32_t* ready = order + 3 * cap_imgs + first;
    uint32_t* done = reinterpret_cast<uint32_t*>(order + 4 * cap_imgs);     // the slot's completion counter
    r.progs = progs; r.order = s.use_order ? order : nullptr; r.n_heavy = s.use_split ? counter : nullptr;
    r.ready = s.use_chain ? ready : nullptr;
    // (the pixel kernels that last read the slot release their dependents before they finish: the resolve kernel that
    //  rewrites it first waits until all of them have counted themselves)
    if (s.use_chain) { r.wait_done = done; r.wait_target = p->done_target[slot]; }
    if (a) {
        a->progs = progs; a->order = r.order; a->n_heavy = r.n_heavy; a->ready = r.ready;
        if (s.use_chain) {
            a->done = done;
            if (a->scratch) a->scratch = (uint8_t*)p->d_scratch + (size_t)slot * s.scratch_slot_bytes;
        }
    }
}

// the mid kernel's launch: its own (taller) bands in bands / geo[0]
static AugParams mid_params(AugParams a, const BandGeom& mid) {
    a.bands = mid.bands; a.geo[0] = mid; a.band_cap = mid.band_cap; a.mat_cap = 0;
    return a;
}

// the byte ranges the step P describes reads and writes
static void step_ranges(const AugParams& P, int out_dtype, uintptr_t in[2], uintptr_t out[2]) {
    const size_t img_bytes = (size_t)P.H * P.W * 3;
    in[0] = (uintptr_t)P.in + (P.in_mod ? 0 : (size_t)P.first * img_bytes);
    in[1] = in[0] + (size_t)(P.in_mod ? P.in_mod : P.B) * img_bytes;
    out[0] = (uintptr_t)P.out;
    out[1] = out[0] + (size_t)P.B * P.out_h * P.out_w * 3 * out_elem_size(out_dtype);
}

// A step may only overlap the previous one if it follows it on the same stream and neither reads what that step wrote
// nor writes what it read or wrote; otherwise its first kernel is a plain dependent launch.  And only if the caller has
// promised that this call's inputs were complete before the previous call was issued (faa_policy_set_overlap /
// faa_augment_many): a kernel launched with programmatic serialization that does not execute griddepcontrol.wait has no
// visibility guarantee for what the kernel right in front of it wrote, and that kernel may be the producer of this batch
// (a gather, a copy).  Within a call every kernel only consumes what its own call's first - stream-ordered - kernel
// already waited for.
static bool may_overlap_previous(const faa_policy* p, const AugParams& P, int out_dtype, cudaStream_t stream) {
    uintptr_t in[2], out[2];
    step_ranges(P, out_dtype, in, out);
    auto overlap = [](const uintptr_t a[2], const uintptr_t b[2]) { return a[0] < b[1] && b[0] < a[1]; };
    return p->overlap_calls && p->chain_live && p->chain_stream == stream && !overlap(in, p->prev_out) &&
           !overlap(out, p->prev_out) && !overlap(out, p->prev_in);
}

// this step is the one the next call on `stream` may overlap
static void record_step(faa_policy* p, const AugParams& P, int out_dtype, cudaStream_t stream) {
    step_ranges(P, out_dtype, p->prev_in, p->prev_out);
    p->chain_live = true; p->chain_stream = stream;
}

// A call on another stream than the previous call first waits for everything issued to that stream so far.  The
// previous call's kernels may still read the program slot, scratch image and tables this call rewrites, and nothing else
// orders them across streams: event-schedule kernels do not count themselves (a chained resolve's completion-counter wait
// passes at once, an event-schedule resolve does not wait at all), and a chained hit would poll a ticket whose resolve
// kernel sits in the other stream and need not have started.  Alternating streams therefore serialise; calls on one
// stream pay nothing.
static int follow_stream(faa_policy* p, cudaStream_t stream) {
    if (p->have_last_stream && p->last_stream != stream) {
        if (!p->ev_switch) CK(cudaEventCreateWithFlags(&p->ev_switch, cudaEventDisableTiming));
        CK(cudaEventRecord(p->ev_switch, p->last_stream));
        CK(cudaStreamWaitEvent(stream, p->ev_switch, 0));
    }
    p->last_stream = stream; p->have_last_stream = true;
    return FAA_OK;
}

// Resolve-ahead: speculate that the next call is this one (`key`) with first_index advanced by the stride seen so far.
// Returns the resolve parameters of that call; the caller binds them to the other slot, launches them and then sets
// ahead_valid.
static ResolveParams speculate_next(faa_policy* p, const faa_policy::AheadKey& key, const ResolveParams& R, int batch) {
    uint64_t stride = (uint64_t)batch;
    faa_policy::AheadKey base = key; base.first_index = 0;
    faa_policy::AheadKey lastb = p->last_key; lastb.first_index = 0;
    if (p->have_last && memcmp(&base, &lastb, sizeof base) == 0 && key.first_index > p->last_key.first_index)
        stride = key.first_index - p->last_key.first_index;
    p->last_key = key; p->have_last = true;
    ResolveParams R2 = R;
    R2.rng.first_index = key.first_index + stride;
    p->ahead_key = key; p->ahead_key.first_index = R2.rng.first_index;
    p->ahead_slot = p->cur_slot ^ 1;
    return R2;
}

// Self-resolving launch: a launch of tiny images is bound by kernel latencies and by the host's launch rate, not by
// bytes.  Thread 0 of every CTA draws its image's decisions and builds the program itself (same Philox counters, same
// build_prog): ONE kernel per step, no program array, no ticket - consecutive steps have no dependency left and overlap
// through programmatic dependent launch.
static int launch_self_resolving(faa_policy* p, const AugParams& P, const ResolveParams& R, bool use_tab, int out_dtype,
                                 cudaStream_t stream) {
    const bool overlap_ok = may_overlap_previous(p, P, out_dtype, stream) && !P.norm_stride;
    AugParams Ps = P;
    Ps.progs = nullptr; Ps.order = nullptr; Ps.n_heavy = nullptr; Ps.ready = nullptr; Ps.done = nullptr; Ps.grid_y = 0;
    Ps.self_resolve = 1;
    Ps.sr_ops = R.ops; Ps.sr_probs = R.probs; Ps.sr_rng = R.rng;
    Ps.sr_n_sub = R.n_sub; Ps.sr_n_op = R.n_op; Ps.sr_op_base = R.op_base; Ps.sr_apply_tail = R.apply_tail;
    // Sharpness -> gather programs are evaluated lazily instead of through the scratch image - the last thing consecutive
    // steps shared - so every CTA may release the next step at once; a step that touches the previous step's buffers is
    // launched as a plain stream-ordered kernel instead
    Ps.sr_allow = R.allow & ~2; Ps.scratch = nullptr;
    Ps.chain = overlap_ok ? CHAIN_SELF_RESOLVING : CHAIN_STREAM_ORDERED; Ps.pdl = 0;
    CK(launch_augment(Ps, out_dtype, use_tab, 0, stream));
    g_launches++;
    p->ahead_valid = false;
    record_step(p, P, out_dtype, stream);
    return FAA_OK;
}

// Chained schedule: resolve(N+1), [cluster(N),] mid(N), light(N) all on the caller's stream with programmatic dependent
// launches, no events and no side streams.  Consecutive steps overlap (the next step's CTAs fill the slots the previous
// step's tail frees); the only true dependency - programs written by the resolve kernel - is a ticket word the pixel
// kernels poll.  The mid and light kernels are persistent: one resident wave each, whose rows loop over their entries,
// so a kernel releases its dependents immediately and consecutive kernels - and steps - overlap for their whole length.
// What the early release no longer orders is ordered explicitly: program slots by completion counters the next resolve
// kernel of the slot waits for, scratch images by a copy per slot.
static int launch_chained(faa_policy* p, const AugParams& P, ResolveParams& R, const Schedule& s,
                          const faa_policy::AheadKey& key, int out_dtype, cudaStream_t stream) {
    // an event-schedule call resolved ahead into the other slot on ahead_stream: this step's resolve-ahead rewrites that
    // slot on `stream` (a chained step never hits an event-schedule speculation: the key differs)
    if (p->ahead_on_side) { CK(cudaStreamWaitEvent(stream, p->ev_ahead, 0)); p->ahead_on_side = false; }
    bool overlap_ok = may_overlap_previous(p, P, out_dtype, stream);
    AugParams Pc = P;
    Pc.chain = CHAIN_STEP; Pc.pdl = 0;
    int slot = p->cur_slot;
    if (s.hit) {
        slot = p->ahead_slot;
        Pc.ticket = p->ahead_ticket;
        bind_slot(p, s, P.first, slot, R, &Pc);
    } else {
        bind_slot(p, s, P.first, slot, R, &Pc);
        R.ticket = ++p->ticket; R.pdl = overlap_ok ? 1 : 0;
        Pc.ticket = R.ticket;
        CK(launch_resolve(R, stream));
        g_launches++;
        overlap_ok = true;                              // the kernels behind it may overlap IT
    }
    p->cur_slot = slot;
    p->ahead_valid = false;
    ResolveParams R2 = speculate_next(p, key, R, P.B);
    bind_slot(p, s, P.first, slot ^ 1, R2, nullptr);
    R2.ticket = ++p->ticket; R2.pdl = overlap_ok ? 1 : 0;
    CK(launch_resolve(R2, stream));
    g_launches++;
    p->ahead_valid = true; p->ahead_ticket = R2.ticket;

    if (!p->sm_count) CK(cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, p->device));
    AugParams Pm = s.use_mid ? mid_params(Pc, s.mid) : Pc;
    // one resident wave each (launch bounds: light CTAs / SM; mid rows: ONE CTA per SM, so that the light CTAs that
    // follow share the SM with it from the start)
    const int lb = P.geo[1].bands > 0 ? P.geo[1].bands : 1;
    const int light = s.lean_light ? 3 : 1;
    Pc.grid_y = (p->sm_count * resident_ctas_per_sm(light)) / lb;
    Pm.grid_y = p->sm_count / (Pm.bands > 0 ? Pm.bands : 1);
    if (Pc.grid_y < 1) Pc.grid_y = 1;
    if (Pm.grid_y < 1) Pm.grid_y = 1;
    auto launch = [&](const AugParams& a, int which) -> int {
        CK(launch_augment(a, out_dtype, s.use_tab, which, stream));
        g_launches++;
        p->done_target[slot] += augment_cta_count(a, which);
        return FAA_OK;
    };
    if (!s.no_heavy) {                                  // the cluster kernel keeps one cluster per entry
        AugParams Pk = Pc; Pk.grid_y = 0;
        if (int e = launch(Pk, 0)) return e;
    }
    if (s.use_split) {
        if (s.use_mid) { if (int e = launch(Pm, 2)) return e; }
        if (int e = launch(Pc, light)) return e;
    }
    record_step(p, P, out_dtype, stream);
    return FAA_OK;
}

// Event schedule, for what cannot be chained (resolved samples, fused Mixup, the host-buffer entry, the windows of
// policies of more than two ops, uint8 output of one pixel kernel): the resolve kernel and the light streaming kernel on
// the caller's stream, the cluster and mid kernels on high-priority side streams, joined by events.
static int launch_event(faa_policy* p, AugParams& P, ResolveParams& R, const Schedule& s, const faa_policy::AheadKey& key,
                        int out_dtype, cudaStream_t stream) {
    p->chain_live = false;
    int slot = p->cur_slot;
    if (s.hit) {
        slot = p->ahead_slot;
        CK(cudaStreamWaitEvent(stream, p->ev_ahead, 0));
        p->ahead_on_side = false;
        P.pdl = 0;                                          // no resolve kernel right in front of the pixel kernel
        bind_slot(p, s, P.first, slot, R, &P);
    } else {
        bind_slot(p, s, P.first, slot, R, &P);
        CK(launch_resolve(R, stream));
        g_launches++;
    }
    p->cur_slot = slot;
    p->ahead_valid = false;
    if (P.n_heavy || s.speculate) {
        if (!p->light_stream) {
            int lo = 0, hi = 0;
            CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));       // hi = numerically lowest = greatest priority
            CK(cudaStreamCreateWithPriority(&p->light_stream, cudaStreamNonBlocking, hi));
            CK(cudaStreamCreateWithPriority(&p->ahead_stream, cudaStreamNonBlocking, hi));   // one block: get a slot promptly
            CK(cudaStreamCreateWithPriority(&p->mid_stream, cudaStreamNonBlocking, hi));
            CK(cudaEventCreateWithFlags(&p->ev_mid, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&p->ev_res, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&p->ev_light, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&p->ev_ahead, cudaEventDisableTiming));
        }
        CK(cudaEventRecord(p->ev_res, stream));               // this batch's programs are ready
    }
    if (s.speculate) {
        ResolveParams R2 = speculate_next(p, key, R, P.B);
        bind_slot(p, s, P.first, slot ^ 1, R2, nullptr);
        CK(cudaStreamWaitEvent(p->ahead_stream, p->ev_res, 0));      // the other slot's last readers are done
        CK(launch_resolve(R2, p->ahead_stream));
        CK(cudaEventRecord(p->ev_ahead, p->ahead_stream));
        g_launches++;
        p->ahead_valid = true; p->ahead_on_side = true;
    }
    if (!P.n_heavy) {                                       // one pixel kernel
        CK(launch_augment(P, out_dtype, s.use_tab, 0, stream));
        g_launches++;
        return FAA_OK;
    }
    // Split pixel kernels, concurrently: the streaming kernel goes FIRST on the caller's stream and fills the machine at
    // once; the clusters of the cluster and mid kernels on the high-priority side streams then take the CTA slots its CTAs
    // free (heavy images finish early, light work fills the gaps; launched first, the thousands of exiting CTAs of the
    // cluster kernels would hold up the work distributor).
    AugParams Ph = P; Ph.pdl = 0;                           // not behind the resolve kernel in its stream
    CK(cudaStreamWaitEvent(p->light_stream, p->ev_res, 0));
    if (s.use_mid) CK(cudaStreamWaitEvent(p->mid_stream, p->ev_res, 0));
    CK(launch_augment(P, out_dtype, s.use_tab, s.lean_light ? 3 : 1, stream));
    g_launches++;
    if (!s.no_heavy) {
        CK(launch_augment(Ph, out_dtype, s.use_tab, 0, p->light_stream));
        g_launches++;
    }
    if (s.use_mid) {
        CK(launch_augment(mid_params(Ph, s.mid), out_dtype, s.use_tab, 2, p->mid_stream));
        g_launches++;
        CK(cudaEventRecord(p->ev_mid, p->mid_stream));
    }
    CK(cudaEventRecord(p->ev_light, p->light_stream));
    if (s.use_mid) CK(cudaStreamWaitEvent(stream, p->ev_mid, 0));
    CK(cudaStreamWaitEvent(stream, p->ev_light, 0));
    return FAA_OK;
}

// One policy launch as an entry point describes it: images [first, first + batch) of the n_all images at `in`, with
// resolved decisions (samples / boxes) or decisions drawn by `rng`.
struct AugRequest {
    const uint8_t* in = nullptr; void* out = nullptr;
    int n_all = 0, first = 0, batch = 0, h = 0, w = 0;
    const faa_tail_t* tail = nullptr; void* stream = nullptr;
    const faa_sample_t* samples = nullptr; const faa_box_t* boxes = nullptr; const faa_rng_t* rng = nullptr;
    int op_base = 0, apply_tail = 1;                // apply_tail: the final window of the policy
    const int32_t* partner = nullptr; float lam = 1.0f, one_minus_lam = 0.0f;    // fused Mixup
    bool allow_ahead = false;                       // the next call's batch may be resolved ahead
    int in_mod = 0;                                 // > 0: replicated launch (TTA), entry v reads input image v % in_mod
    bool own_stream = true;                         // false: a chunk of faa_augment_host on one of its side streams,
                                                    // which that call orders itself
    // multi-policy TTA (faa_augment_tta_policies): entry v draws with candidate cands[v / per_cand]; cands[0] is the
    // handle the call runs on, the others only lend their device tables
    faa_policy_t* const* cands = nullptr; int n_cands = 0, per_cand = 0;
};

// grows one of the handle's per-call table buffers; earlier calls' kernels that may still use it are ordered on `stream`
// (follow_stream), so waiting for it before the free is enough
static int grow_on_stream(void** ptr, size_t* have, size_t need, cudaStream_t stream) {
    if (*have >= need) return FAA_OK;
    if (*ptr) { CK(cudaStreamSynchronize(stream)); CK(cudaFree(*ptr)); *ptr = nullptr; *have = 0; }
    need = std::max(need, (size_t)65536);
    CK(cudaMalloc(ptr, need));
    *have = need;
    return FAA_OK;
}

// The candidates' device tables at h x w (each taken under its own handle's mu), uploaded as the call's PolicyRef array
// on `stream`.
static int upload_candidates(faa_policy* p, faa_policy_t* const* cands, int n_cands, int h, int w, cudaStream_t stream,
                             const PolicyRef** d_refs) {
    std::vector<PolicyRef> refs((size_t)n_cands);
    for (int t = 0; t < n_cands; ++t) {
        faa_policy* c = cands[t];
        if (int e = bind_device(c)) return e;
        if (int e = device_table(c, h, w, true, &refs[(size_t)t].ops)) return e;
        refs[(size_t)t].probs = c->d_probs; refs[(size_t)t].n_sub = c->n_sub; refs[(size_t)t].reserved = 0;
    }
    const size_t bytes = refs.size() * sizeof(PolicyRef);
    if (int e = grow_on_stream(&p->d_cands, &p->d_cands_bytes, bytes, stream)) return e;
    CK(cudaMemcpyAsync(p->d_cands, refs.data(), bytes, cudaMemcpyHostToDevice, stream));   // (pageable: staged at once)
    *d_refs = reinterpret_cast<const PolicyRef*>(p->d_cands);
    return FAA_OK;
}

static int augment_common(faa_policy_t* p, const AugRequest& q) {
    const faa_tail_t* tail = q.tail;
    const int batch = q.batch, h = q.h, w = q.w;
    if (!p || (!q.in && batch > 0) || (!q.out && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0 || q.first < 0 || q.first + batch > q.n_all) return fail(FAA_ERR_VALUE, "bad batch range");
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "at most 65535 images per call (one grid row per image): split the batch");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_tail(tail)) return e;
    if (!q.samples && !q.rng) return fail(FAA_ERR_VALUE, "need either resolved samples or an rng config");
    if (q.rng && !q.samples && q.apply_tail) { if (int e = check_crop(h, w, tail, q.rng->crop_pad > 0 ? q.rng->crop_pad : 0)) return e; }
    if (q.op_base < 0 || q.op_base >= p->n_op) return fail(FAA_ERR_VALUE, "op_base out of range");
    if (tail->out_dtype == FAA_U8_HWC && q.partner) return fail(FAA_ERR_UNSUPPORTED, "mixup needs a float output");
    if (batch > 0) { if (int e = check_alignment(q.in, q.out, w, tail)) return e; }
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (int e = bind_device(p)) return e;
    cudaStream_t stream = (cudaStream_t)q.stream;
    if (q.own_stream) { if (int e = follow_stream(p, stream)) return e; }
    const OpRec* d_ops = nullptr;
    // resolved samples can only reference ops the host sampler validated; Philox can pick anything
    if (int e = device_table(p, h, w, q.samples == nullptr, &d_ops)) return e;
    {   // per-image program buffer (grown, never shrunk; stream-ordered reuse)
        std::lock_guard<std::mutex> lk(p->mu);
        size_t need = (size_t)q.n_all * sizeof(Prog);
        if (p->d_progs_bytes < need) {
            if (p->d_progs) {
                CK(cudaStreamSynchronize(stream));
                if (p->ahead_stream) CK(cudaStreamSynchronize(p->ahead_stream));
                CK(cudaFree(p->d_progs)); CK(cudaFree(p->d_order));
                p->d_progs = p->d_order = nullptr; p->d_progs_bytes = 0;
            }
            need = need < 65536 ? 65536 : need * 2;
            CK(cudaMalloc(&p->d_progs, 2 * need));                                                // two slots (resolve-ahead)
            CK(cudaMalloc(&p->d_order, 2 * (4 * (need / sizeof(Prog)) * sizeof(int32_t) + 32)));  // order + 2 counters per launch + ready words, x2
            CK(cudaMemset(p->d_order, 0, 2 * (4 * (need / sizeof(Prog)) * sizeof(int32_t) + 32)));
            p->d_progs_bytes = need;
            p->ahead_valid = false;
            p->done_target[0] = p->done_target[1] = 0;      // (the completion counters live in d_order and start at zero)
        }
    }
    PlanInput in = {};
    in.H = h; in.W = w; in.out_h = tail->out_h; in.out_w = tail->out_w; in.out_u8 = tail->out_dtype == FAA_U8_HWC;
    in.batch = batch; in.crop_pad = std::min(h, std::max({0, tail->crop_pad, q.rng ? q.rng->crop_pad : 0}));
    in.in_mod16 = (uint32_t)((uintptr_t)q.in % 16); in.out_mod16 = (uint32_t)((uintptr_t)q.out % 16);
    in.two_src = q.partner != nullptr; in.apply_tail = q.apply_tail != 0; in.has_sg = p->has_sg;
    for (int t = 1; t < q.n_cands; ++t) in.has_sg = in.has_sg || q.cands[t]->has_sg;
    in.split_min = kSplitMin;
    if (const char* e = getenv("FAA_SPLIT_MIN")) in.split_min = strtoull(e, nullptr, 10);   // tests: force either path
    in.philox = q.rng && !q.samples; in.allow_ahead = q.allow_ahead;
    Schedule s{plan_launch(in)};
    AugParams P; memset(&P, 0, sizeof P);
    P.in = q.in; P.out = q.out; P.partner = q.partner;
    P.B = batch; P.H = h; P.W = w; P.out_h = tail->out_h; P.out_w = tail->out_w; P.first = q.first; P.in_mod = q.in_mod;
    P.use_zero_box = (tail->use_zero_box && q.apply_tail) ? 1 : 0;
    P.lam = q.lam; P.one_minus_lam = q.one_minus_lam;
    P.bands = s.geo[0].bands; P.geo[0] = s.geo[0]; P.geo[1] = s.geo[1];
    P.stage = s.stage; P.band_cap = s.geo[0].band_cap; P.crop_pad = in.crop_pad; P.octets = s.octets; P.mat_cap = s.mat_cap;
    P.allow = s.allow;
    // fastdiv reciprocals (host side: no divisions in the kernels)
    auto rcp = [](uint32_t d) { return d <= 1 ? 0u : (uint32_t)((0x100000000ull + d - 1) / d); };
    P.rcp_out_qpr = rcp((uint32_t)(tail->out_w + 3) / 4); P.rcp_w = rcp((uint32_t)w); P.rcp_wq = rcp((uint32_t)w / 4);
    P.rcp_opr = (w & 7) ? 0u : rcp((uint32_t)w / 8);
    P.pdl = 1;
    // launch 1: decisions -> programs (the whole pool when partners may be anywhere in it)
    ResolveParams R; memset(&R, 0, sizeof R);
    R.ops = d_ops; R.probs = p->d_probs;
    R.samples = reinterpret_cast<const Sample*>(q.samples); R.boxes = reinterpret_cast<const Box*>(q.boxes);
    if (q.rng) memcpy(&R.rng, q.rng, sizeof(RngCfg));
    R.first = q.partner ? 0 : q.first; R.n = q.partner ? q.n_all : batch;
    R.H = h; R.W = w; R.out_h = tail->out_h; R.out_w = tail->out_w;
    R.n_sub = p->n_sub; R.n_op = p->n_op; R.op_base = q.op_base; R.apply_tail = q.apply_tail;
    R.allow = s.allow; R.split = s.split;
    if (q.n_cands > 1) {
        if (int e = upload_candidates(p, q.cands, q.n_cands, h, w, stream, &R.cands)) return e;
        R.per_cand = q.per_cand;
        // the cluster kernel's self-resolving path draws from one policy: a multi-policy call always resolves first
        s.self_resolving = false;
    }
    if (s.scratch) {            // one scratch image per image, per program slot in the chained schedule
        s.scratch_slot_bytes = (size_t)q.n_all * h * w * 3;
        const size_t need = s.scratch_slot_bytes * (s.use_chain ? 2 : 1);
        if (p->d_scratch_bytes < need) {
            if (p->d_scratch) { CK(cudaStreamSynchronize(stream)); CK(cudaFree(p->d_scratch)); p->d_scratch = nullptr; p->d_scratch_bytes = 0; }
            CK(cudaMalloc(&p->d_scratch, need));
            p->d_scratch_bytes = need;
        }
        P.scratch = (uint8_t*)p->d_scratch;
    }
    if (tail->out_dtype != FAA_U8_HWC) { if (int e = normalisation(p, tail, P, s.use_tab, stream)) return e; }
    else { for (int c = 0; c < 3; ++c) { P.scale[c] = 1.0f; P.bias[c] = 0.0f; } }      // lean paths: the byte value itself
    if (p->lighting_rgb && tail->out_dtype != FAA_U8_HWC && q.apply_tail) {
        // Lighting (augmentations.py:197-215): one normalisation table per image, built on the stream in torch's fp32 order
        if (q.partner) return fail(FAA_ERR_UNSUPPORTED, "Lighting together with fused Mixup is not supported");
        if (p->lighting_n != q.n_all) return fail(FAA_ERR_VALUE, "faa_policy_set_lighting was given a different number of images");
        const size_t need = (size_t)q.n_all * 768 * sizeof(float);
        if (p->d_norm_img_bytes < need) {
            if (p->d_norm_img) { CK(cudaStreamSynchronize(stream)); CK(cudaFree(p->d_norm_img)); p->d_norm_img = nullptr; p->d_norm_img_bytes = 0; }
            CK(cudaMalloc(&p->d_norm_img, need));
            p->d_norm_img_bytes = need;
        }
        CK(launch_lighting_tables(p->lighting_rgb, p->d_norm_img, q.n_all, tail->mean, tail->std, stream));
        g_launches++;
        P.norm_tab = p->d_norm_img; P.norm_stride = 768;
        s.use_tab = true;
    }
    // fused Mixup mixes the fp32 normalised values before the output rounding: the fma shortcut is only proven to round
    // like the exact value for a DIRECT fp16 / bf16 store, so two-source launches always take the exact table
    if (q.partner) s.use_tab = true;
    if (s.self_resolving) return launch_self_resolving(p, P, R, s.use_tab, tail->out_dtype, stream);
    // resolve-ahead: did the previous call already resolve exactly this batch on the side stream?
    faa_policy::AheadKey key; memset(&key, 0, sizeof key);
    if (s.speculate) {
        key.seed = q.rng->seed; key.first_index = q.rng->first_index;
        const int32_t v[16] = {batch, q.n_all, q.first, h, w, tail->out_h, tail->out_w, q.op_base, q.apply_tail, R.allow,
                               R.split, q.rng->crop_pad, q.rng->hflip, q.rng->zero_box_len,
                               (s.use_order ? 1 : 0) | (q.in_mod << 1), (s.use_chain ? 1 : 0) | (P.norm_stride ? 2 : 0)};
        memcpy(key.v, v, sizeof v);
    }
    s.hit = s.speculate && p->ahead_valid && memcmp(&key, &p->ahead_key, sizeof key) == 0;
    if (s.use_chain) return launch_chained(p, P, R, s, key, tail->out_dtype, stream);
    return launch_event(p, P, R, s, key, tail->out_dtype, stream);
}

int faa_augment(faa_policy_t* p, const uint8_t* d_in, void* d_out, int batch, int h, int w, const faa_tail_t* tail,
                const faa_sample_t* d_samples, const faa_box_t* d_boxes, const faa_rng_t* rng, int op_base,
                void* stream) {
    if (!p) return fail(FAA_ERR_VALUE, "null policy");
    // intermediate launch of a chained policy = not the last 2-op window
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    int apply_tail = (op_base + FAA_MAX_FUSED_OPS >= p->n_op) ? 1 : 0;
    if (!apply_tail && tail && (tail->out_dtype != FAA_U8_HWC || tail->out_h != h || tail->out_w != w))
        return fail(FAA_ERR_VALUE, "intermediate launches of a chained policy must write uint8 HWC at the input size");
    AugRequest q;
    q.in = d_in; q.out = d_out; q.n_all = q.batch = batch; q.h = h; q.w = w; q.tail = tail;
    q.samples = d_samples; q.boxes = d_boxes; q.rng = rng; q.op_base = op_base; q.apply_tail = apply_tail;
    q.allow_ahead = p->n_op <= FAA_MAX_FUSED_OPS; q.stream = stream;
    return augment_common(p, q);
}

int faa_policy_set_overlap(faa_policy_t* p, int on) {
    if (!p) return fail(FAA_ERR_VALUE, "null policy");
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    p->overlap_calls = on != 0;
    return FAA_OK;
}

int faa_augment_many(faa_policy_t* p, int n_steps, const uint8_t* const* d_in, void* const* d_out, int batch, int h, int w,
                     const faa_tail_t* tail, const faa_rng_t* rng, uint64_t index_stride, void* stream) {
    if (!p || !rng || !d_in || !d_out) return fail(FAA_ERR_VALUE, "null argument");
    if (n_steps < 0) return fail(FAA_ERR_VALUE, "bad step count");
    if (p->n_op > FAA_MAX_FUSED_OPS) return fail(FAA_ERR_UNSUPPORTED, "multi-step launches support policies of at most 2 ops");
    if (batch > 0) {                                    // refuse before the first step is issued
        if (int e = check_tail(tail)) return e;
        for (int k = 0; k < n_steps; ++k) { if (int e = check_alignment(d_in[k], d_out[k], w, tail)) return e; }
    }
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    faa_rng_t r = *rng;
    AugRequest q;
    q.n_all = q.batch = batch; q.h = h; q.w = w; q.tail = tail; q.rng = &r; q.allow_ahead = true; q.stream = stream;
    const bool saved = p->overlap_calls;
    int rc = FAA_OK;
    for (int k = 0; k < n_steps && rc == FAA_OK; ++k) {
        // every input exists before this call: steps 2.. may overlap their predecessor; step 1 follows whatever the caller
        // issued before (stream order) unless the caller made the promise for whole calls too
        p->overlap_calls = k > 0 ? true : saved;
        q.in = d_in[k]; q.out = d_out[k];
        rc = augment_common(p, q);
        r.first_index += index_stride;
    }
    p->overlap_calls = saved;
    return rc;
}

int faa_augment_tta(faa_policy_t* p, const uint8_t* d_in, void* d_out, int batch, int replicas, int h, int w,
                    const faa_tail_t* tail, const faa_rng_t* rng, void* stream) {
    if (!p || !rng) return fail(FAA_ERR_VALUE, "null argument");
    if (p->n_op > FAA_MAX_FUSED_OPS) return fail(FAA_ERR_UNSUPPORTED, "replicated launches support policies of at most 2 ops");
    if (batch < 0 || replicas < 1) return fail(FAA_ERR_VALUE, "bad batch / replicas");
    if ((long long)batch * replicas > 65535) return fail(FAA_ERR_UNSUPPORTED, "batch * replicas must be <= 65535");
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    // one launch over batch * replicas schedule entries; entry v = r * batch + i reads image i and draws the decisions of
    // global sample first_index + v: replica r equals a plain launch with first_index + r * batch
    AugRequest q;
    q.in = d_in; q.out = d_out; q.n_all = q.batch = batch * replicas; q.h = h; q.w = w; q.tail = tail; q.rng = rng;
    q.allow_ahead = true; q.stream = stream; q.in_mod = replicas > 1 ? batch : 0;
    return augment_common(p, q);
}

// The candidate list of a multi-policy TTA call, checked on the host before anything touches the device.
static int check_candidates(faa_policy_t* const* policies, int n_policies) {
    if (!policies || n_policies < 1) return fail(FAA_ERR_VALUE, "need a non-empty list of candidate policies");
    for (int t = 0; t < n_policies; ++t) {
        if (!policies[t]) return fail(FAA_ERR_VALUE, "candidate " + std::to_string(t) + " is null");
        for (int u = 0; u < t; ++u)
            if (policies[u] == policies[t])
                return fail(FAA_ERR_VALUE, "candidates " + std::to_string(u) + " and " + std::to_string(t) + " are the same handle");
        if (policies[t]->n_op != policies[0]->n_op)
            return fail(FAA_ERR_VALUE, "every candidate needs the same n_op (candidate " + std::to_string(t) + " has " +
                                       std::to_string(policies[t]->n_op) + ", candidate 0 " + std::to_string(policies[0]->n_op) + ")");
    }
    if (policies[0]->n_op > FAA_MAX_FUSED_OPS)
        return fail(FAA_ERR_UNSUPPORTED, "replicated launches support policies of at most 2 ops");
    return FAA_OK;
}

int faa_augment_tta_policies(faa_policy_t* const* policies, int n_policies, const uint8_t* d_in, void* d_out, int batch,
                             int replicas, int h, int w, const faa_tail_t* tail, const faa_rng_t* rng, void* stream) {
    if (int e = check_candidates(policies, n_policies)) return e;
    if (!rng) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0 || replicas < 1) return fail(FAA_ERR_VALUE, "bad batch / replicas");
    if ((long long)n_policies * batch * replicas > 65535)
        return fail(FAA_ERR_UNSUPPORTED, "n_policies * replicas * batch must be <= 65535");
    if (n_policies == 1) return faa_augment_tta(policies[0], d_in, d_out, batch, replicas, h, w, tail, rng, stream);
    faa_policy* p = policies[0];
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    // one launch over n_policies * replicas * batch entries; entry v = (t * replicas + r) * batch + i reads image i and
    // draws the decisions of global sample first_index + v from candidate t.  No resolve-ahead: its speculation is keyed
    // by the handle's own policy.
    AugRequest q;
    q.in = d_in; q.out = d_out; q.n_all = q.batch = n_policies * replicas * batch; q.h = h; q.w = w; q.tail = tail;
    q.rng = rng; q.stream = stream; q.in_mod = batch;
    q.cands = policies; q.n_cands = n_policies; q.per_cand = replicas * batch;
    return augment_common(p, q);
}

int faa_augment_mixup(faa_policy_t* p, const uint8_t* d_in_all, int n_all, int first, void* d_out, int batch, int h,
                      int w, const faa_tail_t* tail, const faa_sample_t* d_samples_all, const faa_box_t* d_boxes_all,
                      const faa_rng_t* rng, const int32_t* d_partner, float lam, float one_minus_lam, void* stream) {
    if (!p) return fail(FAA_ERR_VALUE, "null policy");
    if (p->n_op > FAA_MAX_FUSED_OPS) return fail(FAA_ERR_UNSUPPORTED, "fused mixup supports policies of at most 2 ops");
    if (!(lam >= 0.0f && lam <= 1.0f)) return fail(FAA_ERR_MAGNITUDE, "lam must be in [0, 1]");   // aug_mixup.py:20
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    AugRequest q;
    q.in = d_in_all; q.out = d_out; q.n_all = n_all; q.first = first; q.batch = batch; q.h = h; q.w = w; q.tail = tail;
    q.samples = d_samples_all; q.boxes = d_boxes_all; q.rng = rng; q.stream = stream;
    q.partner = d_partner; q.lam = lam; q.one_minus_lam = one_minus_lam;
    return augment_common(p, q);
}

int faa_policy_set_lighting(faa_policy_t* p, const float* d_rgb, int n) {
    if (!p) return fail(FAA_ERR_VALUE, "null policy");
    if (d_rgb && n <= 0) return fail(FAA_ERR_VALUE, "n must be positive");
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    p->lighting_rgb = d_rgb; p->lighting_n = d_rgb ? n : 0;
    return FAA_OK;
}

int faa_color_jitter(const uint8_t* d_in, uint8_t* d_out, int batch, int h, int w, const faa_jitter_t* d_recs, void* stream) {
    if ((!d_in || !d_out || !d_recs) && batch > 0) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (int e = check_shape(h, w)) return e;
    if (int e = ensure_device()) return e;
    static_assert(sizeof(faa_jitter_t) == 16, "jitter record is 16 bytes");
    CK(launch_color_jitter(d_in, d_out, d_recs, batch, h, w, (cudaStream_t)stream));
    if (batch > 0) g_launches++;
    return FAA_OK;
}

static_assert(sizeof(faa_crop_box_t) == sizeof(CropBox), "crop box layout");
static_assert(sizeof(faa_crop_cfg_t) == sizeof(CropCfg) && offsetof(faa_crop_cfg_t, rng) == offsetof(CropCfg, rng),
              "crop config layout");

int faa_center_crop_box(int h, int w, int img_size, faa_crop_box_t* out) {
    if (!out) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_shape(h, w)) return e;
    if (img_size <= 0) return fail(FAA_ERR_VALUE, "img_size must be positive");
    CropBox b = center_crop_box(h, w, img_size);
    memcpy(out, &b, sizeof b);
    return FAA_OK;
}

static int check_crop_cfg(const faa_crop_cfg_t* c) {
    if (c->mode != FAA_CROP_RANDOM && c->mode != FAA_CROP_CENTER) return fail(FAA_ERR_VALUE, "bad crop mode");
    if (c->img_size <= 0) return fail(FAA_ERR_VALUE, "img_size must be positive");
    if (c->mode == FAA_CROP_RANDOM) {                       // the reference's asserts (data.py:269-272)
        if (!(c->min_covered > 0.0)) return fail(FAA_ERR_MAGNITUDE, "min_covered must be positive");
        if (!(c->aspect_lo > 0.0 && c->aspect_lo <= c->aspect_hi)) return fail(FAA_ERR_MAGNITUDE, "bad aspect_ratio_range");
        if (!(c->area_lo > 0.0 && c->area_lo <= c->area_hi)) return fail(FAA_ERR_MAGNITUDE, "bad area_range");
        if (c->max_attempts < 1) return fail(FAA_ERR_MAGNITUDE, "max_attempts must be >= 1");
    }
    return FAA_OK;
}

// the output and crop configuration of a crop-resize call
static int check_crop_resize(const faa_tail_t* tail, const faa_crop_cfg_t* cfg) {
    if (int e = check_tail(tail)) return e;
    if (int e = check_crop_cfg(cfg)) return e;
    if (tail->out_dtype != FAA_U8_HWC)
        for (int c = 0; c < 3; ++c)
            if (!(tail->std[c] != 0.0f)) return fail(FAA_ERR_VALUE, "std must be non-zero");
    return FAA_OK;
}

// Boxes the kernel draws: the device sampler's boxes lie inside the image; the center box (center mode, and the random
// mode's fallback after failed attempts) can be empty when img_size is small against the short side.
static bool center_box_empty(int h, int w, const faa_crop_cfg_t* cfg) {
    const CropBox b = center_crop_box(h, w, cfg->img_size);
    return b.w <= 0 || b.h <= 0;
}

// Given boxes (device memory): copied back and checked against image i's own size (images[i], or h x w for every image
// when images is null); the host waits for the stream.
static int check_given_boxes(const faa_crop_box_t* d_boxes, int batch, const faa_image_t* images, int h, int w,
                             cudaStream_t stream) {
    std::vector<CropBox> hb((size_t)batch);
    CK(cudaMemcpyAsync(hb.data(), d_boxes, hb.size() * sizeof(CropBox), cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    for (int i = 0; i < batch; ++i) {
        const CropBox& b = hb[(size_t)i];
        const int ih = images ? (int)images[i].h : h, iw = images ? (int)images[i].w : w;
        if (b.w <= 0 || b.h <= 0 || b.x0 < 0 || b.y0 < 0 || b.x0 > iw - b.w || b.y0 > ih - b.h)
            return fail(FAA_ERR_VALUE, "crop box " + std::to_string(i) + " is empty or not inside the image");
    }
    return FAA_OK;
}

int faa_crop_resize(const uint8_t* d_in, void* d_out, int batch, int h, int w, const faa_tail_t* tail,
                    const faa_crop_box_t* d_boxes, const faa_crop_cfg_t* cfg, void* stream) {
    if (!cfg || ((!d_in || !d_out) && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "batch must be <= 65535");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_crop_resize(tail, cfg)) return e;
    if (!d_boxes && center_box_empty(h, w, cfg)) return fail(FAA_ERR_VALUE, "the center crop of this image is empty");
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (d_boxes)
        if (int e = check_given_boxes(d_boxes, batch, nullptr, h, w, (cudaStream_t)stream))
            return e;
    const CropResizeTile t = plan_crop_resize(h, w, tail->out_h, tail->out_w);
    if (t.smem == 0) return fail(FAA_ERR_UNSUPPORTED, "no crop-resize tile fits in shared memory");
    CropCfg c; memcpy(&c, cfg, sizeof c);
    CK(launch_crop_resize(d_in, nullptr, d_out, batch, h, w, tail->out_h, tail->out_w, tail->out_dtype, tail->mean,
                          tail->std, reinterpret_cast<const CropBox*>(d_boxes), c, t, (cudaStream_t)stream));
    g_launches++;
    return FAA_OK;
}

static_assert(sizeof(faa_image_t) == 16 && sizeof(CropImage) == 16 && offsetof(faa_image_t, h) == offsetof(CropImage, h),
              "image descriptor layout");

int faa_crop_resize_ragged(const faa_image_t* h_images, const faa_image_t* d_images, int batch, void* d_out,
                           const faa_tail_t* tail, const faa_crop_box_t* d_boxes, const faa_crop_cfg_t* cfg, void* stream) {
    if (!cfg || ((!h_images || !d_images || !d_out) && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "batch must be <= 65535");
    if (int e = check_crop_resize(tail, cfg)) return e;
    int max_h = 1, max_w = 1;
    for (int i = 0; i < batch; ++i) {
        const faa_image_t& m = h_images[i];
        if (!m.data) return fail(FAA_ERR_VALUE, "image " + std::to_string(i) + " has no data");
        if (int e = check_shape(m.h, m.w)) return e;
        if (!d_boxes && center_box_empty(m.h, m.w, cfg))
            return fail(FAA_ERR_VALUE, "the center crop of image " + std::to_string(i) + " is empty");
        max_h = std::max(max_h, (int)m.h); max_w = std::max(max_w, (int)m.w);
    }
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (d_boxes)
        if (int e = check_given_boxes(d_boxes, batch, h_images, 0, 0, (cudaStream_t)stream))
            return e;
    const CropResizeTile t = plan_crop_resize(max_h, max_w, tail->out_h, tail->out_w);
    if (t.smem == 0) return fail(FAA_ERR_UNSUPPORTED, "no crop-resize tile fits in shared memory");
    CropCfg c; memcpy(&c, cfg, sizeof c);
    CK(launch_crop_resize(nullptr, reinterpret_cast<const CropImage*>(d_images), d_out, batch, max_h, max_w, tail->out_h,
                          tail->out_w, tail->out_dtype, tail->mean, tail->std, reinterpret_cast<const CropBox*>(d_boxes), c,
                          t, (cudaStream_t)stream));
    g_launches++;
    return FAA_OK;
}

static size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// faa_augment_ragged, and faa_augment_ragged_policies when n_cands > 1: image i then draws with candidate
// cands[h_cand[i]] (cands[0] == p runs the call, the others lend their device tables)
static int augment_ragged(faa_policy_t* p, faa_policy_t* const* cands, int n_cands, const int32_t* h_cand,
                          const faa_image_t* h_in, const faa_image_t* d_in, int batch, const faa_image_t* h_out,
                          const faa_image_t* d_out, const faa_sample_t* d_samples, const faa_box_t* d_boxes,
                          const faa_rng_t* rng, int op_base, void* stream_v) {
    if (!p || ((!h_in || !d_in || !h_out || !d_out) && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "at most 65535 images per call (one grid row per image): split the batch");
    if (!d_samples && !rng) return fail(FAA_ERR_VALUE, "need either resolved samples or an rng config");
    if (rng && !d_samples && (rng->crop_pad != 0 || rng->hflip != 0 || rng->zero_box_len != 0))
        return fail(FAA_ERR_VALUE, "a ragged launch writes every image at its own size: the rng must have no crop_pad, hflip or "
                                   "zero_box_len");
    if (op_base < 0 || op_base >= p->n_op) return fail(FAA_ERR_VALUE, "op_base out of range");
    std::vector<RaggedImageIn> ins((size_t)batch);
    for (int i = 0; i < batch; ++i) {
        const faa_image_t& a = h_in[i];
        const faa_image_t& o = h_out[i];
        const std::string who = "image " + std::to_string(i);
        if (!a.data || !o.data) return fail(FAA_ERR_VALUE, who + " has no data");
        if (check_shape(a.h, a.w)) return fail(FAA_ERR_VALUE, who + " has a size out of range");
        if (o.h != a.h || o.w != a.w) return fail(FAA_ERR_VALUE, "output " + who + " is not the size of its input");
        if ((a.w & 3) == 0 && ((uintptr_t)o.data & 3))
            return fail(FAA_ERR_UNSUPPORTED, "output " + who + " must be 4-byte aligned when its width is a multiple of 4 "
                                             "(vector stores)");
        ins[(size_t)i] = {a.h, a.w, (uint32_t)((uintptr_t)a.data % 16), (uint32_t)((uintptr_t)o.data % 16)};
    }
    const bool multi = n_cands > 1;
    if (multi)
        for (int i = 0; i < batch; ++i)
            if (h_cand[i] < 0 || h_cand[i] >= n_cands)
                return fail(FAA_ERR_VALUE, "image " + std::to_string(i) + " names candidate " + std::to_string(h_cand[i]) +
                                           " of " + std::to_string(n_cands));
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (int e = bind_device(p)) return e;
    for (int t = 1; t < n_cands; ++t) { if (int e = bind_device(cands[t])) return e; }
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    cudaStream_t stream = (cudaStream_t)stream_v;
    if (int e = follow_stream(p, stream)) return e;
    bool has_sg = p->has_sg;
    for (int t = 1; t < n_cands; ++t) has_sg = has_sg || cands[t]->has_sg;
    const RaggedPlan plan = plan_ragged(ins.data(), batch, has_sg);

    // per-size launch parameters (in / out / progs / scratch are patched in per image by the kernel)
    const size_t n_geo = plan.geoms.size();
    const int n_tab = multi ? n_cands : 1;
    std::vector<const OpRec*> geo_ops((size_t)n_tab * n_geo);      // [candidate][size]
    std::vector<AugParams> geo(n_geo);
    for (size_t k = 0; k < n_geo; ++k) {
        const RaggedGeom& g = plan.geoms[k];
        // resolved samples can only reference ops the host sampler validated; Philox can pick anything
        for (int t = 0; t < n_tab; ++t)
            if (int e = device_table(multi ? cands[t] : p, g.H, g.W, d_samples == nullptr, &geo_ops[(size_t)t * n_geo + k]))
                return e;
        AugParams& a = geo[k];
        memset(&a, 0, sizeof a);
        a.B = 1; a.H = a.out_h = g.H; a.W = a.out_w = g.W;
        a.bands = g.plan.geo[0].bands; a.geo[0] = g.plan.geo[0]; a.geo[1] = g.plan.geo[1];
        a.stage = g.plan.stage; a.band_cap = g.plan.geo[0].band_cap; a.octets = g.plan.octets; a.mat_cap = g.plan.mat_cap;
        a.rcp_out_qpr = g.rcp_out_qpr; a.rcp_w = g.rcp_w; a.rcp_wq = g.rcp_wq; a.rcp_opr = g.rcp_opr;
        for (int c = 0; c < 3; ++c) { a.scale[c] = 1.0f; a.bias[c] = 0.0f; }      // uint8 output: the byte value itself
    }
    // per image: scratch images (Sharpness -> gather) and re-aligned copies of inputs whose base breaks the 32-bit loads
    // of W % 4 == 0 images, as byte offsets into the handle's buffers.  Descriptors that share a source (the replicas of
    // a TTA batch) share its copy: each distinct (base, bytes) is copied once.
    std::vector<int64_t> scratch_at((size_t)batch, -1), copy_at((size_t)batch, -1);
    std::vector<int> copy_src;                                  // the first image of each copied source
    std::map<std::pair<const uint8_t*, size_t>, int64_t> copied;
    size_t scratch_bytes = 0, copy_bytes = 0;
    for (int i = 0; i < batch; ++i) {
        const RaggedGeom& g = plan.geoms[(size_t)plan.geom_of[(size_t)i]];
        const size_t bytes = (size_t)g.H * g.W * 3;
        if (g.plan.scratch) { scratch_at[(size_t)i] = (int64_t)scratch_bytes; scratch_bytes += align16(bytes); }
        if ((g.W & 3) == 0 && ((uintptr_t)h_in[i].data & 3)) {
            const auto at = copied.emplace(std::make_pair(h_in[i].data, bytes), (int64_t)copy_bytes);
            if (at.second) { copy_bytes += align16(bytes); copy_src.push_back(i); }
            copy_at[(size_t)i] = at.first->second;
        }
    }
    const int n_copy = (int)copy_src.size();
    const size_t off_img = align16(n_geo * sizeof(AugParams));
    const size_t off_list = off_img + align16((size_t)batch * sizeof(RaggedImg));
    const size_t off_copy = off_list + align16((size_t)batch * sizeof(int32_t));
    // multi-policy calls: the candidates' probabilities and n_sub, and each image's candidate
    const size_t off_refs = align16(off_copy + (size_t)n_copy * sizeof(RaggedCopy));
    const size_t off_cand = off_refs + align16((size_t)n_tab * sizeof(PolicyRef));
    const size_t tab_bytes = multi ? off_cand + (size_t)batch * sizeof(int32_t) : off_copy + (size_t)n_copy * sizeof(RaggedCopy);
    if (int e = grow_on_stream(&p->d_rg_tab, &p->d_rg_tab_bytes, tab_bytes, stream)) return e;
    if (int e = grow_on_stream(&p->d_rg_progs, &p->d_rg_progs_bytes, (size_t)batch * sizeof(Prog), stream)) return e;
    if (scratch_bytes) { if (int e = grow_on_stream(&p->d_rg_scratch, &p->d_rg_scratch_bytes, scratch_bytes, stream)) return e; }
    if (copy_bytes) { if (int e = grow_on_stream(&p->d_rg_copy, &p->d_rg_copy_bytes, copy_bytes, stream)) return e; }
    uint8_t* d_tab = (uint8_t*)p->d_rg_tab;
    std::vector<uint8_t> host(tab_bytes, 0);
    memcpy(host.data(), geo.data(), n_geo * sizeof(AugParams));
    RaggedImg* imgs = reinterpret_cast<RaggedImg*>(host.data() + off_img);
    RaggedCopy* copies = reinterpret_cast<RaggedCopy*>(host.data() + off_copy);
    for (int i = 0; i < batch; ++i) {
        const int k = plan.geom_of[(size_t)i];
        RaggedImg& m = imgs[i];
        m.ops = geo_ops[(size_t)(multi ? h_cand[i] : 0) * n_geo + k]; m.H = plan.geoms[(size_t)k].H; m.W = plan.geoms[(size_t)k].W;
        m.allow = plan.geoms[(size_t)k].plan.allow; m.geom = k;
        m.scratch = scratch_at[(size_t)i] < 0 ? nullptr : (uint8_t*)p->d_rg_scratch + scratch_at[(size_t)i];
        m.realigned = copy_at[(size_t)i] < 0 ? nullptr : (uint8_t*)p->d_rg_copy + copy_at[(size_t)i];
    }
    for (int c = 0; c < n_copy; ++c) {
        const int i = copy_src[(size_t)c];
        copies[c] = {h_in[i].data, (uint8_t*)p->d_rg_copy + copy_at[(size_t)i], (uint64_t)imgs[i].H * imgs[i].W * 3};
    }
    memcpy(host.data() + off_list, plan.order.data(), (size_t)batch * sizeof(int32_t));
    if (multi) {
        PolicyRef* refs = reinterpret_cast<PolicyRef*>(host.data() + off_refs);
        for (int t = 0; t < n_cands; ++t) refs[t] = {nullptr, cands[t]->d_probs, cands[t]->n_sub, 0};
        memcpy(host.data() + off_cand, h_cand, (size_t)batch * sizeof(int32_t));
    }
    CK(cudaMemcpyAsync(d_tab, host.data(), tab_bytes, cudaMemcpyHostToDevice, stream));   // (pageable: staged at once)
    const RaggedImg* d_imgs = reinterpret_cast<const RaggedImg*>(d_tab + off_img);
    if (n_copy) {
        CK(launch_realign(reinterpret_cast<const RaggedCopy*>(d_tab + off_copy), n_copy, stream));
        g_launches++;
    }
    // decisions -> programs, each image at its own size (Philox: global sample first_index + batch position)
    ResolveParams R; memset(&R, 0, sizeof R);
    R.probs = p->d_probs;
    R.samples = reinterpret_cast<const Sample*>(d_samples); R.boxes = reinterpret_cast<const Box*>(d_boxes);
    if (rng) memcpy(&R.rng, rng, sizeof(RngCfg));
    R.progs = reinterpret_cast<Prog*>(p->d_rg_progs); R.first = 0; R.n = batch;
    R.n_sub = p->n_sub; R.n_op = p->n_op; R.op_base = op_base;
    R.apply_tail = (op_base + FAA_MAX_FUSED_OPS >= p->n_op) ? 1 : 0;
    if (multi) {
        R.cands = reinterpret_cast<const PolicyRef*>(d_tab + off_refs);
        R.cand_of = reinterpret_cast<const int32_t*>(d_tab + off_cand);
    }
    CK(launch_resolve_ragged(R, d_imgs, stream));
    g_launches++;
    // pixels: one cluster-kernel launch per band count, largest images first
    for (const RaggedLaunch& L : plan.launches) {
        RaggedParams rp;
        rp.geoms = reinterpret_cast<const AugParams*>(d_tab); rp.imgs = d_imgs;
        rp.in = reinterpret_cast<const CropImage*>(d_in); rp.out = reinterpret_cast<const CropImage*>(d_out);
        rp.progs = reinterpret_cast<const Prog*>(p->d_rg_progs);
        rp.list = reinterpret_cast<const int32_t*>(d_tab + off_list) + L.first;
        CK(launch_augment_ragged(rp, L.bands, L.count, L.smem, stream));
        g_launches++;
    }
    p->chain_live = false;                  // the next chained step follows this call in stream order
    return FAA_OK;
}

int faa_augment_ragged(faa_policy_t* p, const faa_image_t* h_in, const faa_image_t* d_in, int batch,
                       const faa_image_t* h_out, const faa_image_t* d_out, const faa_sample_t* d_samples,
                       const faa_box_t* d_boxes, const faa_rng_t* rng, int op_base, void* stream) {
    return augment_ragged(p, nullptr, 1, nullptr, h_in, d_in, batch, h_out, d_out, d_samples, d_boxes, rng, op_base, stream);
}

int faa_augment_ragged_policies(faa_policy_t* const* policies, int n_policies, const faa_image_t* h_in,
                                const faa_image_t* d_in, const int32_t* h_policy, int batch, const faa_image_t* h_out,
                                const faa_image_t* d_out, const faa_rng_t* rng, void* stream) {
    if (int e = check_candidates(policies, n_policies)) return e;
    if (!rng || (!h_policy && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (n_policies == 1) {
        for (int i = 0; i < batch; ++i)
            if (h_policy[i] != 0) return fail(FAA_ERR_VALUE, "image " + std::to_string(i) + " names candidate " +
                                                              std::to_string(h_policy[i]) + " of 1");
        return faa_augment_ragged(policies[0], h_in, d_in, batch, h_out, d_out, nullptr, nullptr, rng, 0, stream);
    }
    return augment_ragged(policies[0], policies, n_policies, h_policy, h_in, d_in, batch, h_out, d_out, nullptr, nullptr,
                          rng, 0, stream);
}

int faa_mix_u8(faa_policy_t* p, const uint8_t* d_a, const uint8_t* d_b, const int32_t* d_partner, const int16_t* d_zero_box_a,
               const int16_t* d_zero_box_b, void* d_out, int batch, int h, int w, const faa_tail_t* tail, float lam,
               float one_minus_lam, void* stream) {
    if (!p || ((!d_a || !d_b || !d_partner || !d_out) && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_tail(tail)) return e;
    if (tail->out_dtype == FAA_U8_HWC) return fail(FAA_ERR_UNSUPPORTED, "mixup needs a float output");
    if (tail->out_h != h || tail->out_w != w) return fail(FAA_ERR_VALUE, "the augmented images already have the output size");
    if ((w & 3) || ((uintptr_t)d_a & 3) || ((uintptr_t)d_b & 3) || ((uintptr_t)d_out & 15))
        return fail(FAA_ERR_UNSUPPORTED, "faa_mix_u8 needs W % 4 == 0 and aligned buffers");
    if (!(lam >= 0.0f && lam <= 1.0f)) return fail(FAA_ERR_MAGNITUDE, "lam must be in [0, 1]");   // aug_mixup.py:20
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (int e = bind_device(p)) return e;
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    AugParams dummy; bool tab = false;
    if (int e = normalisation(p, tail, dummy, tab, (cudaStream_t)stream)) return e;
    CK(launch_mix_u8(d_a, d_b, d_partner, d_zero_box_a, d_zero_box_b, p->d_norm, d_out, batch, h, w, tail->out_dtype, lam,
                     one_minus_lam, (cudaStream_t)stream));
    g_launches++;
    return FAA_OK;
}

int faa_enable_peer_access(int peer_device) {
    if (int e = ensure_device()) return e;
    int dev = -1, can = 0;
    CK(cudaGetDevice(&dev));
    if (peer_device == dev) return FAA_OK;
    CK(cudaDeviceCanAccessPeer(&can, dev, peer_device));
    if (!can) return fail(FAA_ERR_UNSUPPORTED, "device " + std::to_string(dev) + " cannot access the memory of device " + std::to_string(peer_device));
    cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return FAA_OK; }
    CK(e);
    return FAA_OK;
}

// ---- buffers other processes of the node can map (CUDA IPC): the Mixup partner pool -------------------------------
int faa_peer_alloc(size_t bytes, void** d_ptr, unsigned char* handle64) {
    if (!d_ptr || !handle64 || bytes == 0) return fail(FAA_ERR_VALUE, "bad argument");
    if (int e = ensure_device()) return e;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    void* p = nullptr;
    CK(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    if (cudaError_t e = cudaIpcGetMemHandle(&h, p)) { cudaFree(p); CK(e); }
    CK(cudaMemset(p, 0, bytes));
    memcpy(handle64, &h, 64);
    *d_ptr = p;
    return FAA_OK;
}

int faa_peer_open(const unsigned char* handle64, void** d_ptr) {
    if (!d_ptr || !handle64) return fail(FAA_ERR_VALUE, "bad argument");
    if (int e = ensure_device()) return e;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    // opened under the CURRENT device: lazy peer access lets this device's kernels dereference the mapping
    CK(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return FAA_OK;
}

int faa_peer_close(void* d_ptr) { if (d_ptr) CK(cudaIpcCloseMemHandle(d_ptr)); return FAA_OK; }
int faa_peer_free(void* d_ptr) { if (d_ptr) CK(cudaFree(d_ptr)); return FAA_OK; }

static_assert(sizeof(faa_copy_t) == sizeof(RaggedCopy) && sizeof(faa_copy_t) == 24, "copy job layout");

int faa_gather(const faa_copy_t* h_jobs, const faa_copy_t* d_jobs, int n, void* stream) {
    if (!h_jobs || !d_jobs) return fail(FAA_ERR_VALUE, "null argument");
    if (n <= 0) return fail(FAA_ERR_VALUE, "faa_gather needs at least one job");
    uint64_t pieces = 0;
    for (int i = 0; i < n; ++i) {
        if (!h_jobs[i].src || !h_jobs[i].dst) return fail(FAA_ERR_VALUE, "job " + std::to_string(i) + ": null src or dst");
        pieces += (h_jobs[i].bytes + kGatherUnit - 1) / kGatherUnit;
    }
    if (int e = ensure_device()) return e;
    if (pieces == 0) return FAA_OK;
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const uint64_t ctas = std::min<uint64_t>(pieces, (uint64_t)sms * 8);    // 8 CTAs of 256 threads fill an SM
    CK(launch_gather(reinterpret_cast<const RaggedCopy*>(d_jobs), n, (int)ctas, (cudaStream_t)stream));
    g_launches++;
    return FAA_OK;
}

int faa_mix_u8_peer(faa_policy_t* p, const uint8_t* d_a, const uint8_t* const* d_partner_ptrs, const int16_t* d_zero_box_a,
                    const int16_t* d_zero_box_b, void* d_out, int batch, int h, int w, const faa_tail_t* tail, float lam,
                    float one_minus_lam, void* stream) {
    if (!p || ((!d_a || !d_partner_ptrs || !d_out) && batch > 0)) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_tail(tail)) return e;
    if (tail->out_dtype == FAA_U8_HWC) return fail(FAA_ERR_UNSUPPORTED, "mixup needs a float output");
    if (tail->out_h != h || tail->out_w != w) return fail(FAA_ERR_VALUE, "the augmented images already have the output size");
    if ((w & 3) || ((uintptr_t)d_a & 3) || ((uintptr_t)d_out & 15) || ((uintptr_t)d_partner_ptrs & 7))
        return fail(FAA_ERR_UNSUPPORTED, "faa_mix_u8_peer needs W % 4 == 0 and aligned buffers");
    if (!(lam >= 0.0f && lam <= 1.0f)) return fail(FAA_ERR_MAGNITUDE, "lam must be in [0, 1]");   // aug_mixup.py:20
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    if (int e = bind_device(p)) return e;
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    AugParams dummy; bool tab = false;
    if (int e = normalisation(p, tail, dummy, tab, (cudaStream_t)stream)) return e;
    CK(launch_mix_u8(d_a, nullptr, nullptr, d_zero_box_a, d_zero_box_b, p->d_norm, d_out, batch, h, w, tail->out_dtype, lam,
                     one_minus_lam, (cudaStream_t)stream, d_partner_ptrs));
    g_launches++;
    return FAA_OK;
}

int faa_mixup(const void* d_data, void* d_out, const int64_t* d_perm, int batch, int64_t n_per_sample, int dtype,
              float lam, float one_minus_lam, void* stream) {
    if ((!d_data || !d_out || !d_perm) && batch > 0) return fail(FAA_ERR_VALUE, "null argument");
    if (batch < 0 || n_per_sample < 0) return fail(FAA_ERR_VALUE, "negative size");
    if (dtype < 0 || dtype > FAA_F32) return fail(FAA_ERR_VALUE, "bad dtype");
    if (int e = ensure_device()) return e;
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "at most 65535 images per call (one grid row per image): split the batch");
    // a CTA may still be reading a sample as another CTA's partner when its own output is written: no in-place mixing
    const uintptr_t bytes = (uintptr_t)batch * (uintptr_t)n_per_sample * (dtype == FAA_F32 ? 4u : 2u);
    const uintptr_t lo_in = (uintptr_t)d_data, lo_out = (uintptr_t)d_out;
    if (bytes > 0 && lo_out < lo_in + bytes && lo_in < lo_out + bytes)
        return fail(FAA_ERR_VALUE, "out overlaps data: a sample would be overwritten while another reads it as its partner");
    CK(launch_mixup(d_data, d_out, d_perm, batch, n_per_sample, dtype, lam, one_minus_lam, (cudaStream_t)stream));
    if (batch > 0 && n_per_sample > 0) g_launches++;
    return FAA_OK;
}

// ------------------------------------------------------------- host buffers --
static int grow_dev(void** ptr, size_t* have, size_t need) {
    if (*have >= need) return FAA_OK;
    if (*ptr) { CK(cudaFree(*ptr)); *ptr = nullptr; *have = 0; }
    CK(cudaMalloc(ptr, need));
    *have = need;
    return FAA_OK;
}
static int grow_pinned(void** ptr, size_t* have, size_t need) {
    if (*have >= need) return FAA_OK;
    if (*ptr) { CK(cudaFreeHost(*ptr)); *ptr = nullptr; *have = 0; }
    CK(cudaMallocHost(ptr, need));
    *have = need;
    return FAA_OK;
}
static bool is_pinned(const void* ptr) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

int faa_augment_host(faa_policy_t* p, const uint8_t* h_in, void* h_out, void* d_out_keep, int batch, int h, int w,
                     const faa_tail_t* tail, const faa_rng_t* rng, void* stream_v) {
    if (!p || !h_in || !rng) return fail(FAA_ERR_VALUE, "null argument");
    if (p->n_op > FAA_MAX_FUSED_OPS) return fail(FAA_ERR_UNSUPPORTED, "host-buffer entry supports policies of at most 2 ops");
    if (int e = check_shape(h, w)) return e;
    if (int e = check_tail(tail)) return e;
    // (the device input is the policy's own allocation; a caller-owned device output is checked up front, before any
    //  chunk is issued)
    if (d_out_keep && batch > 0) { if (int e = check_alignment(nullptr, d_out_keep, w, tail)) return e; }
    if (int e = ensure_device()) return e;
    if (batch <= 0) return FAA_OK;
    if (int e = bind_device(p)) return e;
    cudaStream_t stream = (cudaStream_t)stream_v;
    std::lock_guard<std::mutex> call_lk(p->call_mu);
    // The policy owns the device input buffer and the pinned stages: the previous call's asynchronous copies must
    // have finished before any of them is rewritten (a pageable source is memcpy'd into the stage right below)
    if (p->host_in_flight) { CK(cudaEventSynchronize(p->ev_host_done)); p->host_in_flight = false; }
    if (int e = follow_stream(p, stream)) return e;        // (the side streams fork from `stream` below)
    if (!p->ev_host_done) CK(cudaEventCreateWithFlags(&p->ev_host_done, cudaEventDisableTiming));
    const size_t in_img = (size_t)h * w * 3;
    const size_t out_img = (size_t)tail->out_h * tail->out_w * 3 * out_elem_size(tail->out_dtype);
    if (int e = grow_dev(&p->d_in, &p->d_in_bytes, in_img * batch)) return e;
    void* d_out = d_out_keep;
    if (!d_out) { if (int e = grow_dev(&p->d_out, &p->d_out_bytes, out_img * batch)) return e; d_out = p->d_out; }
    for (int i = 0; i < 2; ++i) {
        if (!p->side[i]) CK(cudaStreamCreateWithFlags(&p->side[i], cudaStreamNonBlocking));
        if (!p->ev_join[i]) CK(cudaEventCreateWithFlags(&p->ev_join[i], cudaEventDisableTiming));
    }
    if (!p->ev_fork) CK(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));

    // pageable buffers are staged through pinned memory (synchronous host copies)
    const bool in_pinned = is_pinned(h_in);
    const bool out_pinned = !h_out || is_pinned(h_out);
    const uint8_t* src = h_in;
    if (!in_pinned) {
        if (int e = grow_pinned(&p->h_in_stage, &p->h_in_bytes, in_img * batch)) return e;
        memcpy(p->h_in_stage, h_in, in_img * batch);
        src = (const uint8_t*)p->h_in_stage;
    }
    void* dst = h_out;
    if (h_out && !out_pinned) {
        if (int e = grow_pinned(&p->h_out_stage, &p->h_out_bytes, out_img * batch)) return e;
        dst = p->h_out_stage;
    }

    // tables the side streams will read are uploaded on `stream` before the fork
    if (tail->out_dtype != FAA_U8_HWC) {
        AugParams dummy; bool tab = false;
        if (int e = normalisation(p, tail, dummy, tab, stream)) return e;
    }
    {
        const OpRec* d_ops = nullptr;
        if (int e = device_table(p, h, w, true, &d_ops)) return e;
    }
    // chunked pipeline on two side streams: H2D(c+1) overlaps kernel(c) and D2H(c)
    int chunks = batch >= 64 ? 8 : (batch >= 8 ? 2 : 1);
    CK(cudaEventRecord(p->ev_fork, stream));
    CK(cudaStreamWaitEvent(p->side[0], p->ev_fork, 0));
    CK(cudaStreamWaitEvent(p->side[1], p->ev_fork, 0));
    AugRequest q;
    q.in = (const uint8_t*)p->d_in; q.n_all = batch; q.h = h; q.w = w; q.tail = tail; q.rng = rng; q.own_stream = false;
    for (int c = 0; c < chunks; ++c) {
        int b0 = (int)((long long)batch * c / chunks), b1 = (int)((long long)batch * (c + 1) / chunks);
        if (b1 <= b0) continue;
        cudaStream_t s = p->side[c & 1];
        CK(cudaMemcpyAsync((uint8_t*)p->d_in + in_img * b0, src + in_img * b0, in_img * (b1 - b0), cudaMemcpyHostToDevice, s));
        q.out = (uint8_t*)d_out + out_img * b0; q.first = b0; q.batch = b1 - b0; q.stream = s;
        if (int e = augment_common(p, q)) return e;
        if (dst) CK(cudaMemcpyAsync((uint8_t*)dst + out_img * b0, (uint8_t*)d_out + out_img * b0, out_img * (b1 - b0), cudaMemcpyDeviceToHost, s));
    }
    for (int i = 0; i < 2; ++i) {
        CK(cudaEventRecord(p->ev_join[i], p->side[i]));
        CK(cudaStreamWaitEvent(stream, p->ev_join[i], 0));
    }
    CK(cudaEventRecord(p->ev_host_done, stream));
    p->host_in_flight = true;
    if (h_out && !out_pinned) {
        CK(cudaStreamSynchronize(stream));
        memcpy(h_out, p->h_out_stage, out_img * batch);
    }
    return FAA_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ JPEG decode --
static_assert(sizeof(faa_jpeg_header_t) == sizeof(JpegHeader) && sizeof(JpegHeader) == 144 &&
              offsetof(faa_jpeg_header_t, pool) == offsetof(JpegHeader, pool), "JPEG header layout");
static_assert(sizeof(faa_jpeg_table_t) == sizeof(JpegTable), "JPEG table layout");
static_assert(sizeof(faa_jpeg_sync_t) == sizeof(JpegSync) && sizeof(JpegSync) == 16 &&
              offsetof(faa_jpeg_sync_t, pred) == offsetof(JpegSync, pred), "JPEG sync point layout");

struct faa_jpeg_decoder {
    std::mutex mu;
    int device = -1;                      // bound at the first decode, like a policy handle
    void* d_coef = nullptr; size_t coef_bytes = 0;      // int16 coefficients of a call's images
    void* d_segs = nullptr; size_t segs_bytes = 0;      // restart-segment starts
    void* d_jobs = nullptr; size_t jobs_bytes = 0;      // per-call JpegJob table
    cudaStream_t last_stream = nullptr; bool have_last_stream = false;
    cudaEvent_t ev_switch = nullptr;
};

// grows a decoder buffer in stream order: the old one is released behind the work already queued on `stream`, so the
// host never waits
static int grow_async(void** ptr, size_t* have, size_t need, cudaStream_t stream) {
    if (*have >= need) return FAA_OK;
    if (*ptr) { CK(cudaFreeAsync(*ptr, stream)); *ptr = nullptr; *have = 0; }
    need = std::max(need + need / 4, (size_t)65536);
    CK(cudaMallocAsync(ptr, need, stream));
    *have = need;
    return FAA_OK;
}

// a header the JPEG device calls take: baseline (the quantisation and both Huffman pool slots of every component), or,
// when the call gives scans, a progressive one (quantisation slots only: the Huffman tables are the scans').  A
// progressive header's byte ranges and restart intervals are its scans'; its own must be 0, except the scan_len of a
// kJpegScanIndexed header, which is the length of its scan axis (plan_jpeg_jobs checks it against the scans).  The
// entropy and find kernels skip progressive headers by their reserved field.
static int check_jpeg_header(const JpegHeader& h, int n_tables, const std::string& who, bool scans = false) {
    const bool progressive = jpeg_is_progressive(h);
    if (progressive && !scans)
        return fail(FAA_ERR_VALUE, who + ": a progressive header needs the scans group (h_scans, d_scans, h_scan_first, "
                                         "d_scan_first) of faa_jpeg_decode");
    if (progressive && (h.scan_off != 0 || (h.scan_len != 0 && !jpeg_prog_indexed(h)) || h.restart != 0))
        return fail(FAA_ERR_VALUE, who + ": a progressive header has no scan range or restart interval of its own");
    if (h.ncomp != 1 && h.ncomp != 3) return fail(FAA_ERR_VALUE, who + ": component count must be 1 or 3");
    if (check_shape(h.h, h.w)) return fail(FAA_ERR_VALUE, who + ": size out of range");
    const bool samp = h.ncomp == 1 ? (h.hs == 1 && h.vs == 1)
                                   : ((h.hs == 1 && h.vs == 1) || (h.hs == 2 && h.vs == 1) || (h.hs == 2 && h.vs == 2));
    if (!samp) return fail(FAA_ERR_VALUE, who + ": unsupported sampling factors");
    if (h.mcu_x != (h.w + 8 * h.hs - 1) / (8 * h.hs) || h.mcu_y != (h.h + 8 * h.vs - 1) / (8 * h.vs))
        return fail(FAA_ERR_VALUE, who + ": MCU counts do not match the size");
    if (h.restart < 0 || h.offset < 0 || h.len < 0 || h.scan_off < 0 || h.scan_len < 0 || h.scan_off + h.scan_len > h.len)
        return fail(FAA_ERR_VALUE, who + ": restart interval or byte ranges out of range");
    for (int c = 0; c < h.ncomp; ++c)
        for (int k = 0; k < (progressive ? 1 : 3); ++k)
            if (h.pool[3 * k + c] < 0 || h.pool[3 * k + c] >= n_tables)
                return fail(FAA_ERR_VALUE, who + ": table pool index out of range");
    return FAA_OK;
}

extern "C" {

int faa_jpeg_parse(const uint8_t* bytes, size_t len, faa_jpeg_header_t* out) {
    if (!bytes || !out) return fail(FAA_ERR_VALUE, "null argument");
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg(bytes, len, h, &why);
    memcpy(out, &h, sizeof h);
    if (e == JPARSE_UNSUPPORTED) return fail(FAA_ERR_UNSUPPORTED, std::string("unsupported JPEG: ") + why);
    if (e == JPARSE_MALFORMED) return fail(FAA_ERR_VALUE, std::string("malformed JPEG: ") + why);
    return FAA_OK;
}

int faa_jpeg_tables(const uint8_t* bytes, size_t len, const faa_jpeg_header_t* hdr, faa_jpeg_table_t out[9]) {
    if (!bytes || !hdr || !out) return fail(FAA_ERR_VALUE, "null argument");
    JpegHeader h; memcpy(&h, hdr, sizeof h);
    if (h.ncomp != 1 && h.ncomp != 3) return fail(FAA_ERR_VALUE, "header has no 1 or 3 components");
    for (int c = 0; c < h.ncomp; ++c) {
        const size_t qbytes = (h.qprec >> c & 1) ? 128 : 64;
        if (h.table_at[c] < 0 || (size_t)h.table_at[c] + qbytes > len) return fail(FAA_ERR_VALUE, "quantisation table outside the file");
        for (int t = 1; t < 3; ++t) {
            const int32_t at = h.table_at[3 * t + c];
            if (jpeg_std_huff(at)) continue;                 // a standard table, not in the file
            if (at < 0 || (size_t)at + 16 > len) return fail(FAA_ERR_VALUE, "Huffman table outside the file");
            size_t total = 0;
            for (int l = 0; l < 16; ++l) total += bytes[at + l];
            if (total > 256 || (size_t)at + 16 + total > len) return fail(FAA_ERR_VALUE, "Huffman table outside the file");
        }
    }
    jpeg_tables(bytes, h, reinterpret_cast<JpegTable*>(out));
    return FAA_OK;
}

int faa_jpeg_decoder_create(faa_jpeg_decoder_t** out) {
    if (!out) return fail(FAA_ERR_VALUE, "null argument");
    *out = new faa_jpeg_decoder();
    return FAA_OK;
}

int faa_jpeg_decoder_destroy(faa_jpeg_decoder_t* d) {
    if (!d) return FAA_OK;
    for (void* b : {d->d_coef, d->d_segs, d->d_jobs}) if (b) cudaFree(b);      // (waits for the work that uses them)
    if (d->ev_switch) cudaEventDestroy(d->ev_switch);
    delete d;
    return FAA_OK;
}

int faa_jpeg_index_capacity(const faa_jpeg_header_t* hdr) {
    if (!hdr) return 0;
    JpegHeader h; memcpy(&h, hdr, sizeof h);
    return h.reserved == kJpegProgressive ? 0 : jpeg_index_capacity(h);
}

}  // extern "C"

// the point offsets of a call: [batch + 1], non-decreasing, from 0 up
static int check_jpeg_first(const int64_t* h_first, int batch) {
    if (h_first[0] < 0) return fail(FAA_ERR_VALUE, "point offsets: first[0] is negative");
    for (int i = 0; i < batch; ++i)
        if (h_first[i + 1] < h_first[i])
            return fail(FAA_ERR_VALUE, "point offsets: first[" + std::to_string(i + 1) + "] < first[" + std::to_string(i) + "]");
    if (h_first[batch] > (int64_t)INT32_MAX * 16) return fail(FAA_ERR_VALUE, "point offsets out of range");
    return FAA_OK;
}

// the batch sizes the JPEG device calls take: their grids have one CTA per image
static int check_jpeg_batch(int batch) {
    if (batch < 0) return fail(FAA_ERR_VALUE, "negative batch");
    if (batch > 65535) return fail(FAA_ERR_UNSUPPORTED, "at most 65535 images per call: split the batch");
    return FAA_OK;
}

// check_jpeg_header of every image of a call
static int check_jpeg_headers(const faa_jpeg_header_t* h_headers, int batch, int n_tables, bool scans = false) {
    for (int i = 0; i < batch; ++i) {
        JpegHeader h; memcpy(&h, &h_headers[i], sizeof h);
        if (int e = check_jpeg_header(h, n_tables, "image " + std::to_string(i), scans)) return e;
    }
    return FAA_OK;
}

extern "C" {

int faa_jpeg_index_build(const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                         const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                         const int64_t* h_first, const int64_t* d_first, faa_jpeg_sync_t* d_points, int32_t* d_count,
                         int32_t* d_status, void* stream_v) {
    if ((!h_headers || !d_headers || !d_tables || !d_src || !h_first || !d_first || !d_count || !d_status) && batch > 0)
        return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_jpeg_batch(batch)) return e;
    if (batch == 0) return FAA_OK;
    if (int e = check_jpeg_first(h_first, batch)) return e;
    if (!d_points && h_first[batch] > h_first[0]) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_jpeg_headers(h_headers, batch, n_tables)) return e;
    if (int e = ensure_device()) return e;
    JpegDecodeParams P = {};
    P.hdrs = reinterpret_cast<const JpegHeader*>(d_headers);
    P.pool = reinterpret_cast<const JpegTable*>(d_tables);
    P.src = d_src;
    P.status = d_status;
    P.batch = batch;
    P.first = d_first;
    P.points = reinterpret_cast<JpegSync*>(d_points);
    P.count = d_count;
    CK(launch_jpeg_index(P, (cudaStream_t)stream_v));
    g_launches++;
    return FAA_OK;
}

int faa_jpeg_index_find(const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                        const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                        const int64_t* h_first, const int64_t* d_first, faa_jpeg_sync_t* d_points, int32_t* d_count,
                        void* stream_v) {
    if ((!h_headers || !d_headers || !d_tables || !d_src || !h_first || !d_first || !d_count) && batch > 0)
        return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_jpeg_batch(batch)) return e;
    if (batch == 0) return FAA_OK;
    if (int e = check_jpeg_first(h_first, batch)) return e;
    if (!d_points && h_first[batch] > h_first[0]) return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_jpeg_headers(h_headers, batch, n_tables)) return e;
    if (int e = ensure_device()) return e;
    JpegDecodeParams P = {};
    P.hdrs = reinterpret_cast<const JpegHeader*>(d_headers);
    P.pool = reinterpret_cast<const JpegTable*>(d_tables);
    P.src = d_src;
    P.batch = batch;
    P.rec_first = d_first;
    P.rec_points = reinterpret_cast<JpegSync*>(d_points);
    P.count = d_count;
    CK(launch_jpeg_find(P, false, (cudaStream_t)stream_v));
    g_launches++;
    return FAA_OK;
}

}  // extern "C"

// image `who`'s scans [0, n): parameters a progression can have, byte ranges inside the file, pool slots in range, and
// the waves the dependency rule gives (a wrong wave would let two work items race on a coefficient)
static int check_jpeg_scans(const JpegHeader& h, const JpegScan* scans, int64_t n, int n_tables, const std::string& who) {
    if (n < 1 || n > kJpegMaxScans) return fail(FAA_ERR_VALUE, who + ": 1 to 64 scans per image");
    JpegScan w[kJpegMaxScans];
    memcpy(w, scans, (size_t)n * sizeof(JpegScan));
    for (int64_t i = 0; i < n; ++i) {
        const JpegScan& s = scans[i];
        const std::string at = who + " scan " + std::to_string(i);
        if (s.ns < 1 || s.ns > h.ncomp) return fail(FAA_ERR_VALUE, at + ": component count out of range");
        for (int k = 0; k < s.ns; ++k)
            if (s.comp[k] < (k ? s.comp[k - 1] + 1 : 0) || s.comp[k] >= h.ncomp)
                return fail(FAA_ERR_VALUE, at + ": components out of range or out of frame order");
        if (s.ss < 0 || s.ss > s.se || s.se > 63 || (s.ss == 0) != (s.se == 0) || (s.ss > 0 && s.ns != 1) || s.al < 0 ||
            s.al > 13 || (s.ah != 0 && s.ah != s.al + 1))
            return fail(FAA_ERR_VALUE, at + ": spectral band or approximation out of range");
        if (s.restart < 0 || s.off < 0 || s.len < 0 || s.off + s.len > h.len)
            return fail(FAA_ERR_VALUE, at + ": restart interval or byte range out of range");
        for (int k = 0; k < jpeg_scan_tables(s); ++k) {
            const int32_t p = s.pool[s.ss == 0 ? k : 3];
            if (p < 0 || p >= n_tables) return fail(FAA_ERR_VALUE, at + ": table pool index out of range");
        }
    }
    jpeg_scan_waves(w, (int)n);
    for (int64_t i = 0; i < n; ++i)
        if (w[i].wave != scans[i].wave)
            return fail(FAA_ERR_VALUE, who + " scan " + std::to_string(i) + ": wave does not follow the scans' dependencies");
    return FAA_OK;
}

// The JpegJob table of a decode call whose headers are checked: jobs[i] holds where image i's coefficient blocks,
// restart-segment starts and reconstruct tiles begin, jobs[batch] the totals.  Also checks each image's output
// descriptor and, when the call gives scans (image i's are scans[scan_first[i], scan_first[i + 1])), each image's
// scans: a progressive image's, whose segments it counts where a baseline image has jpeg_segments, and that a baseline
// image has none.
static int plan_jpeg_jobs(const faa_jpeg_header_t* h_headers, const faa_image_t* h_out, int batch, int n_tables,
                          const JpegScan* scans, const int64_t* scan_first, std::vector<JpegJob>& jobs) {
    jobs.resize((size_t)batch + 1);
    int64_t blocks = 0, segs = 0, tiles = 0;
    for (int i = 0; i < batch; ++i) {
        JpegHeader h; memcpy(&h, &h_headers[i], sizeof h);
        const std::string who = "image " + std::to_string(i);
        if (!h_out[i].data) return fail(FAA_ERR_VALUE, "output " + who + " has no data");
        if (h_out[i].h != h.h || h_out[i].w != h.w) return fail(FAA_ERR_VALUE, "output " + who + " is not the size of its JPEG");
        jobs[(size_t)i] = {blocks, (int32_t)segs, (int32_t)tiles};
        blocks += jpeg_image_blocks(h);
        if (!jpeg_is_progressive(h)) {
            if (scans && scan_first[i + 1] != scan_first[i])
                return fail(FAA_ERR_VALUE, who + ": a baseline image owns no scans");
            segs += jpeg_segments(h);
        } else {                                   // (check_jpeg_headers refused it if the call gives no scans)
            const int64_t n = scan_first[i + 1] - scan_first[i];
            if (int e = check_jpeg_scans(h, scans + scan_first[i], n, n_tables, who)) return e;
            int64_t axis = 0;
            for (int64_t k = 0; k < n; ++k) {
                segs += jpeg_scan_segments(h, scans[scan_first[i] + k]);
                axis += scans[scan_first[i] + k].len;
            }
            if (jpeg_prog_indexed(h) && h.scan_len != axis)
                return fail(FAA_ERR_VALUE, who + ": a scan-indexed progressive header's scan_len must be the sum of its "
                                                 "scans' lengths");
        }
        tiles += (int64_t)((h.w + kJpegTileW - 1) / kJpegTileW) * ((h.h + kJpegTileH - 1) / kJpegTileH);
        if (segs > INT32_MAX || tiles > INT32_MAX) return fail(FAA_ERR_UNSUPPORTED, "batch too large: split it");
    }
    jobs[(size_t)batch] = {blocks, (int32_t)segs, (int32_t)tiles};
    return FAA_OK;
}

// Binds the handle to the current device, orders this call's use of its scratch after the previous call's, grows the
// coefficient, segment and job buffers to what the call's job table needs and uploads the table.  Every decode call
// goes through here, under the handle's lock until its launches are queued, so calls may follow each other on any
// streams.
static int jpeg_call_scratch(faa_jpeg_decoder_t* d, cudaStream_t stream, const std::vector<JpegJob>& jobs) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return fail(FAA_ERR_NO_DEVICE, "no current CUDA device"); }
    if (d->device < 0) d->device = dev;
    if (d->device != dev)
        return fail(FAA_ERR_VALUE, "JPEG decoder is bound to device " + std::to_string(d->device) + " but the current device is " +
                    std::to_string(dev) + ": create one decoder per device");
    if (d->have_last_stream && d->last_stream != stream) {          // buffers are reused in the order of the calls
        if (!d->ev_switch) CK(cudaEventCreateWithFlags(&d->ev_switch, cudaEventDisableTiming));
        CK(cudaEventRecord(d->ev_switch, d->last_stream));
        CK(cudaStreamWaitEvent(stream, d->ev_switch, 0));
    }
    d->last_stream = stream; d->have_last_stream = true;
    if (int e = grow_async(&d->d_coef, &d->coef_bytes, (size_t)jobs.back().coef * 128, stream)) return e;
    if (int e = grow_async(&d->d_segs, &d->segs_bytes, (size_t)jobs.back().seg * sizeof(int32_t), stream)) return e;
    if (int e = grow_async(&d->d_jobs, &d->jobs_bytes, jobs.size() * sizeof(JpegJob), stream)) return e;
    CK(cudaMemcpyAsync(d->d_jobs, jobs.data(), jobs.size() * sizeof(JpegJob), cudaMemcpyHostToDevice, stream));  // (pageable: staged at once)
    return FAA_OK;
}

extern "C" {

int faa_jpeg_decode(faa_jpeg_decoder_t* d, const faa_jpeg_header_t* h_headers, const faa_jpeg_header_t* d_headers,
                    const faa_jpeg_table_t* d_tables, int n_tables, const uint8_t* d_src, int batch,
                    const faa_image_t* h_out, const faa_image_t* d_out, int32_t* d_status,
                    const faa_jpeg_sync_t* d_points, const int64_t* h_first, const int64_t* d_first,
                    const int64_t* h_cap_first, const int64_t* d_cap_first, faa_jpeg_sync_t* d_points_out,
                    int32_t* d_count, const faa_jpeg_scan_t* h_scans, const faa_jpeg_scan_t* d_scans,
                    const int64_t* h_scan_first, const int64_t* d_scan_first, int find, void* stream_v) {
    if (!d || ((!h_headers || !d_headers || !d_tables || !d_src || !h_out || !d_out || !d_status) && batch > 0))
        return fail(FAA_ERR_VALUE, "null argument");
    if (int e = check_jpeg_batch(batch)) return e;
    const bool indexed = d_points || h_first || d_first;
    const bool recording = h_cap_first || d_cap_first || d_points_out || d_count;
    const bool scans = h_scans || d_scans || h_scan_first || d_scan_first;
    if (find && !recording)
        return fail(FAA_ERR_VALUE, "find needs the recording outputs h_cap_first, d_cap_first, d_points_out and d_count");
    if (recording && batch > 0) {
        if (!h_cap_first || !d_cap_first || !d_count) return fail(FAA_ERR_VALUE, "null argument");
        if (int e = check_jpeg_first(h_cap_first, batch)) return e;
        if (!d_points_out && h_cap_first[batch] > h_cap_first[0]) return fail(FAA_ERR_VALUE, "null argument: d_points_out");
    }
    if (indexed && batch > 0) {
        if (!h_first || !d_first) return fail(FAA_ERR_VALUE, "null argument: point offsets need h_first and d_first");
        if (int e = check_jpeg_first(h_first, batch)) return e;
        if (!d_points && h_first[batch] > h_first[0]) return fail(FAA_ERR_VALUE, "null argument: d_points");
    }
    if (scans && batch > 0) {
        if (!h_scans || !d_scans || !h_scan_first || !d_scan_first)
            return fail(FAA_ERR_VALUE, "null argument: scans need h_scans, d_scans, h_scan_first and d_scan_first");
        if (int e = check_jpeg_first(h_scan_first, batch)) return e;
    }
    if (int e = check_jpeg_headers(h_headers, batch, n_tables, scans)) return e;
    std::vector<JpegJob> jobs;
    if (int e = plan_jpeg_jobs(h_headers, h_out, batch, n_tables, reinterpret_cast<const JpegScan*>(h_scans), h_scan_first,
                               jobs))
        return e;
    if (int e = ensure_device()) return e;
    if (batch == 0) return FAA_OK;
    const int n_prog = (int)std::count_if(h_headers, h_headers + batch,
                                          [](const faa_jpeg_header_t& h) {
                                              return (h.reserved | FAA_JPEG_SCAN_INDEXED) ==
                                                     (FAA_JPEG_PROGRESSIVE | FAA_JPEG_SCAN_INDEXED);
                                          });
    cudaStream_t stream = (cudaStream_t)stream_v;
    std::lock_guard<std::mutex> lk(d->mu);
    if (int e = jpeg_call_scratch(d, stream, jobs)) return e;
    // launch_jpeg_entropy picks its instantiation from the groups: the pointers of one that is not given are null
    JpegDecodeParams P = {};
    P.hdrs = reinterpret_cast<const JpegHeader*>(d_headers);
    P.pool = reinterpret_cast<const JpegTable*>(d_tables);
    P.src = d_src;
    P.jobs = reinterpret_cast<const JpegJob*>(d->d_jobs);
    P.out = reinterpret_cast<const CropImage*>(d_out);
    P.coef = reinterpret_cast<int16_t*>(d->d_coef);
    P.segs = reinterpret_cast<int32_t*>(d->d_segs);
    P.status = d_status;
    P.batch = batch;
    P.first = d_first;
    P.points = const_cast<JpegSync*>(reinterpret_cast<const JpegSync*>(d_points));
    P.rec_first = d_cap_first;
    P.rec_points = reinterpret_cast<JpegSync*>(d_points_out);
    P.count = d_count;
    P.scans = reinterpret_cast<const JpegScan*>(d_scans);
    P.scan_first = d_scan_first;
    if (n_prog < batch) {
        if (find) {
            CK(launch_jpeg_find(P, true, stream));
            g_launches++;
        }
        CK(launch_jpeg_entropy(P, stream, find != 0));
        g_launches++;
    }
    if (n_prog > 0) {
        CK(launch_jpeg_progressive(P, stream));
        g_launches++;
    }
    CK(launch_jpeg_reconstruct(P, jobs.back().tile0, stream));
    g_launches++;
    return FAA_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ progressive JPEG parse --
static_assert(sizeof(faa_jpeg_scan_t) == sizeof(JpegScan) && sizeof(JpegScan) == 112 &&
              offsetof(faa_jpeg_scan_t, pool) == offsetof(JpegScan, pool) && FAA_JPEG_MAX_SCANS == kJpegMaxScans &&
              FAA_JPEG_PROGRESSIVE == kJpegProgressive && FAA_JPEG_SCAN_INDEXED == kJpegScanIndexed, "JPEG scan layout");

extern "C" {

int faa_jpeg_parse_progressive(const uint8_t* bytes, size_t len, faa_jpeg_header_t* out, faa_jpeg_scan_t* scans,
                               int max_scans, int* n_scans) {
    if (!bytes || !out || !scans || !n_scans || max_scans < 1) return fail(FAA_ERR_VALUE, "null argument");
    JpegHeader h;
    const char* why = "";
    const int e = parse_jpeg_progressive(bytes, len, h, reinterpret_cast<JpegScan*>(scans),
                                         std::min(max_scans, kJpegMaxScans), n_scans, &why);
    memcpy(out, &h, sizeof h);
    if (e == JPARSE_UNSUPPORTED) return fail(FAA_ERR_UNSUPPORTED, std::string("unsupported JPEG: ") + why);
    if (e == JPARSE_MALFORMED) return fail(FAA_ERR_VALUE, std::string("malformed JPEG: ") + why);
    return FAA_OK;
}

int faa_jpeg_scan_tables(const uint8_t* bytes, size_t len, const faa_jpeg_header_t* hdr, const faa_jpeg_scan_t* scans,
                         int n_scans, faa_jpeg_table_t* out) {
    if (!bytes || !hdr || !scans || !out) return fail(FAA_ERR_VALUE, "null argument");
    JpegHeader h; memcpy(&h, hdr, sizeof h);
    if (!jpeg_is_progressive(h) || (h.ncomp != 1 && h.ncomp != 3)) return fail(FAA_ERR_VALUE, "not a progressive header");
    if (n_scans < 1 || n_scans > kJpegMaxScans) return fail(FAA_ERR_VALUE, "1 to 64 scans");
    for (int c = 0; c < h.ncomp; ++c) {
        const size_t qbytes = (h.qprec >> c & 1) ? 128 : 64;
        if (h.table_at[c] < 0 || (size_t)h.table_at[c] + qbytes > len) return fail(FAA_ERR_VALUE, "quantisation table outside the file");
    }
    const JpegScan* s = reinterpret_cast<const JpegScan*>(scans);
    for (int i = 0; i < n_scans; ++i)
        for (int k = 0; k < 6; ++k) {
            const int32_t at = k < 3 ? s[i].dc_at[k] : s[i].ac_at[k - 3];
            if (at == -1 || jpeg_std_huff(at)) continue;
            if (at < 0 || (size_t)at + 16 > len) return fail(FAA_ERR_VALUE, "Huffman table outside the file");
            size_t total = 0;
            for (int l = 0; l < 16; ++l) total += bytes[at + l];
            if (total > 256 || (size_t)at + 16 + total > len) return fail(FAA_ERR_VALUE, "Huffman table outside the file");
        }
    jpeg_progressive_tables(bytes, h, s, n_scans, reinterpret_cast<JpegTable*>(out));
    return FAA_OK;
}

}  // extern "C"
