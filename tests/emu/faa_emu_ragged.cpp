// faa_emu_ragged.cpp - HOST build of the positional Philox sampler, TEST INFRASTRUCTURE ONLY.
//
// faa_sample_philox_at runs faa_resolve_kernel with a position array: record k holds the decisions of global sample
// rng.first_index + pos[k].  This drives the same philox_sample of fast_autoaugment_b200/csrc/faa_core.cuh with that
// indexing, so the CPU tests can check the per-size policy groups of a ragged ImageNet batch.  The package never loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

using namespace faa;

extern "C" {

// pos == NULL: positions 0..n-1 (faa_emu_philox)
int faa_emu_philox_at(const void* ops_v, const double* probs, int n_sub, int n_op, const void* rng_v, int n, int H, int W,
                      int out_h, int out_w, const int32_t* pos, void* samples_v, void* boxes_v) {
    const OpRec* ops = (const OpRec*)ops_v;
    RngCfg r; memcpy(&r, rng_v, sizeof r);
    Sample* samples = (Sample*)samples_v;
    Box* boxes = (Box*)boxes_v;
    for (int k = 0; k < n; ++k) {
        Box bx[8];
        const uint64_t at = pos ? (uint64_t)(uint32_t)pos[k] : (uint64_t)k;
        philox_sample(r, r.first_index + at, ops, probs, n_sub, n_op, H, W, out_h, out_w, samples[k], bx);
        for (int j = 0; j < n_op; ++j) boxes[(size_t)k * n_op + j] = bx[j];
    }
    return 0;
}

}  // extern "C"
