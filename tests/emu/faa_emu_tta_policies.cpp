// faa_emu_tta_policies.cpp - HOST build of the multi-policy TTA resolve step, TEST INFRASTRUCTURE ONLY.
//
// faa_augment_tta_policies runs faa_resolve_kernel<true>: schedule entry v draws global sample rng.first_index + v from
// candidate tta_candidate(v, per_cand)'s table, probabilities and n_sub.  This drives the same philox_sample and
// tta_candidate of fast_autoaugment_b200/csrc/faa_core.cuh with that selection, so the CPU tests can check it against
// the single-policy sampler of each candidate.  The package never loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

using namespace faa;

extern "C" {

// ops[t] / probs[t] / n_sub[t]: candidate t's compiled table [n_sub][n_op][2], probabilities [n_sub][n_op], n_sub
int faa_emu_philox_policies(const void* const* ops_v, const double* const* probs, const int32_t* n_sub, int n_cands,
                            int per_cand, int n_op, const void* rng_v, int n, int H, int W, int out_h, int out_w,
                            void* samples_v, void* boxes_v) {
    RngCfg r; memcpy(&r, rng_v, sizeof r);
    Sample* samples = (Sample*)samples_v;
    Box* boxes = (Box*)boxes_v;
    for (int v = 0; v < n; ++v) {
        const int t = tta_candidate(v, per_cand);
        if (t >= n_cands) return -1;
        const PolicyRef c = {(const OpRec*)ops_v[t], probs[t], n_sub[t], 0};
        Box bx[8];
        philox_sample(r, r.first_index + (uint64_t)v, c.ops, c.probs, c.n_sub, n_op, H, W, out_h, out_w, samples[v], bx);
        for (int j = 0; j < n_op; ++j) boxes[(size_t)v * n_op + j] = bx[j];
    }
    return 0;
}

}  // extern "C"
