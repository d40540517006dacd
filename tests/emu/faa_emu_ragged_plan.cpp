// faa_emu_ragged_plan.cpp - HOST build of the ragged launch planner, TEST INFRASTRUCTURE ONLY.
//
// faa_augment_ragged launches what plan_ragged (fast_autoaugment_b200/csrc/faa_core.cuh) returns for the batch's sizes
// and base addresses.  This exports the same function, so the CPU tests check the planner itself.  The package never
// loads it.
#include <cstdint>
#include <cstring>

#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

using namespace faa;

extern "C" {

// per-geometry values, in the order faa_emu_ragged_geom_fields names them
const char* faa_emu_ragged_geom_fields() {
    return "H W bands band_cap stage octets mat_cap allow scratch rcp_out_qpr rcp_w rcp_wq rcp_opr";
}

// hw: [n][2]; in_mod16 / out_mod16: [n] base addresses mod 16.  Writes geom_of [n], order [n], launches [<= 4][4]
// (bands, first, count, dynamic shared memory) and geoms [<= n][13]; returns the number of launches, *n_geoms the number
// of geometries.
int faa_emu_plan_ragged(int n, const int32_t* hw, const int32_t* in_mod16, const int32_t* out_mod16, int has_sg,
                        int32_t* geom_of, int32_t* order, int32_t* launches, int32_t* geoms, int32_t* n_geoms) {
    std::vector<RaggedImageIn> in((size_t)n);
    for (int i = 0; i < n; ++i) in[(size_t)i] = {hw[2 * i], hw[2 * i + 1], (uint32_t)in_mod16[i], (uint32_t)out_mod16[i]};
    const RaggedPlan R = plan_ragged(in.data(), n, has_sg != 0);
    for (int i = 0; i < n; ++i) { geom_of[i] = R.geom_of[(size_t)i]; order[i] = R.order[(size_t)i]; }
    for (size_t l = 0; l < R.launches.size(); ++l) {
        const RaggedLaunch& L = R.launches[l];
        const int32_t v[4] = {L.bands, L.first, L.count, (int32_t)L.smem};
        memcpy(launches + 4 * l, v, sizeof v);
    }
    for (size_t k = 0; k < R.geoms.size(); ++k) {
        const RaggedGeom& g = R.geoms[k];
        const int32_t v[13] = {g.H, g.W, g.plan.geo[0].bands, g.plan.geo[0].band_cap, g.plan.stage, g.plan.octets,
                               g.plan.mat_cap, g.plan.allow, g.plan.scratch, (int32_t)g.rcp_out_qpr, (int32_t)g.rcp_w,
                               (int32_t)g.rcp_wq, (int32_t)g.rcp_opr};
        memcpy(geoms + 13 * k, v, sizeof v);
    }
    *n_geoms = (int32_t)R.geoms.size();
    return (int)R.launches.size();
}

}  // extern "C"
