// Host build of the lean light launch's decisions (faa_core.cuh): which kernel every program runs under a launch's allow
// bits, and the planner's choice of the lean light kernel.  Built on demand by tests/test_lean_light_host.py.
#include "../../fast_autoaugment_b200/csrc/faa_core.cuh"

#include <string.h>

using namespace faa;

extern "C" {

// per image, 5 bytes: weight class (2 light, 1 mid, 0 heavy), program class, op kinds of slots 0 and 1, prog_two_stage
int faa_emu_lean_classes(const void* ops_v, int n_op, const void* samples_v, const void* boxes_v, int B, int H, int W,
                         int allow, uint8_t* out) {
    const OpRec* ops = (const OpRec*)ops_v;
    const Sample* samples = (const Sample*)samples_v;
    const Box* boxes = (const Box*)boxes_v;
    for (int i = 0; i < B; ++i) {
        Prog g;
        build_prog(samples[i], boxes + (size_t)i * n_op, ops, n_op, 0, 1, H, W, W, allow, g);
        lean_order(g, allow);
        uint8_t* o = out + (size_t)i * 5;
        o[0] = prog_is_light(g, allow) ? 2 : prog_is_mid(g, allow) ? 1 : 0;
        o[1] = g.cls; o[2] = (uint8_t)g.op[0].kind; o[3] = (uint8_t)g.op[1].kind;
        o[4] = prog_two_stage(g, allow) ? 1 : 0;
    }
    return 0;
}

// plan_launch of a uniform launch of the final window: allow, lean_light, light bands, light band staged, use_mid, no_heavy
int faa_emu_lean_plan(int H, int W, int batch, int out_u8, int out_mod16, int crop_pad, int philox, int32_t* out) {
    PlanInput in = {};
    in.H = H; in.W = W; in.out_h = H; in.out_w = W; in.batch = batch; in.crop_pad = crop_pad; in.out_u8 = out_u8 != 0;
    in.out_mod16 = (uint32_t)out_mod16; in.apply_tail = true; in.has_sg = true; in.split_min = kSplitMin;
    in.philox = philox != 0; in.allow_ahead = philox != 0;
    const LaunchPlan L = plan_launch(in);
    const int32_t v[] = {L.allow, L.lean_light, L.geo[1].bands, L.geo[1].band_cap > 0, L.use_mid, L.no_heavy};
    memcpy(out, v, sizeof v);
    return (int)(sizeof v / sizeof v[0]);
}

}  // extern "C"
