// Host build of the fused step's RMSprop update (ops/csrc/tfy_fused_step.cuh: tfy_rmsprop_states + the three-state
// tfy_opt_update_rt) over the state layout the K4 kernel uses: s1 = mean square, s2 = momentum buffer then mean
// gradient, each n long and present only when enabled.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

static inline float rsqrtf(float x) { return 1.f / sqrtf(x); }

#include "tfy_fused_step.cuh"

extern "C" void tfy_host_rmsprop_step(TfyOptHyper* hp, int world, float* p, const float* g, float* s1, float* s2,
                                      int n) {
    const TfyStepConsts k = tfy_step_consts(hp, world, TFY_OPT_RMSPROP);
    float* __restrict__ mom = s2;
    float* mg = nullptr;
    tfy_rmsprop_states(hp, (size_t)n, mom, mg);
    for (int i = 0; i < n; ++i) {
        float pi = p[i], a = s1[i], b = mom ? mom[i] : 0.f, c = mg ? mg[i] : 0.f;
        tfy_opt_update_rt<-1>(TFY_OPT_RMSPROP, pi, g[i] * k.gscale, a, b, c, k.lr, k.p1, k.p2, k.eps, k.wd, k.flags,
                              k.lr_bc1, k.bc2_rsqrt, k.first_step);
        p[i] = pi; s1[i] = a;
        if (mom) mom[i] = b;
        if (mg) mg[i] = c;
    }
    hp->step += 1;
}
