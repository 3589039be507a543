// Host build of the fused step's Adamax and Nadam updates (ops/csrc/tfy_fused_step.cuh: tfy_step_consts, the
// two-state tfy_opt_update_rt for Adamax, tfy_nadam_update) followed by what the thread that advances the step does
// (the step counter, a scheduled rate, Nadam's running product in its TfyNadamHyperBlock).
#include <math.h>
#include <stddef.h>
#include <stdint.h>

static inline float rsqrtf(float x) { return 1.f / sqrtf(x); }

#include "tfy_fused_step.cuh"

extern "C" void tfy_host_adamax_nadam_step(TfyOptHyper* hp, int opt, int sched, int world, float* p, const float* g,
                                           float* s1, float* s2, int n) {
    const TfyStepConsts k = tfy_step_consts(hp, world, opt);
    for (int i = 0; i < n; ++i) {
        float pi = p[i], a = s1[i], b = s2[i];
        if (opt == TFY_OPT_NADAM)
            tfy_nadam_update(pi, g[i] * k.gscale, a, b, k);
        else
            tfy_opt_update_rt<-1>(opt, pi, g[i] * k.gscale, a, b, k.lr, k.p1, k.p2, k.eps, k.wd, k.flags, k.lr_bc1,
                                  k.bc2_rsqrt, k.first_step);
        p[i] = pi; s1[i] = a; s2[i] = b;
    }
    const int step = hp->step;
    if (sched) tfy_advance_scheduled_step(hp, step);
    else hp->step = step + 1;
    if (opt == TFY_OPT_NADAM) tfy_nadam_advance(hp, k);
}

extern "C" int tfy_host_nadam_layout(int* out, int cap) {
    int n = 0;
#define PUT(v) do { if (n < cap) out[n] = (int)(v); ++n; } while (0)
    PUT(sizeof(TfyNadamHyperBlock)); PUT(offsetof(TfyNadamHyperBlock, hp)); PUT(offsetof(TfyNadamHyperBlock, sched));
    PUT(offsetof(TfyNadamHyperBlock, mu_product)); PUT(TFY_OPT_ADAMAX); PUT(TFY_OPT_NADAM);
#undef PUT
    return n;
}
