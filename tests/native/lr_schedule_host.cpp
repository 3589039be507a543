// Host build of the learning-rate schedule the fused optimizer step evaluates where it advances its step counter
// (ops/csrc/tfy_lr_schedule.cuh: tfy_lr_schedule_eval), over the structs the device reads (TfyLrSchedule inside
// TfyHyperBlock).
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "tfy_common.cuh"

extern "C" float tfy_host_lr_schedule(const TfyLrSchedule* s, int64_t step) { return tfy_lr_schedule_eval(*s, step); }

extern "C" int tfy_host_lr_schedule_layout(int* out, int cap) {
    int n = 0;
#define PUT(v) do { if (n < cap) out[n] = (int)(v); ++n; } while (0)
    PUT(sizeof(TfyLrSchedule)); PUT(offsetof(TfyLrSchedule, kind)); PUT(offsetof(TfyLrSchedule, flags));
    PUT(offsetof(TfyLrSchedule, n_boundaries)); PUT(offsetof(TfyLrSchedule, pad));
    PUT(offsetof(TfyLrSchedule, initial_lr)); PUT(offsetof(TfyLrSchedule, decay_steps));
    PUT(offsetof(TfyLrSchedule, decay_rate)); PUT(offsetof(TfyLrSchedule, end_lr)); PUT(offsetof(TfyLrSchedule, power));
    PUT(offsetof(TfyLrSchedule, alpha)); PUT(offsetof(TfyLrSchedule, warmup_target));
    PUT(offsetof(TfyLrSchedule, warmup_steps)); PUT(offsetof(TfyLrSchedule, t_mul)); PUT(offsetof(TfyLrSchedule, m_mul));
    PUT(offsetof(TfyLrSchedule, boundaries)); PUT(offsetof(TfyLrSchedule, values)); PUT(offsetof(TfyLrSchedule, pad2));
    PUT(TFY_LR_MAX_BOUNDARIES); PUT(TFY_LR_EXPONENTIAL); PUT(TFY_LR_PIECEWISE); PUT(TFY_LR_POLYNOMIAL);
    PUT(TFY_LR_INVERSE_TIME); PUT(TFY_LR_COSINE); PUT(TFY_LR_COSINE_RESTARTS);
    PUT(sizeof(TfyHyperBlock)); PUT(offsetof(TfyHyperBlock, hp)); PUT(offsetof(TfyHyperBlock, sched));
    PUT(TFY_OPT_LR_SCHEDULE);
#undef PUT
    return n;
}
