// Keras learning-rate schedules (keras.optimizers.schedules), evaluated where the fused optimizer step advances its
// device step counter.
//
// A fused step launched with TFY_OPT_LR_SCHEDULE reads its hyper-parameters from a TfyHyperBlock (tfy_common.cuh):
// the schedule follows the TfyOptHyper in device memory.  The thread of K4 that stores `hp->step = step + 1` then
// also stores `hp->lr = schedule(step + 1)`, so the next launch -- and the communication CTAs of the conv2
// weight-gradient kernel, which read hp->lr as the trailing launch does -- read the rate of the step they perform
// exactly as they read a constant one.  One thread evaluates one scalar per step; every rank evaluates the same
// function on the same step counter, so the ranks agree bit for bit.
//
// The arithmetic is float64, rounded to float once at the end, so the host build of this header and the device agree
// with a float64 reference to float32 rounding.  Every rate the fused step reads is written by this device function:
// the one of the first step and of a restored step too (tfy_lr_schedule_sync), so an interrupted run and an
// uninterrupted one read the same bits whatever the host's libm or FMA contraction would give.  The formulas are
// tf.keras 2.13+ / Keras 3's, `step` being Keras's `iterations`: the batches already trained, which are the updates
// already applied unless gradients are accumulated (the module docstring of tf_yarn_b200/keras/schedules.py states
// each of them).
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#define TFY_LR_NOINLINE __attribute__((noinline))
#else
#define TFY_LR_NOINLINE __noinline__
#endif

#define TFY_LR_MAX_BOUNDARIES 16

enum TfyLrKind {
    TFY_LR_CONSTANT = 0,
    TFY_LR_EXPONENTIAL = 1,
    TFY_LR_PIECEWISE = 2,
    TFY_LR_POLYNOMIAL = 3,
    TFY_LR_INVERSE_TIME = 4,
    TFY_LR_COSINE = 5,
    TFY_LR_COSINE_RESTARTS = 6,
};

struct TfyLrSchedule {
    int32_t kind;            // TfyLrKind
    int32_t flags;           // bit0: staircase (exponential, inverse time) / cycle (polynomial); bit1: warmup (cosine)
    int32_t n_boundaries;    // piecewise: boundaries used, values used = n_boundaries + 1
    int32_t pad;
    double initial_lr;
    double decay_steps;      // first_decay_steps (cosine restarts)
    double decay_rate;
    double end_lr;           // polynomial: end_learning_rate
    double power;            // polynomial
    double alpha;            // cosine, cosine restarts
    double warmup_target;    // cosine (flags bit1)
    double warmup_steps;     // cosine
    double t_mul, m_mul;     // cosine restarts
    double boundaries[TFY_LR_MAX_BOUNDARIES];
    float values[TFY_LR_MAX_BOUNDARIES + 1];
    int32_t pad2;
};

__host__ __device__ inline double tfy_lr_cosine_decay(double step, double decay_steps, double alpha, double from_lr) {
    const double pi = 3.14159265358979323846;
    const double decayed = 0.5 * (1.0 + cos(pi * (step / decay_steps)));
    return from_lr * ((1.0 - alpha) * decayed + alpha);
}

// The learning rate of the update performed after `step` updates.  Not inlined: the call keeps the float64 math out of
// the register allocation of the fused step's main loop.
__host__ __device__ TFY_LR_NOINLINE inline float tfy_lr_schedule_eval(const TfyLrSchedule& s, int64_t step_i) {
    const double step = (double)step_i;
    double lr = s.initial_lr;
    switch (s.kind) {
    case TFY_LR_EXPONENTIAL: {
        double p = step / s.decay_steps;
        if (s.flags & 1) p = floor(p);
        lr = s.initial_lr * pow(s.decay_rate, p);
        break;
    }
    case TFY_LR_PIECEWISE: {
        int i = 0;
        while (i < s.n_boundaries && step > s.boundaries[i]) ++i;
        return s.values[i];
    }
    case TFY_LR_POLYNOMIAL: {
        double ds = s.decay_steps, t = step;
        if (s.flags & 1) {
            if (step > 0) ds *= ceil(step / s.decay_steps);
        } else {
            t = fmin(step, s.decay_steps);
        }
        lr = (s.initial_lr - s.end_lr) * pow(1.0 - t / ds, s.power) + s.end_lr;
        break;
    }
    case TFY_LR_INVERSE_TIME: {
        double p = step / s.decay_steps;
        if (s.flags & 1) p = floor(p);
        lr = s.initial_lr / (1.0 + s.decay_rate * p);
        break;
    }
    case TFY_LR_COSINE: {
        if (!(s.flags & 2)) {
            lr = tfy_lr_cosine_decay(fmin(step, s.decay_steps), s.decay_steps, s.alpha, s.initial_lr);
        } else {
            const double t = fmin(step, s.decay_steps + s.warmup_steps);
            if (t < s.warmup_steps)
                lr = (s.warmup_target - s.initial_lr) * (t / s.warmup_steps) + s.initial_lr;
            else
                lr = tfy_lr_cosine_decay(t - s.warmup_steps, s.decay_steps, s.alpha, s.warmup_target);
        }
        break;
    }
    case TFY_LR_COSINE_RESTARTS: {
        // period i lasts first_decay_steps * t_mul^i steps (t_mul >= 1) and starts (t_mul^i - 1) / (t_mul - 1) periods
        // of first_decay_steps in.  The logarithm only estimates i: the start of the period is then checked on both
        // sides, so a step that begins a period is never rounded into the previous one.
        double frac = step / s.decay_steps, i;
        if (s.t_mul == 1.0) {
            i = floor(frac);
            frac -= i;
        } else {
            const double t = s.t_mul;
            i = floor(log1p(frac * (t - 1.0)) / log(t));
            double start = (pow(t, i) - 1.0) / (t - 1.0);
            while (i > 0.0 && frac < start) { i -= 1.0; start = (pow(t, i) - 1.0) / (t - 1.0); }
            while (frac >= start + pow(t, i)) { start += pow(t, i); i += 1.0; }
            frac = (frac - start) / pow(t, i);
        }
        const double pi = 3.14159265358979323846;
        const double decayed = 0.5 * pow(s.m_mul, i) * (1.0 + cos(pi * frac));
        lr = s.initial_lr * ((1.0 - s.alpha) * decayed + s.alpha);
        break;
    }
    default:
        break;
    }
    return (float)lr;
}
