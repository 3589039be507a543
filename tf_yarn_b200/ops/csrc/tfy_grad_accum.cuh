// Keras gradient accumulation (`gradient_accumulation_steps=N`): the per-element sum and the step-counter advance of
// tfy_grad_accumulate (tfy_grad_accum.cu), in a header that also builds for the host (g++ with
// tests/native/cuda_device_shim.h, where __device__ is empty).
//
// Every batch adds its gradients into an fp32 accumulator of the flat gradient buffer's layout; every N-th batch the
// fused optimizer step (K4) reads the accumulator instead of the gradients, scales it by hp->grad_scale = fl32(1/N),
// applies the update and clears it.  The device step counter counts batches, as Keras 3's `optimizer.iterations`
// does: the dropout kernels draw their masks from it, so the N batches of one update draw different masks, and a
// learning-rate schedule is read at the batch index of the update.  On an accumulation batch the accumulate launch
// advances the counter; on an update batch K4 does.
#pragma once
#include "tfy_common.cuh"

// acc[0..N) += the N gradients of one 16-byte pack, element by element in fp32 (N = 8 for bf16, 4 for fp32).  Each
// element is added once per launch, so the sum over batches is in batch order and bit-reproducible.
template <typename GT>
__device__ __forceinline__ void tfy_grad_accum_pack(const uint4& g, float* acc) {
    TfyPack<GT>::accum(g, acc);
}

// The counter advance of an accumulation batch, by the one thread that performs it: hp->step = step + 1 and, for a
// scheduled learning rate (SCHED: hp heads a TfyHyperBlock), hp->lr = schedule(step + 1) -- what K4 writes when it
// advances the counter, so the rate an update reads is schedule(its batch index) whichever launch advanced last.
template <bool SCHED>
__device__ __forceinline__ void tfy_grad_accum_advance(TfyOptHyper* hp) {
    const int step = hp->step;
    if constexpr (SCHED) tfy_advance_scheduled_step(hp, step);
    else hp->step = step + 1;
}
