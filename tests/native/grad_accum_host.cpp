// Host build of the gradient-accumulation code (ops/csrc/tfy_grad_accum.cuh): the per-pack fp32 sum and the step
// counter / scheduled learning-rate advance of an accumulation batch, next to the advance the fused step performs on
// an update batch (tfy_comm.cu: the thread of K4 that advances the counter).
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "tfy_grad_accum.cuh"

// acc[0..n) += src[0..n) (bf16 bits when `bf16`, else fp32), pack by pack as the kernel does; n a multiple of 8
extern "C" void tfy_host_grad_accumulate(float* acc, const void* src, int bf16, size_t n) {
    const size_t per = bf16 ? 8 : 4;
    for (size_t i = 0; i < n; i += per) {
        uint4 g;
        memcpy(&g, static_cast<const char*>(src) + i * (bf16 ? 2 : 4), 16);
        if (bf16) tfy_grad_accum_pack<__nv_bfloat16>(g, acc + i);
        else tfy_grad_accum_pack<float>(g, acc + i);
    }
}

// one batch of the counter: an accumulation batch (the accumulate launch advances) or an update batch (K4 advances)
extern "C" void tfy_host_batch_advance(TfyHyperBlock* blk, int sched, int update) {
    TfyOptHyper* hp = &blk->hp;
    if (!update) {
        if (sched) tfy_grad_accum_advance<true>(hp);
        else tfy_grad_accum_advance<false>(hp);
        return;
    }
    const int step = hp->step;
    if (sched) tfy_advance_scheduled_step(hp, step);
    else hp->step = step + 1;
}
