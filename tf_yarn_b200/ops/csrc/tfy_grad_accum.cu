// tfy_grad_accumulate: one batch of Keras gradient accumulation (tfy_grad_accum.cuh).
//
//   acc[i] += src[i]   for the n elements of a flat gradient buffer (bf16 or fp32) and its fp32 accumulator,
//
// with 16-byte loads and stores, optionally clearing `src` behind itself (the autograd engine, whose backward adds
// into .grad, as K4 does with zero_grads), and optionally advancing the device step counter once per launch (an
// accumulation batch; on an update batch the fused step that follows advances it).  Constant-rate and scheduled forms
// are separate instantiations, as in K4.
#include "tfy_grad_accum.cuh"

// U groups of 8 elements in flight per thread: every load of a batch is issued before the first store (the asm loads
// carry a memory clobber, so the compiler does not overlap iterations by itself).
template <typename GT, bool SCHED, int U>
__global__ void __launch_bounds__(256) tfy_grad_accumulate_kernel(float* __restrict__ acc, GT* __restrict__ src,
                                                                  size_t n_groups, int clear, TfyOptHyper* hp,
                                                                  int advance) {
    tfy_pdl_sync();                                     // the gradients of this batch are complete
    using GP = TfyPack<GT>;
    constexpr int NG = 8 / GP::N;                       // 16-byte source packs per group of 8 elements
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    for (size_t g0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g0 < n_groups; g0 += nthreads * U) {
        uint4 gv[U][NG], av[U][2];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t g = g0 + (size_t)u * nthreads;
            if (g >= n_groups) continue;
            const char* sp = reinterpret_cast<const char*>(src) + g * 8 * sizeof(GT);
#pragma unroll
            for (int q = 0; q < NG; ++q) gv[u][q] = tfy_ld16(sp + q * 16);
            av[u][0] = tfy_ld16(acc + g * 8);
            av[u][1] = tfy_ld16(acc + g * 8 + 4);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t g = g0 + (size_t)u * nthreads;
            if (g >= n_groups) continue;
            float f[8];
            TfyPack<float>::unpack(av[u][0], f);
            TfyPack<float>::unpack(av[u][1], f + 4);
#pragma unroll
            for (int q = 0; q < NG; ++q) tfy_grad_accum_pack<GT>(gv[u][q], f + q * GP::N);
            tfy_st16(acc + g * 8, TfyPack<float>::pack(f));
            tfy_st16(acc + g * 8 + 4, TfyPack<float>::pack(f + 4));
            if (clear) {
                char* sp = reinterpret_cast<char*>(src) + g * 8 * sizeof(GT);
#pragma unroll
                for (int q = 0; q < NG; ++q) tfy_st16(sp + q * 16, make_uint4(0, 0, 0, 0));
            }
        }
    }
    // no other thread of this launch reads hp: one store, and the kernels of the next batch see it by stream order
    if (advance && blockIdx.x == 0 && threadIdx.x == 0) tfy_grad_accum_advance<SCHED>(hp);
}

// Resident CTAs of `kernel` at `block` threads over the device's SMs: the grid of one wave, so that every thread runs
// the U-groups loop as many times as the buffer needs rather than the grid growing past what the SMs hold at once
// (the register count allows 2 CTAs of 256 threads per SM for fp32 sources and 3 for bf16).
template <typename K>
static size_t tfy_grad_accum_wave(K kernel, int block) {
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0) != cudaSuccess || per_sm < 1)
        return (size_t)TFY_NUM_SMS * 2;
    return (size_t)per_sm * sms;
}

extern "C" {

// n: elements of both buffers (a multiple of 8; both 16-byte aligned).  src_dtype: TFY_BF16 | TFY_F32.  sched: hp heads
// a TfyHyperBlock whose schedule the counter advance evaluates (TFY_OPT_LR_SCHEDULE launches of K4 on the same block).
int tfy_grad_accumulate(float* acc, void* src, int src_dtype, size_t n, int clear, TfyOptHyper* hp, int sched,
                        int advance, cudaStream_t s) {
    if (n % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(acc) | reinterpret_cast<uintptr_t>(src)) % 16) return -3;
    if (advance && hp == nullptr) return -4;
    if (src_dtype != TFY_BF16 && src_dtype != TFY_F32) return -5;
    const size_t n_groups = n / 8;
    const int block = 256;
#define TFY_GA(T, S)                                                                                               \
    do {                                                                                                           \
        static const size_t wave = tfy_grad_accum_wave(tfy_grad_accumulate_kernel<T, S, 4>, block);                \
        size_t grid = (n_groups + block - 1) / block;                                                              \
        if (grid > wave) grid = wave;                                                                              \
        if (grid < 1) grid = 1;                                                                                    \
        tfy_launch_pdl((tfy_grad_accumulate_kernel<T, S, 4>), dim3((unsigned)grid), dim3(block), 0, s, acc,         \
                       reinterpret_cast<T*>(src), n_groups, clear, hp, advance);                                   \
    } while (0)
    if (src_dtype == TFY_BF16) {
        if (sched) TFY_GA(__nv_bfloat16, true);
        else TFY_GA(__nv_bfloat16, false);
    } else {
        if (sched) TFY_GA(float, true);
        else TFY_GA(float, false);
    }
#undef TFY_GA
    return (int)cudaGetLastError();
}

}  // extern "C"
