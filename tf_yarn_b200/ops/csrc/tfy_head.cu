// The canned estimators' head (estimator/canned.py, ops/head.py): the weighted loss of a batch and its logit gradient
// in one launch, for the binary, multi-class, regression, multi-label, Poisson and logistic heads.  The per-element
// math and the loss contract are in tfy_head.cuh.
//
//   binary, regression, multi-label: one thread per logit; CTA c owns one contiguous chunk of the B*C logits.
//     Multi-label is the binary kernel itself at C >= 2 (the same element function, weight i / C, mean over B*C).
//   Poisson, logistic:  the same, in a kernel of its own that also checks each label (tfy_head_label_ok).
//   multi-class:        one warp per row, looping over C in steps of 32 (any C >= 2); CTA c owns a chunk of rows.
//
// Deterministic by construction -- no floating-point atomics, so two runs, and eager vs graph replay, give the same
// bits:
//   * the grid depends only on (B, C, head);
//   * every thread adds its w*l terms in fp64 in a fixed order, the CTA sums them lane by lane and warp by warp in a
//     fixed order and writes the sum into its own slab of the caller's scratch;
//   * the last CTA to finish (ticket counter) sums the slabs in CTA order, writes (float)(S / (B c)) and re-arms the
//     counter.
// A multi-class label outside [0, C) makes its row contribute nothing (zero loss, zero gradient; the row still counts
// in B) and sets bit 0 of the caller's flag word: bad user data is reported on the host, never a device fault.  A
// Poisson label < 0 or a logistic label outside [0, 1] (NaN included) does the same for its element, which still
// counts in B*C.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "tfy_head.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kMaxGrid = 264;                          // two CTAs per H100 SM
constexpr int64_t kMinElemsPerCta = kThreads * 4;      // binary / regression: four logits per thread at least
constexpr int64_t kMinRowsPerCta = kWarps * 4;         // multi-class: four rows per warp at least
constexpr size_t kTicketBytes = 16;                    // the ticket counter heads the scratch; the slabs follow
constexpr uint32_t kBadLabel = 1u;

enum { kLabelF32 = 0, kLabelI32 = 1, kLabelI64 = 2 };

int head_grid(int64_t B, int C, int head) {
    const int64_t items = head == TFY_HEAD_MULTI ? B : B * (int64_t)C;
    const int64_t per = head == TFY_HEAD_MULTI ? kMinRowsPerCta : kMinElemsPerCta;
    const int64_t g = (items + per - 1) / per;
    return (int)(g < 1 ? 1 : (g > kMaxGrid ? kMaxGrid : g));
}

template <int kLabel>
__device__ __forceinline__ float label_value(const void* labels, int64_t i) {
    if (kLabel == kLabelI64) return (float)reinterpret_cast<const long long*>(labels)[i];
    if (kLabel == kLabelI32) return (float)reinterpret_cast<const int*>(labels)[i];
    return reinterpret_cast<const float*>(labels)[i];
}

template <int kLabel>
__device__ __forceinline__ int label_class(const void* labels, int64_t i, int C) {
    if (kLabel == kLabelI64) return tfy_head_class_of(reinterpret_cast<const long long*>(labels)[i], C);
    if (kLabel == kLabelI32) return tfy_head_class_of((long long)reinterpret_cast<const int*>(labels)[i], C);
    return tfy_head_class_of(reinterpret_cast<const float*>(labels)[i], C);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The CTA's sum (thread 0's argument) -> its slab; the last CTA adds the slabs in CTA order and writes the loss.
__device__ __forceinline__ void finish(double cta_sum, double* __restrict__ slabs, uint32_t* __restrict__ ticket,
                                       float* __restrict__ loss, double n) {
    if (threadIdx.x != 0) return;
    slabs[blockIdx.x] = cta_sum;
    __threadfence();
    if (atomicAdd(ticket, 1u) != gridDim.x - 1) return;
    __threadfence();
    double s = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(slabs + c);
    *loss = (float)(s / n);
    *ticket = 0u;                                      // re-armed for the next launch (and graph replay)
}

template <int kHead, int kLabel>
__global__ void __launch_bounds__(kThreads)
tfy_head_elementwise_kernel(const float* __restrict__ z, const void* __restrict__ labels,
                            const float* __restrict__ weights, int64_t B, int C, float scale, float* __restrict__ loss,
                            float* __restrict__ dz, double* __restrict__ slabs, uint32_t* __restrict__ ticket) {
    __shared__ double warp_part[kWarps];
    const int64_t n = B * (int64_t)C;
    const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
    const int64_t begin = (int64_t)blockIdx.x * chunk;
    const int64_t end = begin + chunk < n ? begin + chunk : n;
    double acc = 0.0;
    for (int64_t i = begin + threadIdx.x; i < end; i += kThreads) {
        const float zi = z[i];
        const float yi = label_value<kLabel>(labels, i);
        const float wi = weights != nullptr ? weights[C == 1 ? i : i / C] : 1.f;
        const float l = kHead == TFY_HEAD_BINARY ? tfy_head_binary_loss(zi, yi) : tfy_head_regression_loss(zi, yi);
        acc += (double)wi * (double)l;
        if (dz != nullptr) {
            const float g = kHead == TFY_HEAD_BINARY ? tfy_head_binary_grad(zi, yi) : tfy_head_regression_grad(zi, yi);
            dz[i] = g * (wi * scale);
        }
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    double cta = 0.0;
    if (threadIdx.x == 0)
        for (int v = 0; v < kWarps; ++v) cta += warp_part[v];
    finish(cta, slabs, ticket, loss, (double)n);
}

template <int kHead>
__device__ __forceinline__ float checked_loss(float z, float y) {
    if (kHead == TFY_HEAD_POISSON) return tfy_head_poisson_loss(z, y);
    if (kHead == TFY_HEAD_POISSON_FULL) return tfy_head_poisson_full_loss(z, y);
    return tfy_head_binary_loss(z, y);
}

template <int kHead>
__device__ __forceinline__ float checked_grad(float z, float y) {
    return kHead == TFY_HEAD_LOGISTIC ? tfy_head_binary_grad(z, y) : tfy_head_poisson_grad(z, y);
}

// Poisson and logistic: tfy_head_elementwise_kernel plus the label check and the flag word (a kernel of its own, so
// the binary and regression instantiations keep their parameters and their code).
template <int kHead, int kLabel>
__global__ void __launch_bounds__(kThreads)
tfy_head_checked_kernel(const float* __restrict__ z, const void* __restrict__ labels,
                        const float* __restrict__ weights, int64_t B, int C, float scale, float* __restrict__ loss,
                        float* __restrict__ dz, uint32_t* __restrict__ flags, double* __restrict__ slabs,
                        uint32_t* __restrict__ ticket) {
    __shared__ double warp_part[kWarps];
    const int64_t n = B * (int64_t)C;
    const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
    const int64_t begin = (int64_t)blockIdx.x * chunk;
    const int64_t end = begin + chunk < n ? begin + chunk : n;
    double acc = 0.0;
    bool bad = false;
    for (int64_t i = begin + threadIdx.x; i < end; i += kThreads) {
        const float zi = z[i];
        const float yi = label_value<kLabel>(labels, i);
        float g = 0.f;
        if (tfy_head_label_ok(kHead, yi)) {
            const float wi = weights != nullptr ? weights[C == 1 ? i : i / C] : 1.f;
            acc += (double)wi * (double)checked_loss<kHead>(zi, yi);
            g = checked_grad<kHead>(zi, yi) * (wi * scale);
        } else {
            bad = true;
        }
        if (dz != nullptr) dz[i] = g;
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flags, kBadLabel);
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    double cta = 0.0;
    if (threadIdx.x == 0)
        for (int v = 0; v < kWarps; ++v) cta += warp_part[v];
    finish(cta, slabs, ticket, loss, (double)n);
}

template <int kLabel>
__global__ void __launch_bounds__(kThreads)
tfy_head_multi_kernel(const float* __restrict__ z, const void* __restrict__ labels, const float* __restrict__ weights,
                      int64_t B, int C, float scale, float* __restrict__ loss, float* __restrict__ dz,
                      uint32_t* __restrict__ flags, double* __restrict__ slabs, uint32_t* __restrict__ ticket) {
    __shared__ double warp_part[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t chunk = (B + gridDim.x - 1) / gridDim.x;
    const int64_t begin = (int64_t)blockIdx.x * chunk;
    const int64_t end = begin + chunk < B ? begin + chunk : B;
    double acc = 0.0;                                  // lane 0's running sum of this warp's rows
    bool bad = false;
    for (int64_t r = begin + warp; r < end; r += kWarps) {
        const float* zr = z + r * C;
        float* dr = dz != nullptr ? dz + r * C : nullptr;
        const int y = label_class<kLabel>(labels, r, C);        // the same in every lane: the branch is warp-uniform
        if (y < 0) {
            bad = true;
            if (dr != nullptr)
                for (int j = lane; j < C; j += 32) dr[j] = 0.f;
            continue;
        }
        const float wi = weights != nullptr ? weights[r] : 1.f;
        float m = -INFINITY;
        for (int j = lane; j < C; j += 32) m = fmaxf(m, zr[j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float s = 0.f;
        for (int j = lane; j < C; j += 32) s += expf(zr[j] - m);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);   // equal in every lane
        if (lane == 0) acc += (double)wi * (double)tfy_head_multi_loss(m, s, zr[y]);
        if (dr != nullptr) {
            const float f = wi * scale;
            for (int j = lane; j < C; j += 32) dr[j] = tfy_head_multi_grad(zr[j], m, s, j == y) * f;
        }
    }
    if (bad && lane == 0) atomicOr(flags, kBadLabel);
    if (lane == 0) warp_part[warp] = acc;
    __syncthreads();
    double cta = 0.0;
    if (threadIdx.x == 0)
        for (int v = 0; v < kWarps; ++v) cta += warp_part[v];
    finish(cta, slabs, ticket, loss, (double)B);
}

}  // namespace

extern "C" {

// Bytes of scratch one launch for a batch of B rows of C logits needs: the ticket counter (first 16 bytes, at the same
// address for every grid size, so one buffer serves batches of any B) and then one fp64 slab per CTA.  The caller
// zero-fills it once; every launch leaves the counter at zero again.  B <= 0 asks for the largest grid.
size_t tfy_canned_head_scratch_bytes(int64_t B, int C, int head) {
    const int grid = B > 0 && C > 0 ? head_grid(B, C, head) : kMaxGrid;
    return kTicketBytes + (size_t)grid * sizeof(double);
}

// logits: fp32 [B, C] row-major.  labels: B*C values (binary, logistic: C = 1; regression, Poisson: [B, d];
// multi-label: [B, C]) or B class ids (multi-class), read in place as fp32 (label_dtype 0), int32 (1) or int64 (2).
// weights: null (every example weighs 1) or fp32 [B].  head: 0 binary (C must be 1), 1 multi-class (C >= 2),
// 2 regression (C = d >= 1), 3 multi-label (C >= 2), 4 Poisson and 5 Poisson with the full loss (C = d >= 1),
// 6 logistic (C = 1).  loss: one fp32, the batch's weighted loss sum_i w_i sum_j l_ij / (B c).  dlogits: null (loss
// only) or fp32 [B, C], dL/dlogits.  flags: one uint32 (bit 0: a multi-class label outside [0, C), a Poisson label
// < 0 or a logistic label outside [0, 1]); bits are only ever set; it may be null for heads 0, 2 and 3.  scratch: at
// least tfy_canned_head_scratch_bytes(B, C, head) bytes, zero-filled before the first launch.  Returns 0, -1 for a
// bad head code or a C the head does not allow, -3 for a bad argument, or the CUDA error of the launch.
int tfy_canned_head(const float* logits, const void* labels, int label_dtype, const float* weights, int64_t B, int C,
                    int head, float* loss, float* dlogits, uint32_t* flags, void* scratch, cudaStream_t s) {
    const bool checked = head == TFY_HEAD_POISSON || head == TFY_HEAD_POISSON_FULL || head == TFY_HEAD_LOGISTIC;
    if (head == TFY_HEAD_BINARY || head == TFY_HEAD_LOGISTIC ? C != 1
        : head == TFY_HEAD_MULTI || head == TFY_HEAD_MULTI_LABEL ? C < 2
        : head == TFY_HEAD_REGRESSION || head == TFY_HEAD_POISSON || head == TFY_HEAD_POISSON_FULL ? C < 1
        : true)
        return -1;
    if (B <= 0 || logits == nullptr || labels == nullptr || loss == nullptr || scratch == nullptr) return -3;
    if (label_dtype < kLabelF32 || label_dtype > kLabelI64 || ((head == TFY_HEAD_MULTI || checked) && flags == nullptr))
        return -3;
    const int grid = head_grid(B, C, head);
    const int64_t per_loss = head == TFY_HEAD_MULTI ? B : B * (int64_t)C;      // B c
    const float scale = (float)(1.0 / (double)per_loss);
    uint32_t* ticket = static_cast<uint32_t*>(scratch);
    double* slabs = reinterpret_cast<double*>(static_cast<char*>(scratch) + kTicketBytes);
    auto elementwise = [&](auto kernel) -> int {
        kernel<<<grid, kThreads, 0, s>>>(logits, labels, weights, B, C, scale, loss, dlogits, slabs, ticket);
        return (int)cudaGetLastError();
    };
    auto flagged = [&](auto kernel) -> int {
        kernel<<<grid, kThreads, 0, s>>>(logits, labels, weights, B, C, scale, loss, dlogits, flags, slabs, ticket);
        return (int)cudaGetLastError();
    };
    if (head == TFY_HEAD_MULTI) {
        if (label_dtype == kLabelI64) return flagged(tfy_head_multi_kernel<kLabelI64>);
        if (label_dtype == kLabelI32) return flagged(tfy_head_multi_kernel<kLabelI32>);
        return flagged(tfy_head_multi_kernel<kLabelF32>);
    }
    if (head == TFY_HEAD_POISSON) {
        if (label_dtype == kLabelI64) return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON, kLabelI64>);
        if (label_dtype == kLabelI32) return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON, kLabelI32>);
        return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON, kLabelF32>);
    }
    if (head == TFY_HEAD_POISSON_FULL) {
        if (label_dtype == kLabelI64) return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON_FULL, kLabelI64>);
        if (label_dtype == kLabelI32) return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON_FULL, kLabelI32>);
        return flagged(tfy_head_checked_kernel<TFY_HEAD_POISSON_FULL, kLabelF32>);
    }
    if (head == TFY_HEAD_LOGISTIC) {
        if (label_dtype == kLabelI64) return flagged(tfy_head_checked_kernel<TFY_HEAD_LOGISTIC, kLabelI64>);
        if (label_dtype == kLabelI32) return flagged(tfy_head_checked_kernel<TFY_HEAD_LOGISTIC, kLabelI32>);
        return flagged(tfy_head_checked_kernel<TFY_HEAD_LOGISTIC, kLabelF32>);
    }
    if (head == TFY_HEAD_BINARY || head == TFY_HEAD_MULTI_LABEL) {
        if (label_dtype == kLabelI64) return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_BINARY, kLabelI64>);
        if (label_dtype == kLabelI32) return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_BINARY, kLabelI32>);
        return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_BINARY, kLabelF32>);
    }
    if (label_dtype == kLabelI64) return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_REGRESSION, kLabelI64>);
    if (label_dtype == kLabelI32) return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_REGRESSION, kLabelI32>);
    return elementwise(tfy_head_elementwise_kernel<TFY_HEAD_REGRESSION, kLabelF32>);
}

}  // extern "C"
