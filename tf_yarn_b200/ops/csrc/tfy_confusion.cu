// Thresholded confusion histogram of the Keras AUC / Precision / Recall metrics (keras/metrics.py, ops/confusion.py).
//
// One launch per metric update.  For every element i of the batch, with prediction p, label y and sample weight w:
//     hist[0][b] += y * w        hist[1][b] += (1 - y) * w          (fp64, b = tfy_conf_bucket_*(p))
// added into a persistent accumulator acc[2][T+1] that the metric keeps on the device across updates, so the update
// can run inside a captured CUDA graph (no host sync, no allocation).  The curves are computed on the host from acc.
//
// Deterministic by construction -- no floating-point atomics, so two runs, and eager vs graph replay, give the same
// bits:
//   * the grid depends only on N; CTA c owns one contiguous chunk of the elements;
//   * each warp keeps a private fp64 histogram in shared memory.  Lanes whose elements fall in the same bucket are
//     grouped with __match_any_sync and the group's lowest lane adds their values in lane (= element) order;
//   * the warp histograms are summed in warp order into the CTA's slab of the caller's scratch;
//   * the last CTA to finish (ticket counter) sums the slabs in CTA order into acc and re-arms the counter.
// Invalid input (a prediction outside [0, 1] or NaN, a label outside [0, 1] or NaN) is skipped and reported by OR-ing
// bits into a flag word; the host checks it when the metric's result is read.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "tfy_confusion.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kUnroll = 4;                       // 32-element groups per warp iteration (loads in flight)
constexpr int kMaxGrid = 264;                    // two CTAs per H100 SM
constexpr int64_t kMinPerCta = kThreads * kUnroll;   // one warp iteration per warp: small batches spread over SMs
constexpr int kMaxThresholds = 1000;
constexpr size_t kTicketBytes = 16;              // the ticket counter heads the scratch; the slabs follow

constexpr uint32_t kBadPrediction = 1u;
constexpr uint32_t kBadLabel = 2u;

int conf_grid(int64_t n) {
    const int64_t g = (n + kMinPerCta - 1) / kMinPerCta;
    return (int)(g < 1 ? 1 : (g > kMaxGrid ? kMaxGrid : g));
}

size_t conf_smem_bytes(int T) {
    const size_t bins = 2 * (size_t)(T + 1);
    return (kWarps * bins + kWarps * 32 * 2) * sizeof(double) + (size_t)T * sizeof(float);
}

template <int kPredBf16, int kLabelI64>
__global__ void __launch_bounds__(kThreads)
tfy_confusion_kernel(const void* __restrict__ pred, const void* __restrict__ label, const float* __restrict__ weight,
                     int64_t n, int64_t per_sample, int T, const float* __restrict__ thresholds, int from_logits,
                     double* __restrict__ acc, uint32_t* __restrict__ flags, double* __restrict__ slabs,
                     uint32_t* __restrict__ ticket) {
    extern __shared__ double smem[];
    const int bins = 2 * (T + 1);
    double* hist_all = smem;                                   // [kWarps][2][T+1]
    double* stage_all = smem + kWarps * bins;                  // [kWarps][32][2]
    float* thr = reinterpret_cast<float*>(stage_all + kWarps * 64);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* hist = hist_all + warp * bins;
    double* stage = stage_all + warp * 64;

    for (int k = threadIdx.x; k < kWarps * bins; k += kThreads) hist_all[k] = 0.0;
    if (thresholds != nullptr)
        for (int k = threadIdx.x; k < T; k += kThreads) thr[k] = thresholds[k];
    __syncthreads();

    const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
    const int64_t begin = (int64_t)blockIdx.x * chunk;
    const int64_t end = begin + chunk < n ? begin + chunk : n;
    uint32_t bad = 0;

    for (int64_t base = begin + (int64_t)warp * 32 * kUnroll; base < end; base += (int64_t)kThreads * kUnroll) {
        float p[kUnroll], y[kUnroll], w[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {                    // all loads first: kUnroll of them in flight per lane
            const int64_t i = base + u * 32 + lane;
            p[u] = 0.f; y[u] = 0.f; w[u] = 1.f;
            if (i < end) {
                p[u] = kPredBf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(pred)[i])
                                 : reinterpret_cast<const float*>(pred)[i];
                y[u] = kLabelI64 ? (float)reinterpret_cast<const long long*>(label)[i]
                                 : reinterpret_cast<const float*>(label)[i];
                if (weight != nullptr) w[u] = weight[i / per_sample];
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const int64_t i = base + u * 32 + lane;
            int b = -1;
            double vp = 0.0, vn = 0.0;
            if (i < end) {
                float q = p[u];
                if (from_logits) q = 1.f / (1.f + expf(-q));
                const bool p_ok = q >= 0.f && q <= 1.f;        // false for NaN
                const bool y_ok = y[u] >= 0.f && y[u] <= 1.f;
                bad |= (p_ok ? 0u : kBadPrediction) | (y_ok ? 0u : kBadLabel);
                if (p_ok && y_ok) {
                    b = thresholds != nullptr ? tfy_conf_bucket_sorted(q, thr, T) : tfy_conf_bucket_even(q, T);
                    vp = (double)y[u] * (double)w[u];
                    vn = (1.0 - (double)y[u]) * (double)w[u];
                }
            }
            stage[2 * lane] = vp;
            stage[2 * lane + 1] = vn;
            const unsigned group = __match_any_sync(0xffffffffu, b);
            __syncwarp();
            if (b >= 0 && (__ffs(group) - 1) == lane) {        // the group's lowest lane adds it up in lane order
                double sp = 0.0, sn = 0.0;
                for (unsigned m = group; m != 0; m &= m - 1) {
                    const int l = __ffs(m) - 1;
                    sp += stage[2 * l];
                    sn += stage[2 * l + 1];
                }
                hist[b] += sp;
                hist[T + 1 + b] += sn;
            }
            __syncwarp();
        }
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (bad != 0 && lane == 0) atomicOr(flags, bad);
    __syncthreads();

    // warp histograms -> this CTA's slab, in warp order
    double* slab = slabs + (size_t)blockIdx.x * bins;
    for (int k = threadIdx.x; k < bins; k += kThreads) {
        double s = hist_all[k];
        for (int v = 1; v < kWarps; ++v) s += hist_all[v * bins + k];
        slab[k] = s;
    }
    __threadfence();
    __syncthreads();
    __shared__ uint32_t is_last;
    if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // the last CTA: slabs -> acc, in CTA order
    const int grid = gridDim.x;
    for (int k = threadIdx.x; k < bins; k += kThreads) {
        double s = __ldcg(slabs + k);
        int c = 1;
        for (; c + 4 <= grid; c += 4) {                        // four loads in flight, added in order
            const double a0 = __ldcg(slabs + (size_t)c * bins + k), a1 = __ldcg(slabs + (size_t)(c + 1) * bins + k);
            const double a2 = __ldcg(slabs + (size_t)(c + 2) * bins + k), a3 = __ldcg(slabs + (size_t)(c + 3) * bins + k);
            s += a0; s += a1; s += a2; s += a3;
        }
        for (; c < grid; ++c) s += __ldcg(slabs + (size_t)c * bins + k);
        acc[k] += s;
    }
    if (threadIdx.x == 0) *ticket = 0u;                        // re-armed for the next launch (and graph replay)
}

}  // namespace

extern "C" {

// Bytes of scratch one update of n elements with T thresholds needs: the ticket counter (first 16 bytes, at the same
// address for every grid size, so one buffer serves updates of any n) and then the per-CTA slabs.  The caller
// zero-fills it once; every launch leaves the counter at zero again.  n <= 0 asks for the largest grid.
size_t tfy_confusion_scratch_bytes(int64_t n, int T) {
    const int grid = n > 0 ? conf_grid(n) : kMaxGrid;
    return kTicketBytes + (size_t)grid * 2 * (size_t)(T + 1) * sizeof(double);
}

int tfy_confusion_max_thresholds() { return kMaxThresholds; }

// pred: n fp32 (pred_bf16 = 0) or bf16 (1) values; label: n fp32 (label_i64 = 0) or int64 (1) values; weight: null or
// one fp32 weight per sample, element i belonging to sample i / per_sample; thresholds: null for the evenly spaced
// default, else T fp32 values sorted ascending.  acc: fp64 [2][T+1]; flags: one uint32 (bit 0: a prediction outside
// [0, 1], bit 1: a label outside [0, 1]).  Returns 0, -1 for T out of [2, tfy_confusion_max_thresholds()], -2 for too
// little scratch, -3 for a bad argument, or the CUDA error of the launch.
int tfy_confusion_update(const void* pred, int pred_bf16, const void* label, int label_i64, const float* weight,
                         int64_t n, int64_t per_sample, int T, const float* thresholds, int from_logits, double* acc,
                         uint32_t* flags, void* scratch, size_t scratch_bytes, cudaStream_t s) {
    if (T < 2 || T > kMaxThresholds) return -1;
    if (n <= 0) return 0;
    if (pred == nullptr || label == nullptr || acc == nullptr || flags == nullptr || scratch == nullptr) return -3;
    if (weight != nullptr && per_sample <= 0) return -3;
    if (scratch_bytes < tfy_confusion_scratch_bytes(n, T)) return -2;
    const int grid = conf_grid(n);
    const size_t smem = conf_smem_bytes(T);
    uint32_t* ticket = static_cast<uint32_t*>(scratch);
    double* slabs = reinterpret_cast<double*>(static_cast<char*>(scratch) + kTicketBytes);
    auto launch = [&](auto kernel) -> int {
        if (smem > 48 * 1024) {
            const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return (int)e;
        }
        kernel<<<grid, kThreads, smem, s>>>(pred, label, weight, n, per_sample, T, thresholds, from_logits, acc, flags,
                                            slabs, ticket);
        return (int)cudaGetLastError();
    };
    if (pred_bf16) return label_i64 ? launch(tfy_confusion_kernel<1, 1>) : launch(tfy_confusion_kernel<1, 0>);
    return label_i64 ? launch(tfy_confusion_kernel<0, 1>) : launch(tfy_confusion_kernel<0, 0>);
}

}  // extern "C"
