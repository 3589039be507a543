// Bucket ids of a tower's categorical columns -- identity, hashed, bucketized and crossed, in any mix -- in one launch
// (estimator/ps_hbm.py _TableGroup, through ops/features.py).  Sources are read in place; the descriptors travel by
// value in the launch's __grid_constant__ parameter, so a captured CUDA graph replays the launch with the pointers it
// was captured with, like every other kernel of the parameter-server step.  Integer work only: the ids are bit-equal
// to the torch statement of the columns (feature_column._ids_and_weights).  The per-element math is tfy_features.cuh.
// A group with vocabulary columns first runs tfy_vocab_ids, which translates their raw values into vocabulary ids
// that tfy_feature_ids then reads as identity components.
#include <cuda_runtime.h>
#include <stdint.h>

#include "tfy_features.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocksX = 1056;                 // 8 blocks of 256 per H100 SM, split over blockIdx.y = column

__global__ void __launch_bounds__(kThreads) tfy_feature_ids_kernel(const __grid_constant__ TfyFeatureParams p) {
    const int t = blockIdx.y;
    const long long n = (long long)p.B * p.L_max;
    long long* out = reinterpret_cast<long long*>(p.out) + (size_t)t * (size_t)n;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const int b = (int)(i / p.L_max);
        out[i] = tfy_feat_id(p, t, b, (int)(i - (long long)b * p.L_max));
    }
}

// blockIdx.y = source: its B * width values, grid-stride
__global__ void __launch_bounds__(kThreads) tfy_vocab_ids_kernel(const __grid_constant__ TfyVocabParams p) {
    const TfyVocabSrc& s = p.srcs[blockIdx.y];
    const long long n = (long long)p.B * s.width;
    long long* out = reinterpret_cast<long long*>(s.out);
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads)
        out[i] = tfy_vocab_elem(s, i);
}

}  // namespace

extern "C" {

// p: host copy of the descriptors of T <= kFeatMaxCols columns over n_comps <= kFeatMaxComps components.  Returns 0,
// -1 for a descriptor out of range, -2 for B * L_max beyond int32, -3 for a null pointer, or the launch's CUDA error.
int tfy_feature_ids(const TfyFeatureParams* p, cudaStream_t s) {
    if (p == nullptr) return -3;
    if (p->T < 1 || p->T > kFeatMaxCols || p->n_comps < 1 || p->n_comps > kFeatMaxComps || p->B < 0 || p->L_max < 1)
        return -1;
    for (int t = 0; t < p->T; ++t) {
        const TfyFeatCol& c = p->cols[t];
        if (c.V < 1 || c.L < 1 || c.L > p->L_max || c.n_comps < 1 || c.comp0 < 0 || c.comp0 + c.n_comps > p->n_comps ||
            (!c.crossed && c.n_comps != 1))
            return -1;
        long long L = 1;
        for (int k = c.comp0; k < c.comp0 + c.n_comps; ++k) {
            const TfyFeatComp& q = p->comps[k];
            if (q.src == 0) return -3;
            if (q.width < 1 || (q.kind != TFY_FEAT_RAW && q.kind != TFY_FEAT_BUCKETIZED && q.modulus < 1) ||
                (q.kind == TFY_FEAT_BUCKETIZED && (q.dtype != TFY_FEAT_F32 || q.n_bounds < 1 || p->bounds == 0)) ||
                (q.kind != TFY_FEAT_BUCKETIZED && q.dtype == TFY_FEAT_F32) || (q.kind == TFY_FEAT_RAW && !c.crossed))
                return -1;
            L *= q.width;
        }
        if (L != c.L) return -1;
    }
    if (p->B == 0) return 0;
    if ((long long)p->B * p->L_max > 0x7fffffffLL) return -2;
    if (p->out == 0) return -3;
    const long long n = (long long)p->B * p->L_max;
    long long gx = (n + kThreads - 1) / kThreads;
    const long long cap = (kMaxBlocksX + p->T - 1) / p->T;
    if (gx > cap) gx = cap;
    tfy_feature_ids_kernel<<<dim3((unsigned)gx, (unsigned)p->T), kThreads, 0, s>>>(*p);
    return (int)cudaGetLastError();
}

// p: host copy of the descriptors of S <= kVocabMaxSrcs vocabulary sources.  Returns 0, -1 for a descriptor out of
// range, -2 for B * width beyond int32, -3 for a null pointer, or the launch's CUDA error.
int tfy_vocab_ids(const TfyVocabParams* p, cudaStream_t s) {
    if (p == nullptr) return -3;
    if (p->S < 1 || p->S > kVocabMaxSrcs || p->B < 0) return -1;
    long long n_max = 0;
    for (int k = 0; k < p->S; ++k) {
        const TfyVocabSrc& v = p->srcs[k];
        if (v.n < 1 || v.n_oov < 0 || v.width < 1 || v.dflt < -1 || v.dflt >= v.n ||
            (v.n_oov > 0 && v.dflt != -1) || (v.dtype != TFY_FEAT_I32 && v.dtype != TFY_FEAT_I64))
            return -1;
        if (v.src == 0 || v.keys == 0 || v.ids == 0) return -3;
        const long long n = (long long)p->B * v.width;
        if (n > n_max) n_max = n;
    }
    if (p->B == 0) return 0;
    if (n_max > 0x7fffffffLL) return -2;
    for (int k = 0; k < p->S; ++k)
        if (p->srcs[k].out == 0) return -3;
    long long gx = (n_max + kThreads - 1) / kThreads;
    const long long cap = (kMaxBlocksX + p->S - 1) / p->S;
    if (gx > cap) gx = cap;
    tfy_vocab_ids_kernel<<<dim3((unsigned)gx, (unsigned)p->S), kThreads, 0, s>>>(*p);
    return (int)cudaGetLastError();
}

}  // extern "C"
