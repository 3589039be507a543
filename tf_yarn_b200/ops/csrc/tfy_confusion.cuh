// Bucket of one prediction in the thresholded confusion histogram of the Keras AUC / Precision / Recall metrics
// (tfy_confusion.cu).  Shared by the kernel and by the host-built unit test, so both see the same float32 arithmetic.
//
// Bucket b means "positive at every threshold j <= b": tp_j = sum of the positive weight in buckets b >= j.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define TFY_CONF_HD __host__ __device__ __forceinline__
#else
#define TFY_CONF_HD static inline
#endif

// Evenly spaced thresholds t_0 = -eps, t_j = j/(T-1), t_{T-1} = 1+eps (Keras's default): b = max(ceil(p*(T-1)) - 1, 0)
// in float32, as tf.keras's metrics_utils computes it.  p must lie in [0, 1]; b is then in [0, T-2].
TFY_CONF_HD int tfy_conf_bucket_even(float p, int num_thresholds) {
    const float s = p * (float)(num_thresholds - 1);
    const int b = (int)ceilf(s) - 1;
    return b > 0 ? b : 0;
}

// Explicit thresholds, sorted ascending: p is positive at j iff p > thr[j] (float32 compare).  The number c of
// thresholds below p gives bucket c-1; a p that is positive nowhere goes to the extra bucket T.
TFY_CONF_HD int tfy_conf_bucket_sorted(float p, const float* thr, int num_thresholds) {
    int lo = 0, hi = num_thresholds;
    while (lo < hi) {                       // first index with thr[i] >= p
        const int mid = (lo + hi) >> 1;
        if (thr[mid] < p) lo = mid + 1;
        else hi = mid;
    }
    return lo == 0 ? num_thresholds : lo - 1;
}
