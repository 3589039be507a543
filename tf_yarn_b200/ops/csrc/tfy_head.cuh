// Per-element loss and logit gradient of the canned estimators' heads (tfy_head.cu, ops/head.py).  Shared by the
// kernel and by the host-built unit test, so both see the same float32 arithmetic.
//
// Row i has logits z_i (C values), label y_i and weight w_i.  With c = 1 for the classification heads and c = d for
// regression, the training loss is L = sum_i w_i sum_j l_ij / (B c) and dL/dz_ij = w_i dl_ij/dz_ij / (B c):
//     binary (C = 1)       l = max(z, 0) - z y + log1p(exp(-|z|))      dl/dz = sigmoid(z) - y
//     multi-class          l = logsumexp(z_i) - z_{i, y_i}             dl/dz_j = softmax(z_i)_j - [j = y_i]
//     regression (C = d)   l = (z - y)^2                               dl/dz = 2 (z - y)
// and, with c = C for each of these (every logit is one element of the mean):
//     multi-label (C >= 2) the binary element function on every logit
//     Poisson (C = d)      l = exp(z) - y z                            dl/dz = exp(z) - y
//     Poisson, full loss   the same plus y log y - y + log(2 pi y) / 2 when y > 1 (Stirling's term; 0 for y <= 1)
//     logistic (C = 1)     the binary element function, y in [0, 1]
// A Poisson label must be >= 0 and a logistic label in [0, 1] (tfy_head_label_ok).  exp(z) is not clamped: above
// z ~ 88.7 the Poisson loss is inf, as TF's log_poisson_loss is.
// The build has no --use_fast_math: expf, logf and log1pf are the accurate ones.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define TFY_HEAD_HD __host__ __device__ __forceinline__
#else
#define TFY_HEAD_HD static inline
#endif

enum TfyHead {
    TFY_HEAD_BINARY = 0,
    TFY_HEAD_MULTI = 1,
    TFY_HEAD_REGRESSION = 2,
    TFY_HEAD_MULTI_LABEL = 3,
    TFY_HEAD_POISSON = 4,
    TFY_HEAD_POISSON_FULL = 5,
    TFY_HEAD_LOGISTIC = 6,
};

TFY_HEAD_HD float tfy_head_binary_loss(float z, float y) {
    return fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
}

// sigmoid(z), with exp of a non-positive argument only (no overflow for any z)
TFY_HEAD_HD float tfy_head_sigmoid(float z) {
    const float e = expf(-fabsf(z));
    return z >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

// sigmoid(z) - y
TFY_HEAD_HD float tfy_head_binary_grad(float z, float y) { return tfy_head_sigmoid(z) - y; }

TFY_HEAD_HD float tfy_head_regression_loss(float z, float y) {
    const float r = z - y;
    return r * r;
}

TFY_HEAD_HD float tfy_head_regression_grad(float z, float y) { return 2.f * (z - y); }

TFY_HEAD_HD float tfy_head_poisson_loss(float z, float y) { return expf(z) - y * z; }

// TF's log_poisson_loss(compute_full_loss=True), torch's poisson_nll_loss(full=True)
TFY_HEAD_HD float tfy_head_poisson_full_loss(float z, float y) {
    const float stirling = y > 1.f ? y * logf(y) - y + 0.5f * logf(6.28318531f * y) : 0.f;
    return tfy_head_poisson_loss(z, y) + stirling;
}

TFY_HEAD_HD float tfy_head_poisson_grad(float z, float y) { return expf(z) - y; }

// Whether a Poisson (count >= 0) or logistic (rate in [0, 1]) head accepts label y; NaN is never accepted.
TFY_HEAD_HD bool tfy_head_label_ok(int head, float y) {
    return head == TFY_HEAD_LOGISTIC ? (y >= 0.f && y <= 1.f) : y >= 0.f;
}

// Multi-class, given the row maximum m and s = sum_j exp(z_j - m) (s >= 1): the row's loss from its label's logit,
// and the gradient of one logit.
TFY_HEAD_HD float tfy_head_multi_loss(float m, float s, float z_label) { return (m + logf(s)) - z_label; }

TFY_HEAD_HD float tfy_head_multi_grad(float z, float m, float s, bool is_label) {
    return expf(z - m) / s - (is_label ? 1.f : 0.f);
}

// A multi-class label read as a float (float32 labels): the class it names, truncated toward zero as torch's
// .long() does, or -1 when it names none of [0, C) (NaN included).
TFY_HEAD_HD int tfy_head_class_of(float v, int C) { return (v > -1.f && v < (float)C) ? (int)v : -1; }

TFY_HEAD_HD int tfy_head_class_of(long long v, int C) { return (v >= 0 && v < (long long)C) ? (int)v : -1; }
