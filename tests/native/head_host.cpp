// Host build of the canned heads' per-element math (ops/csrc/tfy_head.cuh), checked against the float64 NumPy
// reference by tests/test_canned_regressors_and_weights.py.  The multi-class row is reduced sequentially here (the
// kernel reduces across a warp); the element functions are the kernel's own.
#include "tfy_head.cuh"

// head 0 (binary) or 2 (regression): l and dl/dz of n elements
extern "C" void tfy_host_head_elementwise(int head, const float* z, const float* y, int n, float* loss, float* grad) {
    for (int i = 0; i < n; ++i) {
        loss[i] = head == TFY_HEAD_BINARY ? tfy_head_binary_loss(z[i], y[i]) : tfy_head_regression_loss(z[i], y[i]);
        grad[i] = head == TFY_HEAD_BINARY ? tfy_head_binary_grad(z[i], y[i]) : tfy_head_regression_grad(z[i], y[i]);
    }
}

// multi-class: the loss of each of B rows of C logits and dl/dz; a rejected label gives 0 and a zero row
extern "C" void tfy_host_head_multi(const float* z, const long long* labels, int B, int C, float* loss, float* grad) {
    for (int r = 0; r < B; ++r) {
        const float* zr = z + (long long)r * C;
        float* gr = grad + (long long)r * C;
        const int y = tfy_head_class_of(labels[r], C);
        if (y < 0) {
            loss[r] = 0.f;
            for (int j = 0; j < C; ++j) gr[j] = 0.f;
            continue;
        }
        float m = -INFINITY;
        for (int j = 0; j < C; ++j) m = fmaxf(m, zr[j]);
        float s = 0.f;
        for (int j = 0; j < C; ++j) s += expf(zr[j] - m);
        loss[r] = tfy_head_multi_loss(m, s, zr[y]);
        for (int j = 0; j < C; ++j) gr[j] = tfy_head_multi_grad(zr[j], m, s, j == y);
    }
}

extern "C" void tfy_host_head_class_of_f32(const float* v, int n, int C, int* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_head_class_of(v[i], C);
}
