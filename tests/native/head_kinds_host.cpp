// Host build of the multi-label, Poisson and logistic heads' per-element math (ops/csrc/tfy_head.cuh), checked against
// the float64 NumPy reference by tests/test_estimator_heads.py.  The element functions and the label check are the
// kernel's own; an invalid label gives 0 and 0, as in tfy_head_checked_kernel.
#include "tfy_head.cuh"

// head 3..6: l and dl/dz of n elements, and whether each label is valid
extern "C" void tfy_host_head_kinds(int head, const float* z, const float* y, int n, float* loss, float* grad,
                                    int* ok) {
    for (int i = 0; i < n; ++i) {
        ok[i] = head == TFY_HEAD_MULTI_LABEL || tfy_head_label_ok(head, y[i]);
        if (!ok[i]) {
            loss[i] = grad[i] = 0.f;
            continue;
        }
        if (head == TFY_HEAD_POISSON || head == TFY_HEAD_POISSON_FULL) {
            loss[i] = head == TFY_HEAD_POISSON ? tfy_head_poisson_loss(z[i], y[i]) : tfy_head_poisson_full_loss(z[i], y[i]);
            grad[i] = tfy_head_poisson_grad(z[i], y[i]);
        } else {
            loss[i] = tfy_head_binary_loss(z[i], y[i]);
            grad[i] = tfy_head_binary_grad(z[i], y[i]);
        }
    }
}
