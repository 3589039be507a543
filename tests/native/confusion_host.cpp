// Host build of the confusion-histogram bucket functions (ops/csrc/tfy_confusion.cuh), checked against the float64
// NumPy reference by tests/test_keras_confusion_metrics.py.
#include "tfy_confusion.cuh"

extern "C" void tfy_host_conf_bucket_even(const float* p, int n, int num_thresholds, int* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_conf_bucket_even(p[i], num_thresholds);
}

extern "C" void tfy_host_conf_bucket_sorted(const float* p, int n, const float* thr, int num_thresholds, int* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_conf_bucket_sorted(p[i], thr, num_thresholds);
}
