// Host build of the per-element math of tfy_feature_ids (ops/csrc/tfy_features.cuh), checked against the NumPy
// reference by tests/test_feature_columns_crossed.py, plus the layout of the parameter struct for its ctypes mirror.
#include <stddef.h>

#include "tfy_features.cuh"

extern "C" {

void tfy_host_fingerprint_cat64(const uint64_t* a, const uint64_t* b, int n, uint64_t* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_fingerprint_cat64(a[i], b[i]);
}

void tfy_host_bucketize(const float* x, int n, const float* bounds, int n_bounds, int* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_feat_bucketize(x[i], bounds, n_bounds);
}

// digits [n_slots, n_widths] of every slot of a cross of the given widths
void tfy_host_digits(const int* widths, int n_widths, int* out) {
    int L = 1;
    for (int k = 0; k < n_widths; ++k) L *= widths[k];
    for (int j = 0; j < L; ++j) {
        int rem = j, span = L;
        for (int k = 0; k < n_widths; ++k) out[j * n_widths + k] = tfy_feat_digit(rem, span, widths[k]);
    }
}

// the whole [T, B, L_max] output of one launch, element by element as the kernel computes it
void tfy_host_feature_ids(const TfyFeatureParams* p) {
    long long* out = reinterpret_cast<long long*>(p->out);
    for (int t = 0; t < p->T; ++t)
        for (int b = 0; b < p->B; ++b)
            for (int j = 0; j < p->L_max; ++j) out[((size_t)t * p->B + b) * p->L_max + j] = tfy_feat_id(*p, t, b, j);
}

int tfy_host_feature_caps(int which) { return which == 0 ? kFeatMaxCols : kFeatMaxComps; }

// sizeof / offsetof of the structs, in the order the test lists them
void tfy_host_feature_layout(long long* out) {
    int i = 0;
#define PUT(x) out[i++] = (long long)(x)
    PUT(sizeof(TfyFeatComp)); PUT(offsetof(TfyFeatComp, src)); PUT(offsetof(TfyFeatComp, modulus));
    PUT(offsetof(TfyFeatComp, kind)); PUT(offsetof(TfyFeatComp, dtype)); PUT(offsetof(TfyFeatComp, width));
    PUT(offsetof(TfyFeatComp, n_bounds)); PUT(offsetof(TfyFeatComp, bounds_off)); PUT(offsetof(TfyFeatComp, pad));
    PUT(sizeof(TfyFeatCol)); PUT(offsetof(TfyFeatCol, hash_key)); PUT(offsetof(TfyFeatCol, V));
    PUT(offsetof(TfyFeatCol, comp0)); PUT(offsetof(TfyFeatCol, n_comps)); PUT(offsetof(TfyFeatCol, L));
    PUT(offsetof(TfyFeatCol, crossed));
    PUT(sizeof(TfyFeatureParams)); PUT(offsetof(TfyFeatureParams, out)); PUT(offsetof(TfyFeatureParams, bounds));
    PUT(offsetof(TfyFeatureParams, B)); PUT(offsetof(TfyFeatureParams, L_max)); PUT(offsetof(TfyFeatureParams, T));
    PUT(offsetof(TfyFeatureParams, n_comps)); PUT(offsetof(TfyFeatureParams, cols));
    PUT(offsetof(TfyFeatureParams, comps));
#undef PUT
}

}  // extern "C"
