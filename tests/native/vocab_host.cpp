// Host build of the per-element lookup of tfy_vocab_ids (ops/csrc/tfy_features.cuh), checked against the NumPy
// reference by tests/test_feature_columns_vocabulary.py, plus the layout of its parameter struct for the ctypes mirror.
#include <stddef.h>

#include "tfy_features.cuh"

extern "C" {

void tfy_host_vocab_lower_bound(const long long* x, int n, const long long* keys, int n_keys, int* out) {
    for (int i = 0; i < n; ++i) out[i] = tfy_vocab_lower_bound(x[i], keys, n_keys);
}

// every source's [B, width] ids of one launch, element by element as the kernel computes them
void tfy_host_vocab_ids(const TfyVocabParams* p) {
    for (int k = 0; k < p->S; ++k) {
        const TfyVocabSrc& s = p->srcs[k];
        long long* out = reinterpret_cast<long long*>(s.out);
        for (long long i = 0; i < (long long)p->B * s.width; ++i) out[i] = tfy_vocab_elem(s, i);
    }
}

// lower_bound of each x over the fake keys key(i) = 2 i, i < n: n up to 2^31 - 1 without storing them
struct EvenKeys {
    long long operator()(int i) const { return 2LL * i; }
};

void tfy_host_vocab_lower_bound_even(const long long* x, int n_x, int n, int* out) {
    for (int i = 0; i < n_x; ++i) out[i] = tfy_vocab_lower_bound_by(x[i], n, EvenKeys{});
}

int tfy_host_vocab_cap() { return kVocabMaxSrcs; }

// sizeof / offsetof of the structs, in the order the test lists them
void tfy_host_vocab_layout(long long* out) {
    int i = 0;
#define PUT(x) out[i++] = (long long)(x)
    PUT(sizeof(TfyVocabSrc)); PUT(offsetof(TfyVocabSrc, src)); PUT(offsetof(TfyVocabSrc, out));
    PUT(offsetof(TfyVocabSrc, keys)); PUT(offsetof(TfyVocabSrc, ids)); PUT(offsetof(TfyVocabSrc, n));
    PUT(offsetof(TfyVocabSrc, n_oov));
    PUT(offsetof(TfyVocabSrc, dflt)); PUT(offsetof(TfyVocabSrc, dtype)); PUT(offsetof(TfyVocabSrc, width));
    PUT(offsetof(TfyVocabSrc, pad));
    PUT(sizeof(TfyVocabParams)); PUT(offsetof(TfyVocabParams, B)); PUT(offsetof(TfyVocabParams, S));
    PUT(offsetof(TfyVocabParams, srcs));
#undef PUT
}

}  // extern "C"
