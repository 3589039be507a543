// Bucket ids of a tower's categorical feature columns (estimator/feature_column.py), one output element at a time.
// Shared by the kernel (tfy_features.cu) and by the host-built unit test, so both run the same integer arithmetic.
//
// Column t of a launch writes ids [B, L_max] of the int64 output [T, B, L_max]; slots j >= its own L are -1.  A column
// is either one component (identity, hashed or bucketized) whose ids are its values, or a cross of several components
// whose slot j is the mixed-radix tuple of component values (the first component varies slowest) hashed by
// FingerprintCat64.  Every id written is in [0, V) or -1.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define TFY_FEAT_HD __host__ __device__ __forceinline__
#else
#define TFY_FEAT_HD static inline
#endif

// Per-launch caps: the parameter structs travel by value in the launch (under the 4 KB kernel-parameter limit).  A
// tower with more columns, components or vocabulary sources is split over several launches by the caller
// (ops/features.py).
constexpr int kFeatMaxCols = 32;
constexpr int kFeatMaxComps = 64;

enum TfyFeatKind : int32_t {
    TFY_FEAT_RAW = 0,         // the value itself (a raw integer key of a cross); negative = missing
    TFY_FEAT_IDENTITY = 1,    // value % modulus; negative = missing
    TFY_FEAT_HASHED = 2,      // ((uint64) value * 2654435761 mod 2^32) % modulus; negative = missing
    TFY_FEAT_BUCKETIZED = 3,  // fp32 value -> upper_bound over its boundaries, + position * (n_bounds + 1)
};
enum TfyFeatDtype : int32_t { TFY_FEAT_I32 = 0, TFY_FEAT_I64 = 1, TFY_FEAT_F32 = 2 };

struct TfyFeatComp {          // one source feature read in place: [B, width] values, row-major
    uint64_t src;
    int64_t modulus;          // identity / hashed: the column's num_buckets
    int32_t kind;             // TfyFeatKind
    int32_t dtype;            // TfyFeatDtype (F32 for bucketized, I32 / I64 otherwise)
    int32_t width;            // values per example
    int32_t n_bounds;         // bucketized: number of boundaries
    int32_t bounds_off;       // bucketized: index of its first boundary in TfyFeatureParams::bounds
    int32_t pad;
};

struct TfyFeatCol {
    uint64_t hash_key;        // crossed: the initial hash
    int64_t V;                // num_buckets (crossed: hash_bucket_size)
    int32_t comp0;            // first component in TfyFeatureParams::comps
    int32_t n_comps;          // 1 unless crossed
    int32_t L;                // slots per example: the component's width, or the product of the widths of a cross
    int32_t crossed;
};

struct TfyFeatureParams {
    uint64_t out;             // int64 [T, B, L_max]
    uint64_t bounds;          // fp32 boundaries of the bucketized components
    int32_t B, L_max, T, n_comps;
    TfyFeatCol cols[kFeatMaxCols];
    TfyFeatComp comps[kFeatMaxComps];
};

TFY_FEAT_HD uint64_t tfy_shift_mix(uint64_t x) { return x ^ (x >> 47); }

// FingerprintCat64 (TF's fingerprint.h, as SparseCrossHashed chains it over a slot's components)
TFY_FEAT_HD uint64_t tfy_fingerprint_cat64(uint64_t a, uint64_t b) {
    const uint64_t M = 0xc6a4a7935bd1e995ull;
    uint64_t r = a ^ M;
    r ^= tfy_shift_mix(b * M) * M;
    r *= M;
    r = tfy_shift_mix(r) * M;
    return tfy_shift_mix(r);
}

// The number of boundaries <= x (std::upper_bound, float32 compare): NaN compares below nothing and lands past the end
TFY_FEAT_HD int tfy_feat_bucketize(float x, const float* bounds, int n) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (x < bounds[mid]) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// Mixed-radix decomposition of a cross's slot, most significant digit first: start with rem = slot and span = L (the
// product of all widths); each call peels off the digit of the next component, of the given width.
TFY_FEAT_HD int tfy_feat_digit(int& rem, int& span, int width) {
    span /= width;
    const int d = rem / span;
    rem -= d * span;
    return d;
}

// Id of value d of example b of one component (-1 = missing)
TFY_FEAT_HD long long tfy_feat_comp_id(const TfyFeatComp& c, const float* bounds, int b, int d) {
    const size_t i = (size_t)b * (size_t)c.width + (size_t)d;
    if (c.kind == TFY_FEAT_BUCKETIZED) {
        const float x = reinterpret_cast<const float*>(c.src)[i];
        return (long long)tfy_feat_bucketize(x, bounds + c.bounds_off, c.n_bounds) + (long long)d * (c.n_bounds + 1);
    }
    const long long raw = c.dtype == TFY_FEAT_I32 ? (long long)reinterpret_cast<const int32_t*>(c.src)[i]
                                                  : reinterpret_cast<const long long*>(c.src)[i];
    if (raw < 0) return -1;
    if (c.kind == TFY_FEAT_RAW) return raw;
    const long long v = c.kind == TFY_FEAT_HASHED
                            ? (long long)(((unsigned long long)raw * 2654435761ull) & 0xffffffffull) : raw;
    return v % c.modulus;
}

// Element (t, b, j) of the output.  The bag and push kernels of a group of mixed V are given the largest V, so this is
// where an id is held to its own column's [0, V): one that is not (a bucketized source wider than its column's shape,
// which the host rejects before the launch) is written as -1, absent, never as a row of another table.
TFY_FEAT_HD long long tfy_feat_id(const TfyFeatureParams& p, int t, int b, int j) {
    const TfyFeatCol& col = p.cols[t];
    if (j >= col.L) return -1;
    const float* bounds = reinterpret_cast<const float*>(p.bounds);
    if (!col.crossed) {
        const long long id = tfy_feat_comp_id(p.comps[col.comp0], bounds, b, j);
        return id < col.V ? id : -1;
    }
    uint64_t h = col.hash_key;
    int rem = j, span = col.L;
    for (int k = 0; k < col.n_comps; ++k) {
        const TfyFeatComp& c = p.comps[col.comp0 + k];
        const long long v = tfy_feat_comp_id(c, bounds, b, tfy_feat_digit(rem, span, c.width));
        if (v < 0) return -1;
        h = tfy_fingerprint_cat64(h, (uint64_t)v);
    }
    return (long long)(h % (uint64_t)col.V);
}

// ---- Vocabulary lookup (tfy_vocab_ids): raw integer values -> vocabulary ids, before tfy_feature_ids
//
// A source is one (feature, vocabulary column) pair: its [B, width] raw values are translated into an int64 [B, width]
// buffer that tfy_feature_ids then reads as an identity component of modulus num_buckets.  A source's vocabulary is an
// int64 array of its n keys sorted ascending and an int32 array of each key's id: the vocabulary's own device copy
// (feature_column.Vocabulary.tables), shared by every group and column that uses it.  A value v maps to -1 if v < 0;
// to its id if it is a key; else to n + ((uint64) v * 2654435761 mod 2^32) % n_oov when n_oov > 0; else to dflt
// (feature_column.VocabularyColumn).  n is at most 2^31 - 1.

constexpr int kVocabMaxSrcs = 32;

struct TfyVocabSrc {
    uint64_t src;             // [B, width] raw values, row-major, int32 or int64
    uint64_t out;             // int64 [B, width] ids
    uint64_t keys;            // int64 [n] sorted keys
    uint64_t ids;             // int32 [n] id of each key
    int32_t n;                // vocabulary length, in [1, 2^31 - 1]
    int32_t n_oov;            // OOV buckets (0: misses take dflt)
    int32_t dflt;             // id of a miss without OOV buckets, in [-1, n)
    int32_t dtype;            // TFY_FEAT_I32 / TFY_FEAT_I64
    int32_t width;            // values per example
    int32_t pad;
};

struct TfyVocabParams {
    int32_t B, S;             // examples, sources
    TfyVocabSrc srcs[kVocabMaxSrcs];
};

// The number of the n keys key(0) <= ... <= key(n - 1) that are < x (std::lower_bound), for any n up to 2^31 - 1:
// the midpoint lo + (hi - lo) / 2 never leaves [lo, hi), where (lo + hi) / 2 would wrap past 2^31 - 1.  `key` is a
// functor, so that the host test can search a fake key sequence of 2^31 - 1 entries without storing it.
template <class Key>
TFY_FEAT_HD int tfy_vocab_lower_bound_by(long long x, int n, const Key& key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (key(mid) < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct TfyVocabKeys {
    const long long* keys;
#if defined(__CUDACC__)
    __host__ __device__ __forceinline__
#endif
    long long operator()(int i) const { return keys[i]; }
};

TFY_FEAT_HD int tfy_vocab_lower_bound(long long x, const long long* keys, int n) {
    return tfy_vocab_lower_bound_by(x, n, TfyVocabKeys{keys});
}

// Id of one raw value of a source (-1 = missing or absent)
TFY_FEAT_HD long long tfy_vocab_id(const TfyVocabSrc& s, long long raw) {
    if (raw < 0) return -1;
    const long long* keys = reinterpret_cast<const long long*>(s.keys);
    const int pos = tfy_vocab_lower_bound(raw, keys, s.n);
    if (pos < s.n && keys[pos] == raw) return (long long)reinterpret_cast<const int32_t*>(s.ids)[pos];
    if (s.n_oov > 0)
        return (long long)s.n +
               (long long)((((unsigned long long)raw * 2654435761ull) & 0xffffffffull) % (unsigned long long)s.n_oov);
    return (long long)s.dflt;
}

// Element i of source s's [B, width] values
TFY_FEAT_HD long long tfy_vocab_elem(const TfyVocabSrc& s, long long i) {
    const long long raw = s.dtype == TFY_FEAT_I32 ? (long long)reinterpret_cast<const int32_t*>(s.src)[i]
                                                  : reinterpret_cast<const long long*>(s.src)[i];
    return tfy_vocab_id(s, raw);
}
