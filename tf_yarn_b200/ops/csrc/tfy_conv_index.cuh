// Patch scheduling and weight-gradient reduction order of the persistent convolution kernels (included by tfy_conv.cu;
// kept in its own header so that the index arithmetic can be unit-tested on the host with g++).
#pragma once
#include <stdint.h>

// Walks the patch list of a persistent CTA: p = blockIdx.x + i * gridDim.x decomposed into (image pair,
// tile row, tile column) incrementally -- no integer division per patch in the hot loops.
struct CPatchIter {
    int tx, ty, bz, sx, sy, sb, tiles_x, tiles_y;
    // n_cta: CTAs sharing the patch list (the whole grid unless the kernel carries extra communication CTAs)
    __device__ __forceinline__ CPatchIter(int tiles_x_, int tiles_y_, int n_cta = (int)gridDim.x)
        : tiles_x(tiles_x_), tiles_y(tiles_y_) {
        const int tiles = tiles_x * tiles_y;
        int p = (int)blockIdx.x;
        bz = p / tiles; p -= bz * tiles; ty = p / tiles_x; tx = p - ty * tiles_x;
        int q = n_cta;
        sb = q / tiles; q -= sb * tiles; sy = q / tiles_x; sx = q - sy * tiles_x;
    }
    __device__ __forceinline__ void next() {
        tx += sx;
        if (tx >= tiles_x) { tx -= tiles_x; ++ty; }
        ty += sy;
        if (ty >= tiles_y) { ty -= tiles_y; ++bz; }
        bz += sb;
    }
};

// Dropout of the conv2 forward (tfy_conv3x3_fprop_pool_kernel).  Its decisions come 4 to a 32-bit hash, one byte each,
// so the rate is quantised to 1/256: thr = rate * 256 rounded to nearest in fp32 (0 when rate <= 0), pooled element e
// is kept iff byte e & 3 of TFY_DROP_HASH(salt, e >> 2) (tfy_common.cuh) is >= thr, and kept values are scaled by
// 256 / (256 - thr), the inverse of the kept fraction.  That keep scale, not 1 / (1 - rate), is what the backward must
// apply (tfy_conv3x3_c32_keep_scale).  A rate of 255.5 / 256 or more drops every element (thr = 256, scale inf).
// (stdint.h only: the host builds of this header include nothing else.)
__host__ __device__ __forceinline__ uint32_t c_drop_thr(float rate) {
    return rate > 0.f ? (uint32_t)(rate * 256.f + 0.5f) : 0u;
}
__host__ __device__ __forceinline__ float c_keep_scale(uint32_t thr) { return 256.f / (256.f - (float)thr); }

// Summation order of the conv2 weight gradient's per-CTA fp32 partials (n_part of them; total4 float4 outputs,
// dW tile then db).  Output f belongs to the slice of owner f / per; the owner's slice length `len` sets how many
// thread groups (`parts`, of a threads-wide CTA) split the list of partials: part p sums partials p, p + parts, ...
// in ascending order starting from 0, and the part sums are added in order p = 0 .. parts - 1 (parts = 1: one
// serial sum).  The wgrad kernel's own reduction and the deferred reduction in the dgrad kernel both follow it, so
// dW and db are the same bits whichever kernel reduces.
struct CWgSlice {
    int lo, len, parts;
};
__host__ __device__ __forceinline__ int c_wg_per(int total4, int n_part) { return (total4 + n_part - 1) / n_part; }
__host__ __device__ __forceinline__ CWgSlice c_wg_slice(int total4, int n_part, int owner, int threads) {
    const int per = c_wg_per(total4, n_part);
    const int lo = owner * per, hi = lo + per < total4 ? lo + per : total4;
    const int len = hi > lo ? hi - lo : 0;
    return {lo, len, (len > 0 && 2 * len <= threads) ? threads / len : 1};
}
