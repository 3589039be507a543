// Host build of the fused step's per-element update (ops/csrc/tfy_fused_step.cuh: tfy_step_consts + tfy_opt_update_rt),
// so that the formulas the K4 kernel applies -- SGD-momentum / Adadelta / Adam(W) / Adagrad / FTRL, bias correction
// from the device-resident step counter included -- can be checked against torch.optim on a CPU-only box.
#include <math.h>
#include <stddef.h>
#include <stdint.h>

static inline float rsqrtf(float x) { return 1.f / sqrtf(x); }

#include "tfy_fused_step.cuh"

extern "C" void tfy_host_opt_step(int opt, TfyOptHyper* hp, int world, float* p, const float* g, float* s1, float* s2,
                                  int n) {
    const TfyStepConsts k = tfy_step_consts(hp, world, opt);
    for (int i = 0; i < n; ++i) {
        float pi = p[i], a = s1[i], b = s2[i];
        tfy_opt_update_rt<-1>(opt, pi, g[i] * k.gscale, a, b, k.lr, k.p1, k.p2, k.eps, k.wd, k.flags, k.lr_bc1,
                              k.bc2_rsqrt, k.first_step);
        p[i] = pi; s1[i] = a; s2[i] = b;
    }
    hp->step += 1;
}

// the counter-based dropout generator shared by the forward kernels and the mask-recomputing backward kernels
extern "C" void tfy_host_uniform(uint32_t seed, uint32_t step, uint64_t idx0, float* out, int n) {
    for (int i = 0; i < n; ++i) out[i] = tfy_uniform(seed, step, idx0 + (uint64_t)i);
}

// fp32 -> bf16 pack (round to nearest even) and back, as the fused step stores parameters and reads gradients
extern "C" void tfy_host_bf16_roundtrip(const float* in, float* out, int n8) {
    for (int i = 0; i < n8; ++i) {
        const uint4 v = TfyPack<__nv_bfloat16>::pack(in + 8 * i);
        TfyPack<__nv_bfloat16>::unpack(v, out + 8 * i);
    }
}

// patch scheduling of the persistent convolution kernels: the (image pair, tile row, tile column) sequence of one CTA
#include "tfy_conv_index.cuh"
extern "C" void tfy_host_patch_walk(int tiles_x, int tiles_y, int n_cta, int block, int grid, int explicit_n_cta,
                                    int count, int* out) {
    blockIdx.x = (unsigned)block;
    gridDim.x = (unsigned)grid;
    CPatchIter it = explicit_n_cta ? CPatchIter(tiles_x, tiles_y, n_cta) : CPatchIter(tiles_x, tiles_y);
    for (int i = 0; i < count; ++i) {
        out[3 * i] = it.bz; out[3 * i + 1] = it.ty; out[3 * i + 2] = it.tx;
        it.next();
    }
}

// the conv2 forward's raw 32-bit dropout hash of element groups idx0 .. idx0 + n - 1 (tfy_drop_salt / TFY_DROP_HASH):
// pooled element e is kept iff byte e & 3 of the hash of group e >> 2 is >= c_drop_thr(rate)
extern "C" void tfy_host_hash_u32(uint32_t seed, uint32_t step, uint64_t idx0, uint32_t* out, int n) {
    const uint32_t salt = tfy_drop_salt(seed, step);
    for (int i = 0; i < n; ++i) out[i] = TFY_DROP_HASH(salt, idx0 + (uint64_t)i);
}

// the conv2 forward's dropout threshold and keep scale at each rate (c_drop_thr, c_keep_scale)
extern "C" void tfy_host_keep_scale(const float* rate, uint32_t* thr, float* scale, int n) {
    for (int i = 0; i < n; ++i) {
        thr[i] = c_drop_thr(rate[i]);
        scale[i] = c_keep_scale(thr[i]);
    }
}

// layout of the structs shared with Python (ctypes mirrors in tf_yarn_b200/ops/native.py)
#include <stddef.h>
extern "C" int tfy_host_struct_layout(int which, int* out, int cap) {
    int n = 0;
#define PUT(v) do { if (n < cap) out[n] = (int)(v); ++n; } while (0)
    if (which == 0) {          // TfyCommCtx
        PUT(sizeof(TfyCommCtx)); PUT(offsetof(TfyCommCtx, peer_base)); PUT(offsetof(TfyCommCtx, mc_base));
        PUT(offsetof(TfyCommCtx, epoch)); PUT(offsetof(TfyCommCtx, rank)); PUT(offsetof(TfyCommCtx, world));
        PUT(TFY_MAX_RANKS); PUT(TFY_MAX_BLOCKS); PUT(TFY_FLAGS_BYTES);
    } else if (which == 1) {   // TfyOptHyper
        PUT(sizeof(TfyOptHyper)); PUT(offsetof(TfyOptHyper, lr)); PUT(offsetof(TfyOptHyper, p1));
        PUT(offsetof(TfyOptHyper, p2)); PUT(offsetof(TfyOptHyper, eps)); PUT(offsetof(TfyOptHyper, weight_decay));
        PUT(offsetof(TfyOptHyper, grad_scale)); PUT(offsetof(TfyOptHyper, step)); PUT(offsetof(TfyOptHyper, flags));
        PUT(offsetof(TfyOptHyper, done)); PUT(offsetof(TfyOptHyper, pad));
    } else if (which == 2) {   // TfyOverlapStep
        PUT(sizeof(TfyOverlapStep)); PUT(offsetof(TfyOverlapStep, c)); PUT(offsetof(TfyOverlapStep, grad_off));
        PUT(offsetof(TfyOverlapStep, param_off)); PUT(offsetof(TfyOverlapStep, shard_n)); PUT(offsetof(TfyOverlapStep, master));
        PUT(offsetof(TfyOverlapStep, s1)); PUT(offsetof(TfyOverlapStep, s2)); PUT(offsetof(TfyOverlapStep, hp));
        PUT(offsetof(TfyOverlapStep, g0)); PUT(offsetof(TfyOverlapStep, g1)); PUT(offsetof(TfyOverlapStep, opt));
        PUT(offsetof(TfyOverlapStep, mode)); PUT(offsetof(TfyOverlapStep, n_cta)); PUT(offsetof(TfyOverlapStep, slot0));
    } else if (which == 3) {   // enums
        PUT(TFY_BF16); PUT(TFY_F32); PUT(TFY_ALGO_ONESHOT); PUT(TFY_ALGO_TWOSHOT); PUT(TFY_ALGO_NVLS);
        PUT(TFY_OPT_SGD); PUT(TFY_OPT_ADADELTA); PUT(TFY_OPT_ADAM); PUT(TFY_OPT_ADAGRAD); PUT(TFY_OPT_FTRL);
        PUT(TFY_MODE_LOCAL); PUT(TFY_MODE_P2P); PUT(TFY_MODE_NVLS);
    }
#undef PUT
    return n;
}
