// K4 building block shared by the stand-alone fused-step kernel (tfy_comm.cu) and by the communication CTAs that
// ride inside the persistent convolution-backward kernel (tfy_conv.cu): reduce-scatter of the owned gradient shard
// (in-switch with multimem.ld_reduce, P2P loads, or local) -> cast + 1/N scale -> optimizer update of the fp32
// master shard and its state -> all-gather of the new parameters (multimem.st / P2P stores / local).
//
// The body processes shard-relative groups of 8 elements [g_lo, g_hi) with U groups in flight per thread: all
// loads of a batch (state, then the gradient reduction, whose NVLink round trip is the long pole) are issued
// before the first dependent instruction, then the updates, then the stores.
#pragma once
#include "tfy_common.cuh"

template <typename T, int MODE_T>
__device__ __forceinline__ void tfy_reduce_pack_rt(const TfyCommCtx& c, int mode_rt, uint64_t byte_off, float* f) {
    using P = TfyPack<T>;
    const int mode = MODE_T >= 0 ? MODE_T : mode_rt;
    if (mode == TFY_MODE_LOCAL) {
        P::unpack(tfy_ld16(reinterpret_cast<const void*>(c.peer_base[c.rank] + byte_off)), f);
    } else if (mode == TFY_MODE_NVLS) {
        P::unpack(P::mc_ld_reduce(reinterpret_cast<const void*>(c.mc_base + byte_off)), f);
    } else {
#pragma unroll
        for (int i = 0; i < P::N; ++i) f[i] = 0.f;
        // fixed rank order => bit-identical result no matter which rank reduces
        for (int r0 = 0; r0 < c.world; r0 += 4) {
            uint4 v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (r0 + j < c.world)
                    v[j] = tfy_ld16_stream(reinterpret_cast<const void*>(c.peer_base[r0 + j] + byte_off));
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (r0 + j < c.world) P::accum(v[j], f);
        }
    }
}

template <int MODE_T>
__device__ __forceinline__ void tfy_bcast_pack_rt(const TfyCommCtx& c, int mode_rt, uint64_t byte_off, uint4 v) {
    const int mode = MODE_T >= 0 ? MODE_T : mode_rt;
    if (mode == TFY_MODE_LOCAL) {
        tfy_st16(reinterpret_cast<void*>(c.peer_base[c.rank] + byte_off), v);
    } else if (mode == TFY_MODE_NVLS) {
        tfy_mc_st16(reinterpret_cast<void*>(c.mc_base + byte_off), v);
    } else {
        for (int r = 0; r < c.world; ++r) {
            // start with my own replica +1 so that the N ranks do not all hit the same peer first
            int p = c.rank + 1 + r;
            if (p >= c.world) p -= c.world;
            tfy_st16_sys(reinterpret_cast<void*>(c.peer_base[p] + byte_off), v);
        }
    }
}

// The update is issue-bound, not bandwidth-bound (measured: ~170 groups of 8 per microsecond per SM with the IEEE
// sqrtf / division sequences, i.e. 38 GB/s per SM), and the communication CTAs only have a handful of SMs: the
// transcendental steps use the SFU approximations (MUFU.RSQ / MUFU.SQRT / MUFU.RCP, <= 2 ulp; inputs are
// optimizer statistics, the fp32 master weights absorb the difference far below bf16 resolution).
// (Without nvcc -- the host-side unit test of the update formulas, tests/test_native_device_code.py -- the three
// helpers are the exact functions.)
__device__ __forceinline__ float tfy_rsqrt_approx(float x) {
#ifdef __CUDACC__
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
#else
    return 1.f / sqrtf(x);
#endif
}
__device__ __forceinline__ float tfy_sqrt_approx(float x) {
#ifdef __CUDACC__
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
#else
    return sqrtf(x);
#endif
}
__device__ __forceinline__ float tfy_div_approx(float a, float b) {
#ifdef __CUDACC__
    float y;
    asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(y) : "f"(a), "f"(b));
    return y;
#else
    return a / b;
#endif
}

// one element of the update; OPT_T >= 0 folds the switch at compile time, -1 dispatches on opt_rt (uniform branch)
template <int OPT_T>
__device__ __forceinline__ void tfy_opt_update_rt(int opt_rt, float& p, float g, float& s1, float& s2, const float lr,
                                                  const float p1, const float p2, const float eps, const float wd,
                                                  const int flags, const float lr_bc1, const float bc2_rsqrt,
                                                  const bool first_step) {
    // lr_bc1 = lr / (1 - beta1^t): Adam's bias-corrected step size, computed once per launch
    const int opt = OPT_T >= 0 ? OPT_T : opt_rt;
    if (opt == TFY_OPT_SGD) {
        g += wd * p;
        if (p1 != 0.f) {
            s1 = first_step ? g : p1 * s1 + (1.f - p2) * g;
            g = (flags & 1) ? g + p1 * s1 : s1;
        }
        p -= lr * g;
    } else if (opt == TFY_OPT_ADADELTA) {
        g += wd * p;
        s1 = p1 * s1 + (1.f - p1) * g * g;                      // E[g^2]
        const float upd = g * tfy_sqrt_approx(s2 + eps) * tfy_rsqrt_approx(s1 + eps);
        s2 = p1 * s2 + (1.f - p1) * upd * upd;                  // E[dx^2]
        p -= lr * upd;
    } else if (opt == TFY_OPT_ADAM) {
        if (flags & 1) p *= (1.f - lr * wd);                    // AdamW
        else g += wd * p;
        s1 = p1 * s1 + (1.f - p1) * g;
        s2 = p2 * s2 + (1.f - p2) * g * g;
        const float denom = tfy_sqrt_approx(s2) * bc2_rsqrt + eps;
        p -= lr_bc1 * tfy_div_approx(s1, denom);
    } else if (opt == TFY_OPT_FTRL) {
        // FTRL-proximal (TF FtrlOptimizer, learning_rate_power = -0.5): s1 = n (squared-gradient accumulator),
        // s2 = z (linear term); p1 = l1, p2 = l2, eps = beta
        g += wd * p;
        const float n_new = s1 + g * g;
        const float sq_new = tfy_sqrt_approx(n_new);
        s2 += g - (sq_new - tfy_sqrt_approx(s1)) * tfy_div_approx(p, lr);
        s1 = n_new;
        p = fabsf(s2) <= p1 ? 0.f : -tfy_div_approx(s2 - copysignf(p1, s2), tfy_div_approx(eps + sq_new, lr) + 2.f * p2);
    } else if (opt == TFY_OPT_ADAMAX) {
        // tf.keras Adamax: s1 = m, s2 = u (exponentially weighted infinity norm), epsilon outside the max
        g += wd * p;
        s1 = p1 * s1 + (1.f - p1) * g;
        s2 = fmaxf(p2 * s2, fabsf(g));
        p -= lr_bc1 * tfy_div_approx(s1, s2 + eps);
    } else {  // Adagrad
        g += wd * p;
        s1 += g * g;
        p -= lr * tfy_div_approx(g, tfy_sqrt_approx(s1) + eps);
    }
}

// Three-state form: RMSprop (tf.keras): s1 = v (mean square), s2 = momentum buffer, s3 = mean gradient (centered);
// p1 = rho, p2 = momentum, flags bit 0 = centered.  As in Keras, epsilon sits inside the square root and lr inside
// the momentum buffer.  Every other optimizer ignores s3.
template <int OPT_T>
__device__ __forceinline__ void tfy_opt_update_rt(int opt_rt, float& p, float g, float& s1, float& s2, float& s3,
                                                  const float lr, const float p1, const float p2, const float eps,
                                                  const float wd, const int flags, const float lr_bc1,
                                                  const float bc2_rsqrt, const bool first_step) {
    const int opt = OPT_T >= 0 ? OPT_T : opt_rt;
    if (opt == TFY_OPT_RMSPROP) {
        g += wd * p;
        s1 = p1 * s1 + (1.f - p1) * g * g;
        float denom = s1;
        if (flags & 1) {
            s3 = p1 * s3 + (1.f - p1) * g;
            denom -= s3 * s3;
        }
        const float inc = lr * g * tfy_rsqrt_approx(denom + eps);
        if (p2 > 0.f) {
            s2 = p2 * s2 + inc;
            p -= s2;
        } else {
            p -= inc;
        }
    } else {
        tfy_opt_update_rt<OPT_T>(opt_rt, p, g, s1, s2, lr, p1, p2, eps, wd, flags, lr_bc1, bc2_rsqrt, first_step);
    }
}

// RMSprop's optional states share the s2 buffer back to back, each shard_n long, momentum first.  On return s2 is
// the momentum buffer and s3 the mean-gradient buffer, each nullptr when that state is off.
__device__ __forceinline__ void tfy_rmsprop_states(const TfyOptHyper* hp, size_t shard_n, float* __restrict__& s2,
                                                   float*& s3) {
    const bool momentum = hp->p2 > 0.f, centered = (hp->flags & 1) != 0;
    s3 = centered ? (momentum ? s2 + shard_n : s2) : nullptr;
    if (!momentum) s2 = nullptr;
}

struct TfyStepConsts {
    float lr, p1, p2, eps, wd, gscale, lr_bc1, bc2_rsqrt;
    int flags;
    bool first_step;
    float lr_mu;          // Nadam: lr mu_{t+1} / (1 - mu_product_t mu_{t+1}), the coefficient of m
    double mu_product;    // Nadam: mu_product_t, which the thread that advances the step stores (tfy_nadam_advance)
};

__device__ __forceinline__ TfyStepConsts tfy_step_consts(const TfyOptHyper* hp, int world, int opt) {
    TfyStepConsts k;
    k.lr = hp->lr; k.p1 = hp->p1; k.p2 = hp->p2; k.eps = hp->eps; k.wd = hp->weight_decay;
    k.gscale = hp->grad_scale / (float)world;
    k.flags = hp->flags;
    const int step = hp->step;  // completed steps; this launch performs step+1
    k.lr_bc1 = k.lr; k.bc2_rsqrt = 1.f;
    if (opt == TFY_OPT_ADAM) {
        const float t = (float)(step + 1);
        k.lr_bc1 = k.lr / (1.f - powf(k.p1, t));
        k.bc2_rsqrt = rsqrtf(1.f - powf(k.p2, t));
    } else if (opt == TFY_OPT_ADAMAX) {
        const float t = (float)(step + 1);
        k.lr_bc1 = k.lr / (1.f - powf(k.p1, t));
    } else if (opt == TFY_OPT_NADAM) {
        // torch.optim.NAdam with momentum_decay = 0.004: mu_t = beta1 (1 - 0.5 * 0.96^(0.004 t)); lr_bc1 is the
        // coefficient of g, lr (1 - mu_t) / (1 - mu_product_t), and lr_mu that of m
        const float t = (float)(step + 1);
        k.bc2_rsqrt = rsqrtf(1.f - powf(k.p2, t));
        const double b1 = k.p1, tt = (double)step + 1.0;
        const double mu = b1 * (1.0 - 0.5 * pow(0.96, 0.004 * tt));
        const double mu_next = b1 * (1.0 - 0.5 * pow(0.96, 0.004 * (tt + 1.0)));
        k.mu_product = reinterpret_cast<const TfyNadamHyperBlock*>(hp)->mu_product * mu;
        k.lr_bc1 = (float)((double)k.lr * (1.0 - mu) / (1.0 - k.mu_product));
        k.lr_mu = (float)((double)k.lr * mu_next / (1.0 - k.mu_product * mu_next));
    }
    k.first_step = (step == 0);
    return k;
}

// Nadam (torch.optim.NAdam, momentum_decay = 0.004; tf.keras 2's schedule_decay): s1 = m, s2 = v,
// d = sqrt(v / (1 - beta2^t)) + eps, p -= (lr_bc1 g + lr_mu m) / d with the coefficients of tfy_step_consts.
__device__ __forceinline__ void tfy_nadam_update(float& p, float g, float& s1, float& s2, const TfyStepConsts& k) {
    g += k.wd * p;
    s1 = k.p1 * s1 + (1.f - k.p1) * g;
    s2 = k.p2 * s2 + (1.f - k.p2) * g * g;
    const float d = tfy_sqrt_approx(s2) * k.bc2_rsqrt + k.eps;
    p -= tfy_div_approx(k.lr_bc1 * g + k.lr_mu * s1, d);
}

// Called by the thread that advances hp.step of a Nadam step, after every CTA has read the product (tfy_step_consts)
__device__ __forceinline__ void tfy_nadam_advance(TfyOptHyper* hp, const TfyStepConsts& k) {
    reinterpret_cast<TfyNadamHyperBlock*>(hp)->mu_product = k.mu_product;
}

// State of U groups held in registers between the (early) state loads and the update; THREE adds the third state
// of RMSprop (s3, see tfy_rmsprop_states).
template <int U, bool THREE = false>
struct TfyStepRegs {
    float4 m[U][2], x[U][2], y[U][2];
};
template <int U>
struct TfyStepRegs<U, true> {
    float4 m[U][2], x[U][2], y[U][2], z[U][2];
};

// RMSprop's s2 / s3 may be nullptr (state off): nothing is loaded or stored for them
template <int OPT_T, int U, bool THREE>
__device__ __forceinline__ void tfy_step_load_state(TfyStepRegs<U, THREE>& r, int opt_rt, const float* master,
                                                    const float* s1, const float* s2, size_t g_first, size_t stride,
                                                    size_t g_hi, const float* s3 = nullptr) {
    const int opt = OPT_T >= 0 ? OPT_T : opt_rt;
    const bool two = (opt == TFY_OPT_ADADELTA || opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL ||
                      opt == TFY_OPT_ADAMAX || opt == TFY_OPT_NADAM) ||
                     (opt == TFY_OPT_RMSPROP && s2 != nullptr);
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const size_t g8 = g_first + (size_t)u * stride;
        if (g8 < g_hi) {
            const float4* mp = reinterpret_cast<const float4*>(master + g8 * 8);
            r.m[u][0] = mp[0]; r.m[u][1] = mp[1];
            const float4* sp = reinterpret_cast<const float4*>(s1 + g8 * 8);
            r.x[u][0] = sp[0]; r.x[u][1] = sp[1];
            if (two) {
                const float4* tp = reinterpret_cast<const float4*>(s2 + g8 * 8);
                r.y[u][0] = tp[0]; r.y[u][1] = tp[1];
            }
            if constexpr (THREE) {
                if (s3 != nullptr) {
                    const float4* zp = reinterpret_cast<const float4*>(s3 + g8 * 8);
                    r.z[u][0] = zp[0]; r.z[u][1] = zp[1];
                }
            }
        }
    }
}

// Groups g_first + u*stride (u < U), all < g_hi handled; state must have been loaded into `r`.
template <typename GT, typename PT, int OPT_T, int MODE_T, int U, bool THREE>
__device__ __forceinline__ void tfy_step_batch(const TfyCommCtx& c, int opt_rt, int mode_rt, const TfyStepConsts& k,
                                               TfyStepRegs<U, THREE>& r, uint64_t grad_off, uint64_t param_off,
                                               size_t shard_start, float* master, float* s1, float* s2,
                                               size_t g_first, size_t stride, size_t g_hi, float* s3 = nullptr) {
    using GP = TfyPack<GT>;
    using PP = TfyPack<PT>;
    constexpr int NG = 8 / GP::N;  // 16-byte packs per 8 gradient elements
    constexpr int NP = 8 / PP::N;
    const int opt = OPT_T >= 0 ? OPT_T : opt_rt;
    const bool two = (opt == TFY_OPT_ADADELTA || opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL ||
                      opt == TFY_OPT_ADAMAX || opt == TFY_OPT_NADAM) ||
                     (opt == TFY_OPT_RMSPROP && s2 != nullptr);
    float g[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const size_t g8 = g_first + (size_t)u * stride;
        if (g8 < g_hi) {
            const size_t e = shard_start + g8 * 8;
#pragma unroll
            for (int q = 0; q < NG; ++q)
                tfy_reduce_pack_rt<GT, MODE_T>(c, mode_rt, grad_off + e * sizeof(GT) + q * 16, g[u] + q * GP::N);
        }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const size_t g8 = g_first + (size_t)u * stride;
        if (g8 >= g_hi) continue;
        const size_t e = shard_start + g8 * 8;
        float p[8] = {r.m[u][0].x, r.m[u][0].y, r.m[u][0].z, r.m[u][0].w,
                      r.m[u][1].x, r.m[u][1].y, r.m[u][1].z, r.m[u][1].w};
        float a[8] = {r.x[u][0].x, r.x[u][0].y, r.x[u][0].z, r.x[u][0].w,
                      r.x[u][1].x, r.x[u][1].y, r.x[u][1].z, r.x[u][1].w};
        float b[8];
        if (two) {
            b[0] = r.y[u][0].x; b[1] = r.y[u][0].y; b[2] = r.y[u][0].z; b[3] = r.y[u][0].w;
            b[4] = r.y[u][1].x; b[5] = r.y[u][1].y; b[6] = r.y[u][1].z; b[7] = r.y[u][1].w;
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) b[q] = 0.f;
        }
        if constexpr (THREE) {
            float z[8];
            if (s3 != nullptr) {
                z[0] = r.z[u][0].x; z[1] = r.z[u][0].y; z[2] = r.z[u][0].z; z[3] = r.z[u][0].w;
                z[4] = r.z[u][1].x; z[5] = r.z[u][1].y; z[6] = r.z[u][1].z; z[7] = r.z[u][1].w;
            } else {
#pragma unroll
                for (int q = 0; q < 8; ++q) z[q] = 0.f;
            }
#pragma unroll
            for (int q = 0; q < 8; ++q)
                tfy_opt_update_rt<OPT_T>(opt_rt, p[q], g[u][q] * k.gscale, a[q], b[q], z[q], k.lr, k.p1, k.p2, k.eps,
                                         k.wd, k.flags, k.lr_bc1, k.bc2_rsqrt, k.first_step);
            if (s3 != nullptr) {
                float4* zp = reinterpret_cast<float4*>(s3 + g8 * 8);
                zp[0] = make_float4(z[0], z[1], z[2], z[3]);
                zp[1] = make_float4(z[4], z[5], z[6], z[7]);
            }
        } else if constexpr (OPT_T == TFY_OPT_NADAM) {
#pragma unroll
            for (int q = 0; q < 8; ++q) tfy_nadam_update(p[q], g[u][q] * k.gscale, a[q], b[q], k);
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q)
                tfy_opt_update_rt<OPT_T>(opt_rt, p[q], g[u][q] * k.gscale, a[q], b[q], k.lr, k.p1, k.p2, k.eps, k.wd,
                                         k.flags, k.lr_bc1, k.bc2_rsqrt, k.first_step);
        }
        float4* mp = reinterpret_cast<float4*>(master + g8 * 8);
        mp[0] = make_float4(p[0], p[1], p[2], p[3]);
        mp[1] = make_float4(p[4], p[5], p[6], p[7]);
        float4* sp = reinterpret_cast<float4*>(s1 + g8 * 8);
        sp[0] = make_float4(a[0], a[1], a[2], a[3]);
        sp[1] = make_float4(a[4], a[5], a[6], a[7]);
        if (two) {
            float4* tp = reinterpret_cast<float4*>(s2 + g8 * 8);
            tp[0] = make_float4(b[0], b[1], b[2], b[3]);
            tp[1] = make_float4(b[4], b[5], b[6], b[7]);
        }
#pragma unroll
        for (int q = 0; q < NP; ++q)
            tfy_bcast_pack_rt<MODE_T>(c, mode_rt, param_off + e * sizeof(PT) + q * 16, PP::pack(p + q * PP::N));
    }
}

// ---------------------------------------------------------------------------------------------------------
// The communication role that rides inside a persistent compute kernel (tfy_conv3x3_wgrad_kernel): `n_cta`
// extra CTAs at the end of the grid run the fused step of shard-relative groups [g0, g1) -- the gradients that
// are final before that kernel starts (the Dense / head parameters of the MNIST-CNN: 98 % of the bytes) --
// while the compute CTAs run the convolution weight gradient.  Co-residency with the compute CTAs is guaranteed
// by construction (one CTA per SM, grid <= #SMs), which a second kernel on a side stream cannot promise.
// bf16 gradients and parameters; optimizer and transport are runtime values (the role is latency-bound).
// RMSprop, Adamax and Nadam have no role instantiation (RMSprop's third state and Nadam's running product are not
// part of TfyOverlapStep): the host never builds a descriptor for them (FusedShardedOptimizer.overlap_step raises)
// and the trailing launch updates every group.
// Cross-GPU protocol: ONE barrier (slots `slot0 + i`) before the reduction; the all-gathered parameters are
// published by the exit barrier of the trailing tfy_fused_step launch of the same step (stream order).
// ---------------------------------------------------------------------------------------------------------
struct TfyOverlapStep {
    TfyCommCtx c;
    uint64_t grad_off, param_off;
    size_t shard_n;
    float* master;
    float* s1;
    float* s2;
    const TfyOptHyper* hp;
    size_t g0, g1;      // shard-relative group range handled by the comm CTAs
    int32_t opt, mode;
    int32_t n_cta;      // 0 = role disabled
    int32_t slot0;      // first barrier slot used by the role
};

// barrier between same-index comm CTAs of every rank on an explicit slot (see tfy_block_barrier)
__device__ __forceinline__ void tfy_slot_barrier(const TfyCommCtx& c, uint32_t slot) {
    __syncthreads();
    if ((int)threadIdx.x < c.world) {
        const int peer = threadIdx.x;
        uint32_t* ep = c.epoch + slot * TFY_MAX_RANKS + peer;
        const uint32_t e = *ep + 1u;
        uint32_t* remote = reinterpret_cast<uint32_t*>(c.peer_base[peer]) + slot * TFY_MAX_RANKS + c.rank;
        tfy_red_release_sys_inc(remote);
        const uint32_t* mine = reinterpret_cast<const uint32_t*>(c.peer_base[c.rank]) + slot * TFY_MAX_RANKS + peer;
        while ((int32_t)(tfy_ld_acquire_sys(mine) - e) < 0) {
        }
        *ep = e;
    }
    __syncthreads();
}

// Role body: U = 2 groups in flight per thread, state held in registers (tfy_step_batch).
// Measured alternatives (round 2, tests/gpu/k4_probe.py + bench at N=1 with TFY_OVERLAP_GROUPS): per-thread cp.async
// (LDGSTS) prefetch of the 96-byte state into shared-memory slots was SLOWER (165 vs 230 groups/us per SM: LDGSTS
// issues ~14 B/clk per SM on this part); the body below moves ~8k groups on 4 SMs inside the 17 us weight gradient.
template <int OPT, int MODE, int NT>
__device__ __forceinline__ void tfy_overlap_role_body(const TfyOverlapStep& ov, int cta, uint8_t* /*smem*/) {
    constexpr int U = 2;
    const TfyCommCtx& c = ov.c;
    const TfyStepConsts k = tfy_step_consts(ov.hp, c.world, OPT);
    const size_t shard_start = (MODE == TFY_MODE_LOCAL) ? 0 : ov.shard_n * (size_t)c.rank;
    const size_t stride = (size_t)ov.n_cta * NT;
    size_t g_first = ov.g0 + (size_t)cta * NT + threadIdx.x;
    TfyStepRegs<U> r;
    tfy_step_load_state<OPT, U>(r, OPT, ov.master, ov.s1, ov.s2, g_first, stride, ov.g1);
    if (MODE != TFY_MODE_LOCAL) tfy_slot_barrier(c, (uint32_t)(ov.slot0 + cta));   // every rank's gradients are final
    for (; g_first < ov.g1; g_first += stride * U) {
        tfy_step_batch<__nv_bfloat16, __nv_bfloat16, OPT, MODE, U>(c, OPT, MODE, k, r, ov.grad_off, ov.param_off,
                                                                 shard_start, ov.master, ov.s1, ov.s2, g_first,
                                                                 stride, ov.g1);
        if (g_first + stride * U < ov.g1)
            tfy_step_load_state<OPT, U>(r, OPT, ov.master, ov.s1, ov.s2, g_first + stride * U, stride, ov.g1);
    }
}

template <int NT>
__device__ __forceinline__ void tfy_overlap_role(const TfyOverlapStep& ov, int cta, uint8_t* smem) {
#define TFY_ROLE_M(O)                                                                          \
    do {                                                                                       \
        if (ov.mode == TFY_MODE_LOCAL) tfy_overlap_role_body<O, TFY_MODE_LOCAL, NT>(ov, cta, smem);     \
        else if (ov.mode == TFY_MODE_P2P) tfy_overlap_role_body<O, TFY_MODE_P2P, NT>(ov, cta, smem);    \
        else tfy_overlap_role_body<O, TFY_MODE_NVLS, NT>(ov, cta, smem);                       \
    } while (0)
    if (ov.opt == TFY_OPT_SGD) TFY_ROLE_M(TFY_OPT_SGD);
    else if (ov.opt == TFY_OPT_ADADELTA) TFY_ROLE_M(TFY_OPT_ADADELTA);
    else if (ov.opt == TFY_OPT_ADAM) TFY_ROLE_M(TFY_OPT_ADAM);
    else if (ov.opt == TFY_OPT_FTRL) TFY_ROLE_M(TFY_OPT_FTRL);
    else TFY_ROLE_M(TFY_OPT_ADAGRAD);
#undef TFY_ROLE_M
}
