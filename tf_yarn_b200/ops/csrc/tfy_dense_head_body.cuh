// Body of the fused classifier-head kernels of tfy_nn.cu (tfy_dense_head_fused_kernel,
// tfy_dense_head_fused_soft_kernel and tfy_dense_head_fused_binary_kernel): a statement sequence, included inside each
// kernel after its tfy_pdl_sync(), in the scope of the kernel's parameters and of the constants TARGET
// (TFY_HEAD_SPARSE, TFY_HEAD_DENSE or TFY_HEAD_BINARY), `labels`, `targets`, `ls` and `sigmoid_out` (the ones a mode
// does not read are null / 0 / false).  It is a textual include rather than a shared
// __device__ function because inlining such a function compiles the existing sparse instantiations to different
// (reordered) SASS; included, they stay instruction for instruction what they were.
    long long* const n_tl = n_timeline;
    const long long n_t0 = clock64();
    extern __shared__ __align__(16) uint8_t head_smem[];
    constexpr int KP = K + 8;                                       // padded row (bank spread)
    constexpr int NRED = WEIGHTED ? 4 : 2;                          // per-warp sums: loss, correct (, w*correct, w)
    __nv_bfloat16* s_h = reinterpret_cast<__nv_bfloat16*>(head_smem);                 // [16][KP]
    float* s_w = reinterpret_cast<float*>(head_smem + (size_t)HEAD_ROWS * KP * 2);    // [16][K], rows >= C are zero
    float* s_dl = s_w + (size_t)HEAD_CMAX * K;                                                // [16][HEAD_CMAX]
    float* s_b = s_dl + HEAD_ROWS * HEAD_CMAX;                                        // [HEAD_CMAX]
    float* s_red = s_b + HEAD_CMAX;                                                   // [warp][NRED]
    float* s_col = s_red + NRED * HEAD_WARPS;                                         // [max(K, 256)], 16-byte aligned
    __shared__ uint32_t s_last;
    const int tid = threadIdx.x;
    const int row0 = blockIdx.x * HEAD_ROWS;
    const int rows = min(HEAD_ROWS, B - row0);
    const size_t slab = (size_t)C * K + HEAD_CMAX + K + 4;          // this CTA's partial sums
    float* g_dw = scratch + blockIdx.x * slab;
    float* g_db2 = g_dw + (size_t)C * K;
    float* g_db1 = g_db2 + HEAD_CMAX;
    float* g_red = g_db1 + K;

    // ---- A: stage this CTA's rows of h (bf16), W2 and b2 (fp32)
    const int kv = K / 8;
    for (int i = tid; i < HEAD_ROWS * kv; i += HEAD_THREADS) {
        const int r = i / kv, g = i - r * kv;
        *reinterpret_cast<uint4*>(s_h + (size_t)r * KP + g * 8) =
            r < rows ? tfy_ld16(h + (size_t)(row0 + r) * K + g * 8) : make_uint4(0, 0, 0, 0);
    }
    {
        constexpr int WV = HEAD_CMAX * K / 8 / HEAD_THREADS;        // 16-byte packs of W2 per thread (upper bound)
        uint4 wv[WV];
#pragma unroll
        for (int q = 0; q < WV; ++q) {
            const int i = tid + q * HEAD_THREADS;
            wv[q] = i < C * K / 8 ? tfy_ld16(w2 + (size_t)i * 8) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int q = 0; q < WV; ++q) {                          // packs beyond C*K/8 were loaded as zeros
            const int i = tid + q * HEAD_THREADS;
            TfyPack<__nv_bfloat16>::unpack(wv[q], s_w + (size_t)i * 8);
        }
    }
    if (tid < HEAD_CMAX) s_b[tid] = (tid < C && b2) ? bf16_to_f(b2[tid]) : 0.f;
    for (int i = tid; i < HEAD_ROWS * HEAD_CMAX; i += HEAD_THREADS) s_dl[i] = 0.f;
    __syncthreads();

    N_MARK(1);
    // ---- B/C: logits (16 threads per row), softmax, loss, dlogits
    const float invB = 1.f / (float)B;
    {
        // Classes are padded to 16 with zero weights (no per-class branches) and taken 4 at a time in a ROLLED
        // loop: this code runs once per launch on 8 warps, so it is instruction-fetch bound -- the fully
        // unrolled version (2400 instructions) spent 7k cycles here, mostly waiting for the I-cache.
        const int r = tid >> 4, part = tid & 15;
        constexpr int kq = K / 16;
        // the row's class, issued early: used after the GEMV (DENSE: argmax_c y_rc, y_rc held by lane c; BINARY: the
        // same for C > 1, round(y_r0) half to even for C = 1)
        int lab = -1;
        [[maybe_unused]] float y = 0.f;                            // DENSE, BINARY: this lane's target y_rc
        if constexpr (TARGET == TFY_HEAD_SPARSE) {
            lab = r < rows ? (int)labels[row0 + r] : -1;
        } else {
            const bool in = r < rows && part < C;
            y = in ? targets[(size_t)(row0 + r) * C + part] : 0.f;
            float ym = in ? y : -INFINITY;
            int ya = part;
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, ym, off);
                const int oa = __shfl_xor_sync(0xffffffffu, ya, off);
                if (ov > ym || (ov == ym && oa < ya)) { ym = ov; ya = oa; }
            }
            if (r < rows) lab = ya;
            if constexpr (TARGET == TFY_HEAD_BINARY) {
                if (r < rows && C == 1) lab = __float2int_rn(ym);      // ym: the row's only target
            }
        }
        float wr = 0.f;                                             // this row's weight (WEIGHTED only)
        if constexpr (WEIGHTED) {
            if (r < rows) {
                wr = sample_w ? sample_w[row0 + r] : 1.f;
                // (a binary head's class table has max(C, 2) entries: classes 0 and 1 when C = 1)
                if (class_w && lab >= 0 && lab < (TARGET == TFY_HEAD_BINARY ? max(C, 2) : C)) wr *= class_w[lab];
            }
        }
        const __nv_bfloat16* hr = s_h + (size_t)r * KP + part * kq;
        float* s_logit = s_col;                                     // [16][16] scratch (s_col is used later)
#pragma unroll 1
        for (int cb = 0; cb < HEAD_CMAX; cb += 4) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
            for (int k = 0; k < kq; k += 8) {
                float hv[8];
                TfyPack<__nv_bfloat16>::unpack(*reinterpret_cast<const uint4*>(hr + k), hv);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float* wp = s_w + (size_t)(cb + c) * K + part * kq + k;
                    const float4 w0 = *reinterpret_cast<const float4*>(wp);
                    const float4 w1 = *reinterpret_cast<const float4*>(wp + 4);
                    acc[c] = fmaf(hv[0], w0.x, acc[c]); acc[c] = fmaf(hv[1], w0.y, acc[c]);
                    acc[c] = fmaf(hv[2], w0.z, acc[c]); acc[c] = fmaf(hv[3], w0.w, acc[c]);
                    acc[c] = fmaf(hv[4], w1.x, acc[c]); acc[c] = fmaf(hv[5], w1.y, acc[c]);
                    acc[c] = fmaf(hv[6], w1.z, acc[c]); acc[c] = fmaf(hv[7], w1.w, acc[c]);
                }
            }
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) {
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], off);
            }
            if (part == 0) *reinterpret_cast<float4*>(s_logit + r * HEAD_CMAX + cb) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        }
        __syncwarp();
        // softmax / cross-entropy with one lane per class (the 16 lanes of a row group): a handful of shuffle
        // steps instead of three serial 10-iteration loops on one lane per row
        if constexpr (TARGET == TFY_HEAD_BINARY) {
            // sigmoid cross-entropy, one lane per output: every logit is one element of the row's mean
            const int c = part;
            const bool live = c < C && r < rows;
            const float z = live ? s_logit[r * HEAD_CMAX + c] + s_b[c] : 0.f;
            const float t = fmaf(y, 1.f - ls, 0.5f * ls);
            const float sg = tfy_head_sigmoid(z);
            const float invC = 1.f / (float)C;
            const float out = sigmoid_out ? sg : z;                 // the model's output, as binary_accuracy reads it
            const bool hit = live && ((out > 0.5f) == (y > 0.5f));
            float dz = (sg - t) * (invB * invC);
            if constexpr (WEIGHTED) dz *= wr;
            if (live) s_dl[r * HEAD_CMAX + c] = dz;
            float my_loss = live ? tfy_head_binary_loss(z, t) * invC : 0.f;
            float my_correct = hit ? 1.f : 0.f;
            float my_wcorrect = 0.f, my_w = 0.f;
            if constexpr (WEIGHTED) {
                my_loss *= wr;
                my_wcorrect = hit ? wr * invC : 0.f;
                my_w = (c == 0 && r < rows) ? wr : 0.f;             // once per row
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                my_loss += __shfl_xor_sync(0xffffffffu, my_loss, off);
                my_correct += __shfl_xor_sync(0xffffffffu, my_correct, off);
                if constexpr (WEIGHTED) {
                    my_wcorrect += __shfl_xor_sync(0xffffffffu, my_wcorrect, off);
                    my_w += __shfl_xor_sync(0xffffffffu, my_w, off);
                }
            }
            if ((tid & 31) == 0) {
                s_red[NRED * (tid >> 5)] = my_loss;
                s_red[NRED * (tid >> 5) + 1] = my_correct;
                if constexpr (WEIGHTED) {
                    s_red[NRED * (tid >> 5) + 2] = my_wcorrect;
                    s_red[NRED * (tid >> 5) + 3] = my_w;
                }
            }
        } else {
            const int c = part;
            const bool live = c < C && r < rows;
            const float v = live ? s_logit[r * HEAD_CMAX + c] + s_b[c] : -3.0e38f;
            float mx = v;
            int amax = c;
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, mx, off);
                const int oa = __shfl_xor_sync(0xffffffffu, amax, off);
                if (ov > mx || (ov == mx && oa < amax)) { mx = ov; amax = oa; }
            }
            const float e = live ? __expf(v - mx) : 0.f;
            float se = e;
#pragma unroll
            for (int off = 1; off < 16; off <<= 1) se += __shfl_xor_sync(0xffffffffu, se, off);
            const bool hit = live && c == lab;
            if constexpr (TARGET == TFY_HEAD_SPARSE) {
                if constexpr (WEIGHTED) {
                    if (live) s_dl[r * HEAD_CMAX + c] = (e / se - (hit ? 1.f : 0.f)) * invB * wr;
                } else {
                    if (live) s_dl[r * HEAD_CMAX + c] = (e / se - (hit ? 1.f : 0.f)) * invB;
                }
            }
            float my_loss = hit ? (mx + __logf(se)) - v : 0.f;
            if constexpr (TARGET == TFY_HEAD_DENSE) {
                const float t = live ? fmaf(y, 1.f - ls, ls / (float)C) : 0.f;
                float S = t;
#pragma unroll
                for (int off = 1; off < 16; off <<= 1) S += __shfl_xor_sync(0xffffffffu, S, off);
                if constexpr (WEIGHTED) {
                    if (live) s_dl[r * HEAD_CMAX + c] = (e / se * S - t) * invB * wr;
                } else {
                    if (live) s_dl[r * HEAD_CMAX + c] = (e / se * S - t) * invB;
                }
                my_loss = live ? t * ((mx + __logf(se)) - v) : 0.f;
            }
            float my_correct = (hit && amax == lab) ? 1.f : 0.f;
            float my_wcorrect = 0.f, my_w = 0.f;
            if constexpr (WEIGHTED) {
                my_loss *= wr;
                my_wcorrect = my_correct * wr;
                my_w = (c == 0 && r < rows) ? wr : 0.f;             // once per row
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                my_loss += __shfl_xor_sync(0xffffffffu, my_loss, off);
                my_correct += __shfl_xor_sync(0xffffffffu, my_correct, off);
                if constexpr (WEIGHTED) {
                    my_wcorrect += __shfl_xor_sync(0xffffffffu, my_wcorrect, off);
                    my_w += __shfl_xor_sync(0xffffffffu, my_w, off);
                }
            }
            if ((tid & 31) == 0) {
                s_red[NRED * (tid >> 5)] = my_loss;
                s_red[NRED * (tid >> 5) + 1] = my_correct;
                if constexpr (WEIGHTED) {
                    s_red[NRED * (tid >> 5) + 2] = my_wcorrect;
                    s_red[NRED * (tid >> 5) + 3] = my_w;
                }
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < K; i += HEAD_THREADS) s_col[i] = 0.f;     // s_logit scratch -> column sums
    __syncthreads();
    if (tid == 0) {
        float l = 0.f, c = 0.f;
        for (int w = 0; w < HEAD_WARPS; ++w) { l += s_red[NRED * w]; c += s_red[NRED * w + 1]; }
        __stcg(g_red, l);
        __stcg(g_red + 1, c);
        if constexpr (WEIGHTED) {
            float wc = 0.f, ws = 0.f;
            for (int w = 0; w < HEAD_WARPS; ++w) { wc += s_red[NRED * w + 2]; ws += s_red[NRED * w + 3]; }
            __stcg(g_red + 2, wc);
            __stcg(g_red + 3, ws);
        }
    }

    N_MARK(2);
    // ---- D: partial dW2[c][k] = sum_r dl[r][c] h[r][k]; db2[c] = sum_r dl[r][c]
    {
        // a thread keeps one column k of h (16 values) in registers and runs over the classes it owns
        constexpr int KREP = K >= HEAD_THREADS ? K / HEAD_THREADS : 1;
        constexpr int CSTEP = K >= HEAD_THREADS ? 1 : HEAD_THREADS / K;
#pragma unroll
        for (int kr = 0; kr < KREP; ++kr) {
            const int k = (K >= HEAD_THREADS) ? tid + kr * HEAD_THREADS : tid % K;
            float hc[HEAD_ROWS];
#pragma unroll
            for (int r = 0; r < HEAD_ROWS; ++r) hc[r] = bf16_to_f(s_h[(size_t)r * KP + k]);
#pragma unroll 1
            for (int cc = 0; cc < HEAD_CMAX / CSTEP; ++cc) {
                const int c = cc * CSTEP + ((K >= HEAD_THREADS) ? 0 : tid / K);
                if (c >= C) break;
                float a = 0.f;
#pragma unroll
                for (int r = 0; r < HEAD_ROWS; ++r) a = fmaf(s_dl[r * HEAD_CMAX + c], hc[r], a);
                if (c < C) __stcg(g_dw + (size_t)c * K + k, a);
            }
        }
    }
    if (tid < C) {
        float a = 0.f;
#pragma unroll
        for (int r = 0; r < HEAD_ROWS; ++r) a += s_dl[r * HEAD_CMAX + tid];
        __stcg(g_db2 + tid, a);
    }

    N_MARK(3);
    // ---- E: dh[r][k] = (sum_c dl[r][c] W2[c][k]) * gate * scale; db1[k] = sum_r dh[r][k]
    if (dh) {
        // a thread keeps one column k of W2 (16 classes) in registers and runs over the rows it owns
        constexpr int KREP = K >= HEAD_THREADS ? K / HEAD_THREADS : 1;
        constexpr int RSTEP = K >= HEAD_THREADS ? 1 : HEAD_THREADS / K;
#pragma unroll
        for (int kr = 0; kr < KREP; ++kr) {
            const int k = (K >= HEAD_THREADS) ? tid + kr * HEAD_THREADS : tid % K;
            const int rbase = (K >= HEAD_THREADS) ? 0 : tid / K;
            float wk[HEAD_CMAX];
#pragma unroll
            for (int c = 0; c < HEAD_CMAX; ++c) wk[c] = s_w[(size_t)c * K + k];
            uint32_t mkbits = 0;                                    // gate bits of the rows this thread owns
#pragma unroll
            for (int j = 0; j < HEAD_ROWS / RSTEP; ++j) {
                const int r = rbase + j * RSTEP;
                const uint32_t bit = (mask1 && r < rows) ? (uint32_t)(mask1[(size_t)(row0 + r) * K + k] & 1) : 1u;
                mkbits |= bit << j;
            }
            float col = 0.f;
#pragma unroll 2
            for (int j = 0; j < HEAD_ROWS / RSTEP; ++j) {
                const int r = rbase + j * RSTEP;
                float v = 0.f;
#pragma unroll
                for (int c4 = 0; c4 < HEAD_CMAX; c4 += 4) {
                    const float4 d = *reinterpret_cast<const float4*>(s_dl + r * HEAD_CMAX + c4);
                    v = fmaf(d.x, wk[c4], v); v = fmaf(d.y, wk[c4 + 1], v);
                    v = fmaf(d.z, wk[c4 + 2], v); v = fmaf(d.w, wk[c4 + 3], v);
                }
                if (mask1) v = ((mkbits >> j) & 1u) ? v * scale1 : 0.f;
                if (r < rows) {
                    dh[(size_t)(row0 + r) * K + k] = __float2bfloat16(v);
                    col += v;
                }
            }
            if (db1) atomicAdd(&s_col[k], col);     // at most two addends per column: order-independent
        }
        if (db1) {
            __syncthreads();
            for (int k = tid; k < K; k += HEAD_THREADS) __stcg(g_db1 + k, s_col[k]);
        }
    }

    N_MARK(4);
    // ---- the last CTA converts the batch sums and clears the scratch buffer
    __threadfence();
    __syncthreads();
    N_MARK(5);
    if (tid == 0) s_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
    __syncthreads();
    N_MARK(6);
    if (s_last) {
        __threadfence();
        const int G = (int)gridDim.x;
        {
            constexpr int FV = HEAD_CMAX * K / 4 / HEAD_THREADS;    // float4 packs per thread (upper bound)
            float4 fv[FV];
#pragma unroll
            for (int q = 0; q < FV; ++q) fv[q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
            for (int g = 0; g < G; ++g) {                           // CTA order; unrolled: loads in flight together
                float4* src = reinterpret_cast<float4*>(scratch + (size_t)g * slab);
#pragma unroll
                for (int q = 0; q < FV; ++q) {
                    const int i = tid + q * HEAD_THREADS;
                    if (i < C * K / 4) {
                        const float4 v = __ldcg(src + i);
                        fv[q].x += v.x; fv[q].y += v.y; fv[q].z += v.z; fv[q].w += v.w;
                        __stcg(src + i, make_float4(0.f, 0.f, 0.f, 0.f));
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < FV; ++q) {
                const int i = tid + q * HEAD_THREADS;
                if (i < C * K / 4) {
                    __nv_bfloat162 lo = __floats2bfloat162_rn(fv[q].x, fv[q].y), hi = __floats2bfloat162_rn(fv[q].z, fv[q].w);
                    uint2 packed;
                    packed.x = *reinterpret_cast<uint32_t*>(&lo);
                    packed.y = *reinterpret_cast<uint32_t*>(&hi);
                    *reinterpret_cast<uint2*>(dw2 + (size_t)i * 4) = packed;
                }
            }
        }
        const size_t o_db2 = (size_t)C * K, o_db1 = o_db2 + HEAD_CMAX, o_red = o_db1 + K;
        if (tid < HEAD_CMAX) {
            float a = 0.f;
#pragma unroll 8
            for (int g = 0; g < G; ++g) {
                a += __ldcg(scratch + g * slab + o_db2 + tid);
                __stcg(scratch + g * slab + o_db2 + tid, 0.f);
            }
            if (tid < C && db2) db2[tid] = __float2bfloat16(a);
        }
        for (int k = tid; k < K; k += HEAD_THREADS) {
            float a = 0.f;
#pragma unroll 8
            for (int g = 0; g < G; ++g) {
                a += __ldcg(scratch + g * slab + o_db1 + k);
                __stcg(scratch + g * slab + o_db1 + k, 0.f);
            }
            if (db1) db1[k] = __float2bfloat16(a);
        }
        if (tid == 0) {
            float l = 0.f, c = 0.f;
#pragma unroll 8
            for (int g = 0; g < G; ++g) {
                l += __ldcg(scratch + g * slab + o_red);
                c += __ldcg(scratch + g * slab + o_red + 1);
                __stcg(scratch + g * slab + o_red, 0.f);
                __stcg(scratch + g * slab + o_red + 1, 0.f);
            }
            const float mean_loss = l * invB;
            *loss = mean_loss;
            if (loss_host) *loss_host = mean_loss;      // pinned host scalar (UVA): no D2H copy node per step
            if constexpr (TARGET == TFY_HEAD_BINARY) {
                if (stats) { stats[0] += c; stats[1] += (float)B * (float)C; }      // hits over elements
            } else {
                if (stats) { stats[0] += c; stats[1] += (float)B; }
            }
            if constexpr (WEIGHTED) {
                float wc = 0.f, ws = 0.f;
#pragma unroll 8
                for (int g = 0; g < G; ++g) {
                    wc += __ldcg(scratch + g * slab + o_red + 2);
                    ws += __ldcg(scratch + g * slab + o_red + 3);
                    __stcg(scratch + g * slab + o_red + 2, 0.f);
                    __stcg(scratch + g * slab + o_red + 3, 0.f);
                }
                if (stats) { stats[2] += wc; stats[3] += ws; }
            }
            *counter = 0u;
        }
    }
    N_MARK(7);
