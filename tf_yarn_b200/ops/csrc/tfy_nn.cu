// Fused layer kernels of the mini-Keras fast path (sm_90a, bf16 activations, NHWC).
//
// The stock-PyTorch rendition of the MNIST-CNN step launches 53 kernels, most of
// them tiny elementwise / reduction kernels around the cuDNN/cuBLAS calls (bias
// add, clamp, max-pool fwd/bwd, dropout, bias-gradient reductions, the softmax /
// NLL chain, gradient accumulation adds) -- see profiles/launches_r1a_*.csv.
// These kernels fuse each such chain into ONE launch and write parameter
// gradients straight into the flat symmetric gradient buffer that the K4
// reduce-scatter/optimizer/all-gather kernel consumes:
//
//   tfy_conv3x3_c1_fwd        direct 3x3 conv for C_in = 1 + bias + ReLU
//   tfy_conv3x3_c1_wgrad      its weight gradient (reduction over all output pixels)
//   tfy_bias_act_drop_fwd     y = dropout(act(z + bias)) over [rows, C], keep-mask byte
//   tfy_act_drop_bwd_bias     dz = dy * mask (+ dbias[C] reduced and stored as bf16)
//   tfy_bias_relu_pool_drop_fwd   z -> bias + ReLU + 2x2 max-pool + dropout (+1 code byte)
//   tfy_pool_drop_relu_bwd        its backward (+ dbias[C])
//   tfy_softmax_xent          logits(+bias) -> mean loss, dlogits = (softmax - onehot)/B, dbias, #correct
//                             (tfy_softmax_xent_weighted: the same with Keras sample / class weights)
//                             (tfy_softmax_xent_soft: fp32 one-hot / soft targets with Keras label smoothing)
//   tfy_sigmoid_xent          its sigmoid twin (Keras BinaryCrossentropy, binary and multi-label)
//
// Dropout randomness is counter based: hash(seed, layer salt, optimizer step, element) with the
// step read from the device-resident TfyOptHyper, so a replayed CUDA graph draws fresh masks.
#include "tfy_common.cuh"
#include "tfy_head.cuh"

namespace {

__device__ __forceinline__ float bf16_to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

// The batch reductions below (bias and first-layer weight gradients) are summed in a fixed order -- threads of a
// CTA in thread order, CTAs in CTA order, no float atomics -- so that two runs give the same bits.
//
// Cross-CTA column sums: every CTA has stored its C column sums into its own row `blockIdx.x` of `partial`
// (plain stores; `partial` holds gridDim.x * C floats, any content on entry).  The CTA that arrives last on
// `counter` sums the rows in CTA order, stores the bf16 result and re-arms the counter (zero on entry, left zero).
// With C < blockDim.x, P = blockDim.x / C thread groups each sum every P-th row (loads in flight together) and the
// P part sums are added in order; s_tmp: >= blockDim.x floats of shared scratch.
__device__ void tfy_rows_publish(int C, const float* partial, __nv_bfloat16* out, uint32_t* counter, float* s_tmp) {
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const int rows = (int)gridDim.x;
    const int P = C < (int)blockDim.x ? (int)blockDim.x / C : 1;
    if (P > 1) {
        const int c = (int)threadIdx.x % C, part = (int)threadIdx.x / C;
        if (part < P) {
            float a = 0.f;
#pragma unroll 8
            for (int r = part; r < rows; r += P) a += __ldcg(partial + (size_t)r * C + c);
            s_tmp[part * C + c] = a;
        }
        __syncthreads();
        if ((int)threadIdx.x < C) {
            float a = s_tmp[threadIdx.x];
            for (int q = 1; q < P; ++q) a += s_tmp[q * C + threadIdx.x];
            out[threadIdx.x] = __float2bfloat16(a);
        }
    } else {
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            float a = 0.f;
#pragma unroll 8
            for (int r = 0; r < rows; ++r) a += __ldcg(partial + (size_t)r * C + c);
            out[c] = __float2bfloat16(a);
        }
    }
    if (threadIdx.x == 0) *counter = 0;
}

// Column sums of values held 8-per-thread (column group g = (global thread index) % G of G = C/8, fixed by a grid
// stride that is a multiple of G; threads at or beyond `stride` hold nothing): every thread parks its 8 sums in
// s_thr ([blockDim.x][8] floats), column c of this CTA is the sum over the threads of group c/8 in thread order,
// stored into row blockIdx.x of `partial`; then tfy_rows_publish.
__device__ __forceinline__ void tfy_block_colsum_publish(const float (&colacc)[8], int C, size_t stride, float* s_thr,
                                                         float* partial, __nv_bfloat16* out, uint32_t* counter) {
    const int G = C / 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) s_thr[threadIdx.x * 8 + k] = colacc[k];
    __syncthreads();
    const size_t base = (size_t)blockIdx.x * blockDim.x;
    const int live = stride > base ? (int)min((size_t)blockDim.x, stride - base) : 0;     // threads holding sums
    const int g0 = (int)(base % G);                                                          // group of thread 0
    float* row = partial + (size_t)blockIdx.x * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c >> 3, k = c & 7;
        float a = 0.f;
        for (int t = (g - g0 + G) % G; t < live; t += G) a += s_thr[t * 8 + k];
        __stcg(row + c, a);
    }
    tfy_rows_publish(C, partial, out, counter, s_thr);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// conv 3x3, C_in = 1, stride 1, VALID, + bias + ReLU.   x: [B,H,W] (fp32 or bf16), w: [O][9] bf16,
// y: [B,H-2,W-2,O] bf16.  One thread = one output pixel, all O channels: x loads are coalesced across
// the warp, the weights are warp-broadcast reads from shared memory, each thread writes O*2 contiguous
// bytes.
// ---------------------------------------------------------------------------------------------
template <typename XT>
__global__ void __launch_bounds__(256)
tfy_conv3x3_c1_fwd_kernel(const XT* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                          const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int B, int H, int W,
                          int O) {
    tfy_pdl_sync();
    extern __shared__ float s_w[];  // [9][O] + [O] bias
    for (int i = threadIdx.x; i < 9 * O; i += blockDim.x) {
        const int o = i % O, t = i / O;
        s_w[i] = bf16_to_f(w[o * 9 + t]);
    }
    for (int i = threadIdx.x; i < O; i += blockDim.x) s_w[9 * O + i] = bf16_to_f(bias[i]);
    __syncthreads();
    const int OH = H - 2, OW = W - 2;
    const size_t total = (size_t)B * OH * OW;
    for (size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
         pix += (size_t)gridDim.x * blockDim.x) {
        const int ow = pix % OW;
        const size_t r = pix / OW;
        const int oh = r % OH;
        const int b = r / OH;
        const XT* xp = x + ((size_t)b * H + oh) * W + ow;
        float xin[9];
#pragma unroll
        for (int kh = 0; kh < 3; ++kh)
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) xin[kh * 3 + kw] = (float)xp[kh * W + kw];
        __nv_bfloat16* yp = y + pix * O;
        for (int g = 0; g < O; g += 8) {
            float acc[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = s_w[9 * O + g + k];
#pragma unroll
            for (int t = 0; t < 9; ++t)
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = fmaf(xin[t], s_w[t * O + g + k], acc[k]);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = fmaxf(acc[k], 0.f);
            tfy_st16(yp + g, TfyPack<__nv_bfloat16>::pack(acc));
        }
    }
}

// dW[o][t] = sum over (b,oh,ow) x[b,oh+kh,ow+kw] * dz[b,oh,ow,o].
// lane <-> output channel (blocks of 32 channels).  A warp owns whole output rows (b, oh): it loads the
// three input rows it needs ONCE (coalesced, lane = column; W <= 32 fast path) and walks ow with the
// window values coming from warp shuffles -- per pixel one 64-byte dz load, 9 shuffles, 9 FMAs and no
// integer division.  Warps are combined in warp order through one shared row per warp, CTAs through
// tfy_rows_publish.
template <typename XT>
__global__ void __launch_bounds__(256)
tfy_conv3x3_c1_wgrad_kernel(const XT* __restrict__ x, const __nv_bfloat16* __restrict__ dz,
                            float* __restrict__ partial, __nv_bfloat16* __restrict__ dw, uint32_t* counter, int B,
                            int H, int W, int O) {
    extern __shared__ float s_acc[];   // [9*O] CTA sums | [warps][9][32] this channel block's per-warp sums
    const int OH = H - 2, OW = W - 2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    float* s_warp = s_acc + 9 * O;
    const int nrows = B * OH;
    const int gw = blockIdx.x * nwarps + warp, tw = gridDim.x * nwarps;
    for (int o0 = 0; o0 < O; o0 += 32) {
        const int o = o0 + lane;
        const bool o_ok = o < O;
        float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int row = gw; row < nrows; row += tw) {
            const int b = row / OH, oh = row - b * OH;
            const XT* xr = x + ((size_t)b * H + oh) * W;
            const __nv_bfloat16* dzr = dz + (size_t)row * OW * O + o;
            if (W <= 32) {
                const float r0 = lane < W ? (float)xr[lane] : 0.f;
                const float r1 = lane < W ? (float)xr[W + lane] : 0.f;
                const float r2 = lane < W ? (float)xr[2 * W + lane] : 0.f;
#pragma unroll 2
                for (int ow = 0; ow < OW; ++ow) {
                    const float d = o_ok ? bf16_to_f(dzr[(size_t)ow * O]) : 0.f;
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw) {
                        acc[0 + kw] = fmaf(__shfl_sync(0xffffffffu, r0, ow + kw), d, acc[0 + kw]);
                        acc[3 + kw] = fmaf(__shfl_sync(0xffffffffu, r1, ow + kw), d, acc[3 + kw]);
                        acc[6 + kw] = fmaf(__shfl_sync(0xffffffffu, r2, ow + kw), d, acc[6 + kw]);
                    }
                }
            } else {
                for (int ow = 0; ow < OW; ++ow) {
                    const float d = o_ok ? bf16_to_f(dzr[(size_t)ow * O]) : 0.f;
#pragma unroll
                    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                        for (int kw = 0; kw < 3; ++kw)
                            acc[kh * 3 + kw] = fmaf((float)xr[kh * W + ow + kw], d, acc[kh * 3 + kw]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < 9; ++t) s_warp[(warp * 9 + t) * 32 + lane] = acc[t];
        __syncthreads();
        for (int i = threadIdx.x; i < 9 * 32; i += blockDim.x) {       // i = t * 32 + lane of channel o0 + lane
            const int t = i >> 5, o = o0 + (i & 31);
            float a = 0.f;
            for (int w = 0; w < nwarps; ++w) a += s_warp[w * 9 * 32 + i];
            if (o < O) s_acc[o * 9 + t] = a;
        }
        __syncthreads();
    }
    float* row = partial + (size_t)blockIdx.x * 9 * O;
    for (int i = threadIdx.x; i < 9 * O; i += blockDim.x) __stcg(row + i, s_acc[i]);
    tfy_rows_publish(9 * O, partial, dw, counter, s_warp);
}

// ---------------------------------------------------------------------------------------------
// y = dropout(act(z + bias[c])) over a [rows, C] bf16 matrix (C % 8 == 0); y may alias z.
// mask (optional, 1 byte per element): 1 = gradient flows (act'(.) != 0 and kept).
// ---------------------------------------------------------------------------------------------
template <typename ZT>
__global__ void __launch_bounds__(256)
tfy_bias_act_drop_fwd_kernel(ZT* z, const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* y,
                             uint8_t* __restrict__ mask, size_t rows, int C, int relu, float drop_rate, uint32_t seed,
                             const TfyOptHyper* __restrict__ hp) {
    tfy_pdl_sync();
    const int G = C / 8;
    const size_t total = rows * G;
    const uint32_t step = hp ? (uint32_t)hp->step : 0u;
    const float keep_scale = drop_rate > 0.f ? 1.f / (1.f - drop_rate) : 1.f;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % G;
        float v[8], bv[8];
        TfyPack<__nv_bfloat16>::unpack(tfy_ld16(reinterpret_cast<const __nv_bfloat16*>(z) + idx * 8), v);
        if (bias) {
            TfyPack<__nv_bfloat16>::unpack(tfy_ld16(bias + g * 8), bv);
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] += bv[k];
        }
        uint32_t m_lo = 0, m_hi = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            bool on = true;
            if (relu) { on = v[k] > 0.f; v[k] = on ? v[k] : 0.f; }
            if (drop_rate > 0.f) {
                const bool keep = tfy_uniform(seed, step, idx * 8 + k) >= drop_rate;
                v[k] = keep ? v[k] * keep_scale : 0.f;
                on = on && keep;
            }
            if (k < 4) m_lo |= (on ? 1u : 0u) << (8 * k);
            else m_hi |= (on ? 1u : 0u) << (8 * (k - 4));
        }
        tfy_st16(y + idx * 8, TfyPack<__nv_bfloat16>::pack(v));
        if (mask) *reinterpret_cast<uint2*>(mask + idx * 8) = make_uint2(m_lo, m_hi);
    }
}

// Same, from the `splits` fp32 partial-product slabs z32 ([splits][rows][C]) of the split-K GEMM, summed in slab
// order (the same result on every run).  It sits between the GEMM and the head on the step's critical path and moves
// little data, so its time is L2 latency: one thread per 4 elements (one float4 per slab) and every slab's load in
// flight at once.  Element e draws tfy_uniform(seed, step, e), as in the bf16 kernel above.
__global__ void __launch_bounds__(32)
tfy_bias_act_drop_fwd_kernel_slabs(const float* __restrict__ z32, const __nv_bfloat16* __restrict__ bias,
                                   __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ mask, size_t n4, int C,
                                   int relu, float drop_rate, uint32_t seed, const TfyOptHyper* __restrict__ hp,
                                   int splits) {
    tfy_pdl_sync();
    const uint32_t step = hp ? (uint32_t)hp->step : 0u;
    const float keep_scale = drop_rate > 0.f ? 1.f / (1.f - drop_rate) : 1.f;
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += (size_t)gridDim.x * blockDim.x) {
        const size_t e0 = q * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (int s0 = 0; s0 < splits; s0 += 24) {          // up to 24 loads issued before the first add
            float4 a[24];
#pragma unroll
            for (int j = 0; j < 24; ++j)
                if (s0 + j < splits) a[j] = __ldcg(reinterpret_cast<const float4*>(z32) + (size_t)(s0 + j) * n4 + q);
#pragma unroll
            for (int j = 0; j < 24; ++j)
                if (s0 + j < splits) { v[0] += a[j].x; v[1] += a[j].y; v[2] += a[j].z; v[3] += a[j].w; }
        }
        if (bias) {
            const uint2 b = *reinterpret_cast<const uint2*>(bias + e0 % C);
            v[0] += tfy_bf16lo(b.x); v[1] += tfy_bf16hi(b.x); v[2] += tfy_bf16lo(b.y); v[3] += tfy_bf16hi(b.y);
        }
        uint32_t m = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            bool on = true;
            if (relu) { on = v[k] > 0.f; v[k] = on ? v[k] : 0.f; }
            if (drop_rate > 0.f) {
                const bool keep = tfy_uniform(seed, step, e0 + k) >= drop_rate;
                v[k] = keep ? v[k] * keep_scale : 0.f;
                on = on && keep;
            }
            m |= (on ? 1u : 0u) << (8 * k);
        }
        *reinterpret_cast<uint2*>(y + e0) = make_uint2(tfy_pack_bf16x2(v[0], v[1]), tfy_pack_bf16x2(v[2], v[3]));
        if (mask) *reinterpret_cast<uint32_t*>(mask + e0) = m;
    }
}

// dz = dy * gate * scale, where gate comes from `mask` bytes (if given) or from y > 0; dbias[c] = sum_rows dz.
__global__ void __launch_bounds__(256)
tfy_act_drop_bwd_bias_kernel(const __nv_bfloat16* dy, const uint8_t* __restrict__ mask,
                             const __nv_bfloat16* __restrict__ y, __nv_bfloat16* dz, float scale, size_t rows, int C,
                             float* __restrict__ partial, __nv_bfloat16* __restrict__ dbias, uint32_t* counter) {
    tfy_pdl_sync();
    extern __shared__ float s_thr[];  // [blockDim.x][8] per-thread column sums
    const int G = C / 8;
    const size_t total = rows * G;
    // each thread keeps a fixed column group: stride must be a multiple of G
    const size_t stride = ((size_t)gridDim.x * blockDim.x / G) * G;
    float colacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = start < stride;
    if (active) {
        for (size_t idx = start; idx < total; idx += stride) {
            float v[8];
            TfyPack<__nv_bfloat16>::unpack(tfy_ld16(dy + idx * 8), v);
            if (mask) {
                const uint2 m = *reinterpret_cast<const uint2*>(mask + idx * 8);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t bit = (k < 4 ? (m.x >> (8 * k)) : (m.y >> (8 * (k - 4)))) & 1u;
                    v[k] = bit ? v[k] * scale : 0.f;
                }
            } else if (y) {
                float yv[8];
                TfyPack<__nv_bfloat16>::unpack(tfy_ld16(y + idx * 8), yv);
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = yv[k] > 0.f ? v[k] * scale : 0.f;
            }
            if (dz) tfy_st16(dz + idx * 8, TfyPack<__nv_bfloat16>::pack(v));
#pragma unroll
            for (int k = 0; k < 8; ++k) colacc[k] += v[k];
        }
    }
    if (dbias) tfy_block_colsum_publish(colacc, C, stride, s_thr, partial, dbias, counter);
}

// ---------------------------------------------------------------------------------------------
// z [B,H,W,C] (conv output, pre-bias) -> p [B,H/2,W/2,C] = dropout(maxpool2x2(relu(z + bias)))
// code byte per pooled element: bits 0-1 = argmax position (dy*2+dx), bit 2 = gradient flows.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tfy_bias_relu_pool_drop_fwd_kernel(const __nv_bfloat16* __restrict__ z, const __nv_bfloat16* __restrict__ bias,
                                   __nv_bfloat16* __restrict__ p, uint8_t* __restrict__ code, int B, int H, int W,
                                   int C, float drop_rate, uint32_t seed, const TfyOptHyper* __restrict__ hp) {
    const int PH = H / 2, PW = W / 2, G = C / 8;
    const size_t total = (size_t)B * PH * PW * G;
    const uint32_t step = hp ? (uint32_t)hp->step : 0u;
    const float keep_scale = drop_rate > 0.f ? 1.f / (1.f - drop_rate) : 1.f;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % G;
        size_t r = idx / G;
        const int pw = r % PW;
        r /= PW;
        const int ph = r % PH;
        const int b = r / PH;
        float bv[8], best[8];
        int arg[8];
        TfyPack<__nv_bfloat16>::unpack(tfy_ld16(bias + g * 8), bv);
#pragma unroll
        for (int k = 0; k < 8; ++k) { best[k] = -3.0e38f; arg[k] = 0; }
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                float v[8];
                const size_t off = (((size_t)b * H + ph * 2 + dy) * W + pw * 2 + dx) * C + g * 8;
                TfyPack<__nv_bfloat16>::unpack(tfy_ld16(z + off), v);
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (v[k] > best[k]) { best[k] = v[k]; arg[k] = dy * 2 + dx; }
            }
        uint32_t c_lo = 0, c_hi = 0;
        float out[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float v = best[k] + bv[k];
            bool on = v > 0.f;
            v = on ? v : 0.f;
            if (drop_rate > 0.f) {
                const bool keep = tfy_uniform(seed, step, idx * 8 + k) >= drop_rate;
                v = keep ? v * keep_scale : 0.f;
                on = on && keep;
            }
            out[k] = v;
            const uint32_t cb = (uint32_t)arg[k] | (on ? 4u : 0u);
            if (k < 4) c_lo |= cb << (8 * k);
            else c_hi |= cb << (8 * (k - 4));
        }
        tfy_st16(p + idx * 8, TfyPack<__nv_bfloat16>::pack(out));
        *reinterpret_cast<uint2*>(code + idx * 8) = make_uint2(c_lo, c_hi);
    }
}

// dp [B,PH,PW,C] + code -> dz [B,H,W,C] (gradient wrt the conv output), dbias[C] = sum dz.
__global__ void __launch_bounds__(256)
tfy_pool_drop_relu_bwd_kernel(const __nv_bfloat16* __restrict__ dp, const uint8_t* __restrict__ code,
                              __nv_bfloat16* __restrict__ dz, float scale, int B, int H, int W, int C,
                              float* __restrict__ partial, __nv_bfloat16* __restrict__ dbias, uint32_t* counter) {
    tfy_pdl_sync();
    extern __shared__ float s_thr[];  // [blockDim.x][8] per-thread column sums
    const int PH = H / 2, PW = W / 2, G = C / 8;
    const size_t total = (size_t)B * PH * PW * G;
    const size_t stride = ((size_t)gridDim.x * blockDim.x / G) * G;
    const size_t start = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = start < stride;
    const int g = (int)(start % G);
    float colacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
        for (size_t idx = start; idx < total; idx += stride) {
            size_t r = idx / G;
            const int pw = r % PW;
            r /= PW;
            const int ph = r % PH;
            const int b = r / PH;
            float d[8];
            TfyPack<__nv_bfloat16>::unpack(tfy_ld16(dp + idx * 8), d);
            const uint2 cd = *reinterpret_cast<const uint2*>(code + idx * 8);
            int arg[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t cb = (k < 4 ? (cd.x >> (8 * k)) : (cd.y >> (8 * (k - 4)))) & 0xffu;
                d[k] = (cb & 4u) ? d[k] * scale : 0.f;
                arg[k] = cb & 3u;
                colacc[k] += d[k];
            }
#pragma unroll
            for (int pos = 0; pos < 4; ++pos) {
                float o[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = arg[k] == pos ? d[k] : 0.f;
                const size_t off = (((size_t)b * H + ph * 2 + (pos >> 1)) * W + pw * 2 + (pos & 1)) * C + g * 8;
                tfy_st16(dz + off, TfyPack<__nv_bfloat16>::pack(o));
            }
        }
    }
    if (dbias) tfy_block_colsum_publish(colacc, C, stride, s_thr, partial, dbias, counter);
}

// ---------------------------------------------------------------------------------------------
// softmax cross-entropy head.  logits [B,C] bf16 (+ optional bias[C]), labels int64.  Single CTA (B rows strided
// over the threads).  Row r weighs w_r = sample_w[r] * class_w[label_r] (Keras sample_weight / class_weight; a null
// pointer, or a label outside [0, C), counts as 1): loss = sum_r w_r l_r / B (fp32), dlogits = w_r (softmax - onehot)
// / B (bf16), dbias = column sums of dlogits (bf16), stats[0..n_stats) += [hits, B, sum w*hit, sum w] (n_stats 2 or
// 4).  Every block-level sum is taken in a fixed order (warp shuffles, then warps in index order; dbias from one
// partial row per warp), so the result is the same bit for bit on every run.
//
// Target modes of the classifier-head kernels.  SPARSE: int64 class labels.  DENSE (Keras CategoricalCrossentropy):
// fp32 targets y [B, C], one-hot or soft, smoothed as t_c = y_c (1 - ls) + ls / C; with S = sum_c t_c, a row's loss
// is sum_c t_c (lse - v_c) and its dlogits (p_c S - t_c) w_r / B; its class (hit test, class weight) is argmax_c y_c,
// ties to the lowest index.  A one-hot row with ls = 0 has t = onehot and S = 1 exactly, and every expression keeps
// the SPARSE mode's order of operations, so the two modes give the same bits.
// BINARY (Keras BinaryCrossentropy; the fused head and tfy_sigmoid_xent): fp32 targets y [B, C], every logit z one
// element of the row's mean, t = y (1 - ls) + ls / 2, l = max(z, 0) - z t + log1p(exp(-|z|)) (tfy_head.cuh's binary
// element function), a row's loss (1/C) sum_c l_c and its dlogits w_r (sigmoid(z) - t) / (B C).  Its hits are per
// element, (out > 0.5) == (y > 0.5) with out the model's output (sigmoid(z), or z after a linear layer), and stats
// count [hits, B C, sum_r w_r hits_r / C, sum_r w_r]; a row's class (class weight) is round(y) half to even for C = 1,
// argmax_c y_c otherwise, in a class table of max(C, 2) entries.  The mode shares TfyHead's TFY_HEAD_BINARY (the
// canned binary head, whose element functions it computes); the softmax modes are numbered after TfyHead's.
// ---------------------------------------------------------------------------------------------
enum : int { TFY_HEAD_SPARSE = TFY_HEAD_LOGISTIC + 1, TFY_HEAD_DENSE };

template <int TARGET>
__device__ __forceinline__ void
tfy_softmax_xent_body(const __nv_bfloat16* __restrict__ logits, const __nv_bfloat16* __restrict__ bias,
                      const long long* __restrict__ labels, const float* __restrict__ targets, float ls,
                      const float* __restrict__ sample_w, const float* __restrict__ class_w, float* __restrict__ loss,
                      __nv_bfloat16* __restrict__ dlogits, __nv_bfloat16* __restrict__ dbias,
                      float* __restrict__ stats, int n_stats, int B, int C) {
    extern __shared__ float sm[];  // [C] bias | [warps][C] dbias partials | [warps][4] loss, hits, w*hits, w
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s_bias = sm;
    float* s_db = sm + C;
    float* s_red = s_db + (size_t)warps * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_bias[c] = bias ? bf16_to_f(bias[c]) : 0.f;
    for (int i = threadIdx.x; i < warps * C; i += blockDim.x) s_db[i] = 0.f;
    __syncthreads();
    const float invB = 1.f / (float)B;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};        // loss, hits, w*hits, w
    const int rounds = (B + blockDim.x - 1) / blockDim.x;      // same trip count on every warp: shuffles converge
    const float keep = 1.f - ls, add = ls / (float)C;            // DENSE: t = y * keep + add
    for (int it = 0; it < rounds; ++it) {
        const int r = it * blockDim.x + threadIdx.x;
        const bool ok = r < B;
        const __nv_bfloat16* row = logits + (size_t)(ok ? r : 0) * C;
        const float* trow = nullptr;
        int lab = -1;
        float S = 0.f;                                           // DENSE: sum of this row's smoothed targets
        if constexpr (TARGET == TFY_HEAD_SPARSE) {
            lab = ok ? (int)labels[r] : -1;
        } else if (ok) {
            trow = targets + (size_t)r * C;
            float ym = -INFINITY;
            lab = 0;
            for (int c = 0; c < C; ++c) {
                const float y = trow[c];
                if (y > ym) { ym = y; lab = c; }
                S += fmaf(y, keep, add);
            }
        }
        float wr = 0.f;
        if (ok) {
            wr = sample_w ? sample_w[r] : 1.f;
            if (class_w && lab >= 0 && lab < C) wr *= class_w[lab];
        }
        float mx = -3.0e38f;
        int amax = 0;
        for (int c = 0; c < C; ++c) {
            const float v = bf16_to_f(row[c]) + s_bias[c];
            if (v > mx) { mx = v; amax = c; }
        }
        float se = 0.f;
        for (int c = 0; c < C; ++c) se += __expf(bf16_to_f(row[c]) + s_bias[c] - mx);
        const float lse = mx + __logf(se);
        const float inv_se = 1.f / se;
        float lrow = 0.f;                                        // DENSE: sum_c t_c (lse - v_c)
        for (int c = 0; c < C; ++c) {
            const float v = bf16_to_f(row[c]) + s_bias[c];
            float d;
            if constexpr (TARGET == TFY_HEAD_SPARSE) {
                d = (__expf(v - mx) * inv_se - (c == lab ? 1.f : 0.f)) * invB * wr;
            } else {
                // p S - t as one fma of (e, inv_se S): the SPARSE mode's fma(e, inv_se, -onehot) when S = 1
                const float t = ok ? fmaf(trow[c], keep, add) : 0.f;
                d = fmaf(__expf(v - mx), inv_se * S, -t) * invB * wr;
                lrow = fmaf(t, lse - v, lrow);
            }
            if (!ok) d = 0.f;
            if (ok) {
                if constexpr (TARGET == TFY_HEAD_SPARSE) {
                    if (c == lab) acc[0] += wr * (lse - v);
                }
                dlogits[(size_t)r * C + c] = __float2bfloat16(d);
            }
            if (dbias) {
                float t = d;
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
                if (lane == 0) s_db[(size_t)warp * C + c] += t;        // one writer per (warp, class)
            }
        }
        if constexpr (TARGET == TFY_HEAD_DENSE) {
            if (ok) acc[0] += wr * lrow;
        }
        if (ok && amax == lab) { acc[1] += 1.f; acc[2] += wr; }
        acc[3] += wr;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) s_red[warp * 4 + k] = acc[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t[4] = {0.f, 0.f, 0.f, 0.f};
        for (int w = 0; w < warps; ++w)
            for (int k = 0; k < 4; ++k) t[k] += s_red[w * 4 + k];
        *loss = t[0] * invB;
        if (stats) {
            stats[0] += t[1];
            stats[1] += (float)B;
            if (n_stats > 2) { stats[2] += t[2]; stats[3] += t[3]; }
        }
    }
    if (dbias)
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            float a = 0.f;
            for (int w = 0; w < warps; ++w) a += s_db[(size_t)w * C + c];
            dbias[c] = __float2bfloat16(a);
        }
}

__global__ void __launch_bounds__(1024)
tfy_softmax_xent_weighted_kernel(const __nv_bfloat16* __restrict__ logits, const __nv_bfloat16* __restrict__ bias,
                                 const long long* __restrict__ labels, const float* __restrict__ sample_w,
                                 const float* __restrict__ class_w, float* __restrict__ loss,
                                 __nv_bfloat16* __restrict__ dlogits, __nv_bfloat16* __restrict__ dbias,
                                 float* __restrict__ stats, int n_stats, int B, int C) {
    tfy_pdl_sync();
    tfy_softmax_xent_body<TFY_HEAD_SPARSE>(logits, bias, labels, nullptr, 0.f, sample_w, class_w, loss, dlogits, dbias,
                                           stats, n_stats, B, C);
}

// DENSE target mode: targets [B, C] fp32, label smoothing ls
__global__ void __launch_bounds__(1024)
tfy_softmax_xent_soft_kernel(const __nv_bfloat16* __restrict__ logits, const __nv_bfloat16* __restrict__ bias,
                             const float* __restrict__ targets, float ls, const float* __restrict__ sample_w,
                             const float* __restrict__ class_w, float* __restrict__ loss,
                             __nv_bfloat16* __restrict__ dlogits, __nv_bfloat16* __restrict__ dbias,
                             float* __restrict__ stats, int n_stats, int B, int C) {
    tfy_pdl_sync();
    tfy_softmax_xent_body<TFY_HEAD_DENSE>(logits, bias, nullptr, targets, ls, sample_w, class_w, loss, dlogits, dbias,
                                          stats, n_stats, B, C);
}

// BINARY target mode: targets [B, C] fp32, label smoothing ls, sigmoid_out: the model's output is sigmoid(z) (else z).
// The block shape, shared-memory layout and reduction order are tfy_softmax_xent_body's.
__global__ void __launch_bounds__(1024)
tfy_sigmoid_xent_kernel(const __nv_bfloat16* __restrict__ logits, const __nv_bfloat16* __restrict__ bias,
                        const float* __restrict__ targets, float ls, int sigmoid_out,
                        const float* __restrict__ sample_w, const float* __restrict__ class_w, float* __restrict__ loss,
                        __nv_bfloat16* __restrict__ dlogits, __nv_bfloat16* __restrict__ dbias,
                        float* __restrict__ stats, int n_stats, int B, int C) {
    tfy_pdl_sync();
    extern __shared__ float sm[];  // [C] bias | [warps][C] dbias partials | [warps][4] loss, hits, w*hits/C, w
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s_bias = sm;
    float* s_db = sm + C;
    float* s_red = s_db + (size_t)warps * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_bias[c] = bias ? bf16_to_f(bias[c]) : 0.f;
    for (int i = threadIdx.x; i < warps * C; i += blockDim.x) s_db[i] = 0.f;
    __syncthreads();
    const float invB = 1.f / (float)B, invC = 1.f / (float)C;
    const int n_cls = max(C, 2);                                 // class-weight table entries
    float acc[4] = {0.f, 0.f, 0.f, 0.f};        // loss, hits, w*hits/C, w
    const int rounds = (B + blockDim.x - 1) / blockDim.x;      // same trip count on every warp: shuffles converge
    const float keep = 1.f - ls, add = 0.5f * ls;               // t = y * keep + add
    for (int it = 0; it < rounds; ++it) {
        const int r = it * blockDim.x + threadIdx.x;
        const bool ok = r < B;
        const __nv_bfloat16* row = logits + (size_t)(ok ? r : 0) * C;
        const float* trow = targets + (size_t)(ok ? r : 0) * C;
        float wr = 0.f;
        if (ok) {
            int lab = 0;
            if (C == 1) {
                lab = __float2int_rn(trow[0]);
            } else {
                float ym = -INFINITY;
                for (int c = 0; c < C; ++c)
                    if (trow[c] > ym) { ym = trow[c]; lab = c; }
            }
            wr = sample_w ? sample_w[r] : 1.f;
            if (class_w && lab >= 0 && lab < n_cls) wr *= class_w[lab];
        }
        float lrow = 0.f, hrow = 0.f;                            // sum_c l_c, hits of the row
        for (int c = 0; c < C; ++c) {
            float d = 0.f;
            if (ok) {
                const float z = bf16_to_f(row[c]) + s_bias[c];
                const float y = trow[c];
                const float t = fmaf(y, keep, add);
                const float sg = tfy_head_sigmoid(z);
                lrow += tfy_head_binary_loss(z, t);
                hrow += ((sigmoid_out ? sg : z) > 0.5f) == (y > 0.5f) ? 1.f : 0.f;
                d = (sg - t) * (invB * invC) * wr;
                dlogits[(size_t)r * C + c] = __float2bfloat16(d);
            }
            if (dbias) {
                float t = d;
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
                if (lane == 0) s_db[(size_t)warp * C + c] += t;        // one writer per (warp, class)
            }
        }
        if (ok) {
            acc[0] += wr * (lrow * invC);
            acc[1] += hrow;
            acc[2] += wr * (hrow * invC);
            acc[3] += wr;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) s_red[warp * 4 + k] = acc[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t[4] = {0.f, 0.f, 0.f, 0.f};
        for (int w = 0; w < warps; ++w)
            for (int k = 0; k < 4; ++k) t[k] += s_red[w * 4 + k];
        *loss = t[0] * invB;
        if (stats) {
            stats[0] += t[1];
            stats[1] += (float)B * (float)C;
            if (n_stats > 2) { stats[2] += t[2]; stats[3] += t[3]; }
        }
    }
    if (dbias)
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            float a = 0.f;
            for (int w = 0; w < warps; ++w) a += s_db[(size_t)w * C + c];
            dbias[c] = __float2bfloat16(a);
        }
}


// ---------------------------------------------------------------------------------------------
// Classifier head, forward AND backward, in one launch (the whole problem is ~0.5 MFLOP):
//   logits = h W2^T + b2 ; loss = mean CE(softmax(logits), labels) ; dlogits = (p - onehot) / B
//   dW2 = dlogits^T h ; db2 = colsum(dlogits)
//   dh  = (dlogits W2) * gate(mask1) * scale1 ; db1 = colsum(dh)          (the previous Dense layer's
//                                                                          ReLU / dropout gate + bias gradient)
// Replaces a cuBLAS GEMM, the softmax/CE kernel, two more cuBLAS GEMMs and the gate/bias-gradient kernel
// (3.9 + 6.6 + 4.6 + 4.1 + 6.9 us of launches for 128 x 128 x 10).  Intermediates stay in fp32.
// One CTA per 16 rows; every CTA stores its part of the batch reductions (dW2, db2, db1, loss) in its own slab of
// an fp32 scratch buffer and the last CTA to finish sums the slabs in CTA order (no float atomics: the result is
// the same bit for bit on every run), converts and clears them.
// h: [B, K] bf16, W2: [C, K] bf16, b2: [C] bf16, labels: [B] int64, mask1: [B, K] uint8 (bit 0 = gradient
// flows) or null.  K in {128, 256, 512}, C <= 16.
// scratch: one slab [C*K | 16 | K | 4] floats per CTA, zero on entry and on exit; counter: one uint32, same.
// WEIGHTED (Keras sample_weight / class_weight): row r weighs w_r = sample_w[r] * class_w[label_r] (a null table, or a
// label outside [0, C), counts as 1).  Its dlogits row is scaled by w_r, so dW2, db2, dh and db1 follow; the loss is
// sum_r w_r l_r / B, and stats holds 4 floats [hits, B, sum w*hit, sum w].  The two extra sums use the spare floats
// of each CTA's reduction slab and are summed in CTA order like the others.
// TARGET (TFY_HEAD_SPARSE / TFY_HEAD_DENSE, see tfy_softmax_xent_body): the DENSE mode reads targets [B, C] fp32 and
// the label smoothing ls; lane c of a row's 16 loads y_rc, and two more 16-lane shuffle reductions give the row's
// class (argmax_c y_rc) and S.  Only the s_dl tile and the per-row loss / hit differ: everything after them is shared.
// ---------------------------------------------------------------------------------------------
// debug: per-CTA event timeline of the head kernel (16 slots of SM-clock deltas per CTA), see tfy_nn_set_timeline
__device__ long long* n_timeline = nullptr;
#define N_MARK(k)                                                                    \
    do {                                                                             \
        if (n_tl && threadIdx.x == 0) n_tl[(size_t)blockIdx.x * 16 + (k)] = clock64() - n_t0; \
    } while (0)

constexpr int HEAD_THREADS = 256, HEAD_CMAX = 16, HEAD_ROWS = 16, HEAD_WARPS = HEAD_THREADS / 32;


template <int K, bool WEIGHTED>
__global__ void __launch_bounds__(HEAD_THREADS)
tfy_dense_head_fused_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w2,
                            const __nv_bfloat16* __restrict__ b2, const long long* __restrict__ labels,
                            const uint8_t* __restrict__ mask1, float scale1, float* __restrict__ loss,
                            float* __restrict__ loss_host, float* __restrict__ stats,
                            __nv_bfloat16* __restrict__ dw2,
                            __nv_bfloat16* __restrict__ db2, __nv_bfloat16* __restrict__ dh,
                            __nv_bfloat16* __restrict__ db1, float* __restrict__ scratch,
                            uint32_t* __restrict__ counter, int B, int C,
                            const float* __restrict__ sample_w, const float* __restrict__ class_w) {
    // (the weights come last: the parameter offsets of the unweighted instantiations do not move)
    // K is a template parameter: every loop that waits on global memory has a constant trip count and is
    // fully unrolled, so its loads are issued back to back (the first version had ~18 serialised L2 round
    // trips in five-iteration loops: 15 us for 0.5 MFLOP).
    tfy_pdl_sync();
    constexpr int TARGET = TFY_HEAD_SPARSE;
    [[maybe_unused]] const float* const targets = nullptr;
    [[maybe_unused]] const float ls = 0.f;
    [[maybe_unused]] const int sigmoid_out = 0;
#include "tfy_dense_head_body.cuh"
}

// DENSE target mode: targets [B, C] fp32, label smoothing ls
template <int K, bool WEIGHTED>
__global__ void __launch_bounds__(HEAD_THREADS)
tfy_dense_head_fused_soft_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w2,
                                 const __nv_bfloat16* __restrict__ b2, const float* __restrict__ targets, float ls,
                                 const uint8_t* __restrict__ mask1, float scale1, float* __restrict__ loss,
                                 float* __restrict__ loss_host, float* __restrict__ stats,
                                 __nv_bfloat16* __restrict__ dw2,
                                 __nv_bfloat16* __restrict__ db2, __nv_bfloat16* __restrict__ dh,
                                 __nv_bfloat16* __restrict__ db1, float* __restrict__ scratch,
                                 uint32_t* __restrict__ counter, int B, int C,
                                 const float* __restrict__ sample_w, const float* __restrict__ class_w) {
    tfy_pdl_sync();
    constexpr int TARGET = TFY_HEAD_DENSE;
    [[maybe_unused]] const long long* const labels = nullptr;
    [[maybe_unused]] const int sigmoid_out = 0;
#include "tfy_dense_head_body.cuh"
}

// BINARY target mode: targets [B, C] fp32, label smoothing ls, sigmoid_out: the model's output is sigmoid(z) (else z)
template <int K, bool WEIGHTED>
__global__ void __launch_bounds__(HEAD_THREADS)
tfy_dense_head_fused_binary_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w2,
                                   const __nv_bfloat16* __restrict__ b2, const float* __restrict__ targets, float ls,
                                   int sigmoid_out, const uint8_t* __restrict__ mask1, float scale1,
                                   float* __restrict__ loss, float* __restrict__ loss_host, float* __restrict__ stats,
                                   __nv_bfloat16* __restrict__ dw2,
                                   __nv_bfloat16* __restrict__ db2, __nv_bfloat16* __restrict__ dh,
                                   __nv_bfloat16* __restrict__ db1, float* __restrict__ scratch,
                                   uint32_t* __restrict__ counter, int B, int C,
                                   const float* __restrict__ sample_w, const float* __restrict__ class_w) {
    tfy_pdl_sync();
    constexpr int TARGET = TFY_HEAD_BINARY;
    [[maybe_unused]] const long long* const labels = nullptr;
#include "tfy_dense_head_body.cuh"
}

// ---------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------
static inline int tfy_grid_for(size_t items, int block, int cap) {
    size_t g = (items + block - 1) / block;
    if (g < 1) g = 1;
    if (g > (size_t)cap) g = cap;
    return (int)g;
}

extern "C" {

// The kernels with a bias / weight-gradient reduction (tfy_conv3x3_c1_wgrad, tfy_act_drop_bwd_bias,
// tfy_pool_drop_relu_bwd) take `partial`: one row of their reduction width per CTA, for at most
// TFY_PARTIAL_BLOCKS CTAs (the launchers refuse a larger grid with -3), and `counter`: one zero-initialised u32,
// left zero.
#define TFY_PARTIAL_BLOCKS 592
size_t tfy_nn_max_partial_blocks() { return TFY_PARTIAL_BLOCKS; }

int tfy_conv3x3_c1_fwd(const void* x, int x_is_f32, const void* w, const void* bias, void* y, int B, int H, int W,
                       int O, cudaStream_t s) {
    if (O % 8) return -2;
    const size_t total = (size_t)B * (H - 2) * (W - 2);
    const int grid = tfy_grid_for(total, 256, TFY_NUM_SMS * 8);
    const size_t smem = (size_t)(10 * O) * sizeof(float);
    if (x_is_f32)
        tfy_launch_pdl((tfy_conv3x3_c1_fwd_kernel<float>), dim3(grid), dim3(256), smem, s, (const float*)x, (const __nv_bfloat16*)w,
                                                                  (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, B, H,
                                                                  W, O);
    else
        tfy_launch_pdl((tfy_conv3x3_c1_fwd_kernel<__nv_bfloat16>), dim3(grid), dim3(256), smem, s, 
            (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, B, H, W, O);
    return (int)cudaGetLastError();
}

int tfy_conv3x3_c1_wgrad(const void* x, int x_is_f32, const void* dz, float* partial, void* dw, uint32_t* counter,
                         int B, int H, int W, int O, cudaStream_t s) {
    if (O < 1 || B < 1 || H < 3 || W < 3) return -2;
    const int grid = 296, block = 256;
    static_assert(296 <= TFY_PARTIAL_BLOCKS, "one partial row per CTA");
    const size_t smem = ((size_t)9 * O + (size_t)(block / 32) * 9 * 32) * sizeof(float);
    if (smem > 48 * 1024) return -2;
    if (x_is_f32)
        tfy_conv3x3_c1_wgrad_kernel<float><<<grid, block, smem, s>>>((const float*)x, (const __nv_bfloat16*)dz, partial,
                                                                    (__nv_bfloat16*)dw, counter, B, H, W, O);
    else
        tfy_conv3x3_c1_wgrad_kernel<__nv_bfloat16><<<grid, block, smem, s>>>(
            (const __nv_bfloat16*)x, (const __nv_bfloat16*)dz, partial, (__nv_bfloat16*)dw, counter, B, H, W, O);
    return (int)cudaGetLastError();
}

int tfy_bias_act_drop_fwd(const void* z, const void* bias, void* y, void* mask, size_t rows, int C, int relu,
                          float drop_rate, uint32_t seed, const TfyOptHyper* hp, cudaStream_t s) {
    if (C % 8) return -2;
    const int grid = tfy_grid_for(rows * (C / 8), 256, TFY_NUM_SMS * 8);
    tfy_launch_pdl((tfy_bias_act_drop_fwd_kernel<__nv_bfloat16>), dim3(grid), dim3(256), 0, s, (__nv_bfloat16*)z, (const __nv_bfloat16*)bias,
                                                                     (__nv_bfloat16*)y, (uint8_t*)mask, rows, C, relu,
                                                                     drop_rate, seed, hp);
    return (int)cudaGetLastError();
}

// same, summing the `splits` fp32 split-K slabs z32 [splits][rows][C] of tfy_gemm_bf16 in slab order
int tfy_bias_act_drop_fwd_f32(void* z32, const void* bias, void* y, void* mask, size_t rows, int C, int relu,
                              float drop_rate, uint32_t seed, const TfyOptHyper* hp, int splits, cudaStream_t s) {
    if (C % 8 || splits < 1) return -2;
    // one warp per block: every thread reads `splits` slabs, so the reads are spread over as many SMs as possible
    const size_t n4 = rows * (size_t)(C / 4);
    const int grid = tfy_grid_for(n4, 32, TFY_NUM_SMS * 16);
    tfy_launch_pdl(tfy_bias_act_drop_fwd_kernel_slabs, dim3(grid), dim3(32), 0, s, (const float*)z32,
                   (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, (uint8_t*)mask, n4, C, relu, drop_rate, seed, hp,
                   splits);
    return (int)cudaGetLastError();
}

int tfy_act_drop_bwd_bias(const void* dy, const void* mask, const void* y, void* dz, float scale, size_t rows, int C,
                          float* partial, void* dbias, uint32_t* counter, cudaStream_t s) {
    if (C % 8) return -2;
    int grid = tfy_grid_for(rows * (C / 8), 256, TFY_PARTIAL_BLOCKS);
    // the kernel needs gridDim*blockDim >= C/8 so that every column group has a thread
    if ((size_t)grid * 256 < (size_t)(C / 8)) grid = (C / 8 + 255) / 256;
    if (dbias && grid > TFY_PARTIAL_BLOCKS) return -3;
    tfy_launch_pdl((tfy_act_drop_bwd_bias_kernel), dim3(grid), dim3(256), 256 * 8 * sizeof(float), s, 
        (const __nv_bfloat16*)dy, (const uint8_t*)mask, (const __nv_bfloat16*)y, (__nv_bfloat16*)dz, scale, rows, C,
        partial, (__nv_bfloat16*)dbias, counter);
    return (int)cudaGetLastError();
}

int tfy_bias_relu_pool_drop_fwd(const void* z, const void* bias, void* p, void* code, int B, int H, int W, int C,
                                float drop_rate, uint32_t seed, const TfyOptHyper* hp, cudaStream_t s) {
    if (C % 8 || H % 2 || W % 2) return -2;
    const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 8);
    const int grid = tfy_grid_for(total, 256, TFY_NUM_SMS * 8);
    tfy_bias_relu_pool_drop_fwd_kernel<<<grid, 256, 0, s>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)bias,
                                                            (__nv_bfloat16*)p, (uint8_t*)code, B, H, W, C, drop_rate,
                                                            seed, hp);
    return (int)cudaGetLastError();
}

int tfy_pool_drop_relu_bwd(const void* dp, const void* code, void* dz, float scale, int B, int H, int W, int C,
                           float* partial, void* dbias, uint32_t* counter, cudaStream_t s) {
    if (C % 8 || H % 2 || W % 2) return -2;
    const size_t total = (size_t)B * (H / 2) * (W / 2) * (C / 8);
    const int grid = tfy_grid_for(total, 256, TFY_PARTIAL_BLOCKS);
    if ((size_t)grid * 256 < (size_t)(C / 8)) return -3;      // every column group needs a thread
    tfy_launch_pdl((tfy_pool_drop_relu_bwd_kernel), dim3(grid), dim3(256), 256 * 8 * sizeof(float), s, 
        (const __nv_bfloat16*)dp, (const uint8_t*)code, (__nv_bfloat16*)dz, scale, B, H, W, C, partial,
        (__nv_bfloat16*)dbias, counter);
    return (int)cudaGetLastError();
}

// Block of the single-CTA cross-entropy kernels (one row per thread, at most 32 warps) and its shared memory: the
// bias, one partial row of dbias per warp and 4 sums per warp.  False when C is too wide for that (C > 9000 or so).
static bool tfy_xent_block(int B, int C, int* warps, size_t* smem) {
    if (B < 1 || C < 1) return false;
    const int max_warps = (int)((48 * 1024 / sizeof(float) - (size_t)C) / ((size_t)C + 4));
    if ((size_t)C >= 48 * 1024 / sizeof(float) || max_warps < 1) return false;
    int w = (B + 31) / 32;
    if (w > 32) w = 32;
    if (w > max_warps) w = max_warps;
    *warps = w;
    *smem = ((size_t)C + (size_t)w * (C + 4)) * sizeof(float);
    return true;
}

// labels (int64, SPARSE mode) or targets (fp32 [B, C], DENSE mode with label smoothing ls): exactly one is non-null
static int tfy_softmax_xent_launch(const void* logits, const void* bias, const void* labels, const float* targets,
                                   float ls, const float* sample_w, const float* class_w, float* loss, void* dlogits,
                                   void* dbias, float* stats, int n_stats, int B, int C, cudaStream_t s) {
    int warps;
    size_t smem;
    if (!tfy_xent_block(B, C, &warps, &smem)) return -2;
    if (targets)
        tfy_launch_pdl((tfy_softmax_xent_soft_kernel), dim3(1), dim3(warps * 32), smem, s,
                       (const __nv_bfloat16*)logits, (const __nv_bfloat16*)bias, targets, ls, sample_w, class_w, loss,
                       (__nv_bfloat16*)dlogits, (__nv_bfloat16*)dbias, stats, n_stats, B, C);
    else
        tfy_launch_pdl((tfy_softmax_xent_weighted_kernel), dim3(1), dim3(warps * 32), smem, s,
                       (const __nv_bfloat16*)logits, (const __nv_bfloat16*)bias, (const long long*)labels, sample_w,
                       class_w, loss, (__nv_bfloat16*)dlogits, (__nv_bfloat16*)dbias, stats, n_stats, B, C);
    return (int)cudaGetLastError();
}

// Keras label smoothing: a finite ls in [0, 1]
static inline bool tfy_valid_smoothing(float ls) { return ls >= 0.f && ls <= 1.f; }

// unweighted head (every weight 1), stats null or 2 floats [hits, B]; returns -2 when C is too wide for one partial
// row of dbias per warp (C > 9000 or so)
int tfy_softmax_xent(const void* logits, const void* bias, const void* labels, float* loss, void* dlogits,
                     void* dbias, float* stats, int B, int C, cudaStream_t s) {
    return tfy_softmax_xent_launch(logits, bias, labels, nullptr, 0.f, nullptr, nullptr, loss, dlogits, dbias, stats, 2,
                                   B, C, s);
}

// weighted variant: sample_w [B] and class_w [C] fp32 (either may be null), stats null or 4 floats
// [hits, B, sum w*hit, sum w]; same return codes
int tfy_softmax_xent_weighted(const void* logits, const void* bias, const void* labels, const float* sample_w,
                              const float* class_w, float* loss, void* dlogits, void* dbias, float* stats, int B, int C,
                              cudaStream_t s) {
    return tfy_softmax_xent_launch(logits, bias, labels, nullptr, 0.f, sample_w, class_w, loss, dlogits, dbias, stats, 4,
                                   B, C, s);
}

// dense-target variant (Keras CategoricalCrossentropy): targets [B, C] fp32, one-hot or soft, label smoothing ls in
// [0, 1]; sample_w and class_w as above (either may be null; the class of a row is argmax_c targets[r][c]).  stats
// null, or 2 floats [hits, B] when both weight pointers are null, else 4.  -2 also when ls is outside [0, 1] or
// B * C exceeds INT_MAX.
int tfy_softmax_xent_soft(const void* logits, const void* bias, const float* targets, float ls, const float* sample_w,
                          const float* class_w, float* loss, void* dlogits, void* dbias, float* stats, int B, int C,
                          cudaStream_t s) {
    if (!targets || !tfy_valid_smoothing(ls) || (long long)B * C > INT_MAX) return -2;
    return tfy_softmax_xent_launch(logits, bias, nullptr, targets, ls, sample_w, class_w, loss, dlogits, dbias, stats,
                                   (sample_w || class_w) ? 4 : 2, B, C, s);
}

// sigmoid twin of tfy_softmax_xent_soft (Keras BinaryCrossentropy, binary C = 1 or multi-label C > 1): targets [B, C]
// fp32, label smoothing ls in [0, 1], sigmoid_out non-zero when the model's output is sigmoid(z) (a sigmoid layer)
// rather than z (hit test only); sample_w [B] and class_w [max(C, 2)] fp32, either may be null (the class of a row is
// round(y) for C = 1, argmax_c y_c otherwise).  loss = sum_r w_r (1/C) sum_c l_rc / B, dlogits [B, C] and dbias [C]
// bf16, stats null or [hits, B C] (+ [sum w hits / C, sum w] when a weight pointer is non-null).  Same return codes
// as tfy_softmax_xent_soft.
int tfy_sigmoid_xent(const void* logits, const void* bias, const float* targets, float ls, int sigmoid_out,
                     const float* sample_w, const float* class_w, float* loss, void* dlogits, void* dbias,
                     float* stats, int B, int C, cudaStream_t s) {
    int warps;
    size_t smem;
    if (!targets || !tfy_valid_smoothing(ls) || (long long)B * C > INT_MAX) return -2;
    if (!tfy_xent_block(B, C, &warps, &smem)) return -2;
    tfy_launch_pdl((tfy_sigmoid_xent_kernel), dim3(1), dim3(warps * 32), smem, s, (const __nv_bfloat16*)logits,
                   (const __nv_bfloat16*)bias, targets, ls, sigmoid_out ? 1 : 0, sample_w, class_w, loss,
                   (__nv_bfloat16*)dlogits, (__nv_bfloat16*)dbias, stats, (sample_w || class_w) ? 4 : 2, B, C);
    return (int)cudaGetLastError();
}

// thin cudaMemcpyAsync wrapper: the input pipeline issues its per-step copies through ctypes (about 1 us per call
// instead of ~10 us for Tensor.copy_ under a stream context manager)
int tfy_memcpy_async(void* dst, const void* src, size_t bytes, cudaStream_t s) {
    return (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s);
}

int tfy_nn_set_timeline(long long* buf) { return (int)cudaMemcpyToSymbol(n_timeline, &buf, sizeof(buf)); }

// fused classifier head (forward + backward); returns -2 when the shape is outside the kernel's envelope, -3 when h,
// w2 or scratch is not 16-byte aligned or dw2 not 8-byte aligned.
// scratch: tfy_dense_head_scratch_elems(K, C, B) floats and counter: one uint32, zero on entry (left zero).
// loss_host: optional second destination of the loss, e.g. a pinned host scalar (device-accessible under UVA).
size_t tfy_dense_head_scratch_elems(int K, int C, int B) {
    return (size_t)((B + HEAD_ROWS - 1) / HEAD_ROWS) * ((size_t)C * K + HEAD_CMAX + K + 4);
}

}  // extern "C"

// TARGET: TFY_HEAD_SPARSE reads `labels` (int64), TFY_HEAD_DENSE reads `targets` (fp32 [B, C]) and `ls`,
// TFY_HEAD_BINARY also `sigmoid_out`
template <bool WEIGHTED, int TARGET>
static int tfy_dense_head_launch(const void* h, const void* w2, const void* b2, const void* labels,
                                 const float* targets, float ls, int sigmoid_out, const void* mask1,
                                 float scale1, float* loss, float* loss_host, float* stats, void* dw2, void* db2,
                                 void* dh, void* db1, float* scratch, uint32_t* counter, int B, int K, int C,
                                 const float* sample_w, const float* class_w, cudaStream_t s) {
    if (!(K == 128 || K == 256 || K == 512) || C < 1 || C > HEAD_CMAX || B < 1) return -2;
    // h, W2 and the scratch slabs are read 16 bytes at a time, dW2 written 8 bytes at a time
    if ((((uintptr_t)h | (uintptr_t)w2 | (uintptr_t)scratch) & 15) || ((uintptr_t)dw2 & 7)) return -3;
    constexpr int NRED = WEIGHTED ? 4 : 2;
    const size_t smem = (size_t)HEAD_ROWS * (K + 8) * 2 +
                        ((size_t)HEAD_CMAX * K + HEAD_ROWS * HEAD_CMAX + HEAD_CMAX + NRED * HEAD_WARPS + (K > 256 ? K : 256)) * 4;
    const int grid = (B + HEAD_ROWS - 1) / HEAD_ROWS;
#define TFY_HEAD_SMEM(KERNEL)                                                                                          \
    do {                                                                                                               \
        static bool configured = false;                                                                                \
        if (smem > 48 * 1024 && !configured) {                                                                         \
            if (cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024) != cudaSuccess)   \
                return -5;                                                                                             \
            configured = true;                                                                                         \
        }                                                                                                              \
    } while (0)
#define TFY_HEAD(KK)                                                                                                   \
    do {                                                                                                               \
        if constexpr (TARGET == TFY_HEAD_SPARSE) {                                                                     \
            TFY_HEAD_SMEM((tfy_dense_head_fused_kernel<KK, WEIGHTED>));                                                \
            tfy_launch_pdl((tfy_dense_head_fused_kernel<KK, WEIGHTED>), dim3(grid), dim3(HEAD_THREADS), smem, s,       \
                           (const __nv_bfloat16*)h, (const __nv_bfloat16*)w2, (const __nv_bfloat16*)b2,                \
                           (const long long*)labels, (const uint8_t*)mask1, scale1, loss, loss_host, stats,            \
                           (__nv_bfloat16*)dw2, (__nv_bfloat16*)db2, (__nv_bfloat16*)dh, (__nv_bfloat16*)db1, scratch, \
                           counter, B, C, sample_w, class_w);                                                          \
        } else if constexpr (TARGET == TFY_HEAD_BINARY) {                                                              \
            TFY_HEAD_SMEM((tfy_dense_head_fused_binary_kernel<KK, WEIGHTED>));                                         \
            tfy_launch_pdl((tfy_dense_head_fused_binary_kernel<KK, WEIGHTED>), dim3(grid), dim3(HEAD_THREADS), smem,   \
                           s, (const __nv_bfloat16*)h, (const __nv_bfloat16*)w2, (const __nv_bfloat16*)b2, targets,    \
                           ls, sigmoid_out, (const uint8_t*)mask1, scale1, loss, loss_host, stats,                     \
                           (__nv_bfloat16*)dw2, (__nv_bfloat16*)db2, (__nv_bfloat16*)dh, (__nv_bfloat16*)db1, scratch, \
                           counter, B, C, sample_w, class_w);                                                          \
        } else {                                                                                                       \
            TFY_HEAD_SMEM((tfy_dense_head_fused_soft_kernel<KK, WEIGHTED>));                                           \
            tfy_launch_pdl((tfy_dense_head_fused_soft_kernel<KK, WEIGHTED>), dim3(grid), dim3(HEAD_THREADS), smem, s,  \
                           (const __nv_bfloat16*)h, (const __nv_bfloat16*)w2, (const __nv_bfloat16*)b2, targets, ls,   \
                           (const uint8_t*)mask1, scale1, loss, loss_host, stats, (__nv_bfloat16*)dw2,                 \
                           (__nv_bfloat16*)db2, (__nv_bfloat16*)dh, (__nv_bfloat16*)db1, scratch, counter, B, C,       \
                           sample_w, class_w);                                                                         \
        }                                                                                                              \
    } while (0)
    if (K == 128) TFY_HEAD(128);
    else if (K == 256) TFY_HEAD(256);
    else TFY_HEAD(512);
#undef TFY_HEAD
#undef TFY_HEAD_SMEM
    return (int)cudaGetLastError();
}

extern "C" {

int tfy_dense_head_fused(const void* h, const void* w2, const void* b2, const void* labels, const void* mask1,
                         float scale1, float* loss, float* loss_host, float* stats, void* dw2, void* db2, void* dh,
                         void* db1,
                         float* scratch, uint32_t* counter, int B, int K, int C, cudaStream_t s) {
    return tfy_dense_head_launch<false, TFY_HEAD_SPARSE>(h, w2, b2, labels, nullptr, 0.f, 0, mask1, scale1, loss,
                                                         loss_host, stats, dw2, db2, dh, db1, scratch, counter, B, K,
                                                         C, nullptr, nullptr, s);
}

// weighted variant: sample_w [B] and class_w [C] fp32 (either may be null), stats null or 4 floats
// [hits, B, sum w*hit, sum w]; same envelope, scratch size and return codes as tfy_dense_head_fused
int tfy_dense_head_fused_weighted(const void* h, const void* w2, const void* b2, const void* labels, const void* mask1,
                                  float scale1, float* loss, float* loss_host, float* stats, void* dw2, void* db2,
                                  void* dh, void* db1, float* scratch, uint32_t* counter, int B, int K, int C,
                                  const float* sample_w, const float* class_w, cudaStream_t s) {
    return tfy_dense_head_launch<true, TFY_HEAD_SPARSE>(h, w2, b2, labels, nullptr, 0.f, 0, mask1, scale1, loss,
                                                        loss_host, stats, dw2, db2, dh, db1, scratch, counter, B, K, C,
                                                        sample_w, class_w, s);
}

// dense-target variant (Keras CategoricalCrossentropy): targets [B, C] fp32, one-hot or soft, label smoothing ls in
// [0, 1]; sample_w [B] and class_w [C] fp32, either may be null (the class of a row is argmax_c targets[r][c]).  The
// unweighted kernel runs when both are null (stats null or 2 floats [hits, B]), the weighted one otherwise (stats
// null or 4 floats).  Same envelope, scratch size and return codes as tfy_dense_head_fused; -2 also when targets is
// null, ls is outside [0, 1] or B * C exceeds INT_MAX.
int tfy_dense_head_fused_soft(const void* h, const void* w2, const void* b2, const float* targets, float ls,
                              const void* mask1, float scale1, float* loss, float* loss_host, float* stats, void* dw2,
                              void* db2, void* dh, void* db1, float* scratch, uint32_t* counter, int B, int K, int C,
                              const float* sample_w, const float* class_w, cudaStream_t s) {
    if (!targets || !tfy_valid_smoothing(ls) || (long long)B * C > INT_MAX) return -2;
    if (sample_w || class_w)
        return tfy_dense_head_launch<true, TFY_HEAD_DENSE>(h, w2, b2, nullptr, targets, ls, 0, mask1, scale1, loss,
                                                           loss_host, stats, dw2, db2, dh, db1, scratch, counter, B, K,
                                                           C, sample_w, class_w, s);
    return tfy_dense_head_launch<false, TFY_HEAD_DENSE>(h, w2, b2, nullptr, targets, ls, 0, mask1, scale1, loss,
                                                        loss_host, stats, dw2, db2, dh, db1, scratch, counter, B, K, C,
                                                        nullptr, nullptr, s);
}

// sigmoid variant (Keras BinaryCrossentropy, binary C = 1 or multi-label C > 1): targets [B, C] fp32, label smoothing
// ls in [0, 1], sigmoid_out non-zero when the model's output is sigmoid(z) (a sigmoid layer) rather than z (hit test
// only: the loss is computed from z either way); sample_w [B] and class_w [max(C, 2)] fp32, either may be null (the
// class of a row is round(y) for C = 1, argmax_c y_c otherwise).  stats null or [hits, B C] (+ [sum w hits / C,
// sum w] when a weight pointer is non-null).  Same envelope, scratch size and return codes as
// tfy_dense_head_fused_soft.
int tfy_dense_head_fused_binary(const void* h, const void* w2, const void* b2, const float* targets, float ls,
                                int sigmoid_out, const void* mask1, float scale1, float* loss, float* loss_host,
                                float* stats, void* dw2, void* db2, void* dh, void* db1, float* scratch,
                                uint32_t* counter, int B, int K, int C, const float* sample_w, const float* class_w,
                                cudaStream_t s) {
    if (!targets || !tfy_valid_smoothing(ls) || (long long)B * C > INT_MAX) return -2;
    sigmoid_out = sigmoid_out ? 1 : 0;
    if (sample_w || class_w)
        return tfy_dense_head_launch<true, TFY_HEAD_BINARY>(h, w2, b2, nullptr, targets, ls, sigmoid_out, mask1,
                                                            scale1, loss, loss_host, stats, dw2, db2, dh, db1, scratch,
                                                            counter, B, K, C, sample_w, class_w, s);
    return tfy_dense_head_launch<false, TFY_HEAD_BINARY>(h, w2, b2, nullptr, targets, ls, sigmoid_out, mask1, scale1,
                                                         loss, loss_host, stats, dw2, db2, dh, db1, scratch, counter, B,
                                                         K, C, nullptr, nullptr, s);
}

}  // extern "C"
