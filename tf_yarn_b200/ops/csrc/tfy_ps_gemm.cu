// K5, the parameter-server PULL fused with the GEMM that consumes it (sm_90a).
//
// First deep layer of a wide-and-deep model on the parameter-server path:
//     y[b, :] = concat_t( table_t[ids[t, b], :] ) ++ numeric[b, :]   .   W^T  + bias
// The reference's stack does this as T sparse RecvTensor pulls (one per embedding table), a concat and a MatMul
// against a weight that was itself pulled from another ps task (reference: tf_yarn/tensorflow/cluster.py:41-67).
// Here ONE kernel does it, and nothing it reads is ever copied to the worker first:
//   * A operand: producer warps GATHER the embedding rows of the batch straight from the ps ranks' HBM over NVLink
//     (16-byte peer loads of the fp32 master rows), convert them to bf16 and write them into the 128-byte-swizzled
//     shared-memory tile the tensor core reads -- the "embedding_bag" of a one-hot column is the operand producer
//     of the GEMM;
//   * B operand: the layer's weights stay on THEIR ps rank; TMA streams the bf16 shadow (row pitch padded to 8
//     elements) tile by tile into shared memory;
//   * a warpgroup runs wgmma M64 N64 K16 on the eight 64 x 64 pieces of the 128 x 256 tile; each piece's
//     chunk product is added into an fp32 accumulator kept in shared memory (in fragment order, so every thread
//     reads and writes only its own words -- the whole tile would not fit the warpgroup's registers next to the
//     producers'); the epilogue adds the bias and stores bf16.
// The gathered activations are also written out once (bf16, [B, Kp]) because the backward needs them
// (dW = dy^T x, tfy_dense_bwd).  K chunk c < T is table c (embedding dim 64); chunk T holds the numeric features.
// warps 0-15: A-tile producers (4 threads per row, 3 chunks in flight each: a gather is a dependent id -> row round
// trip to (remote) HBM per chunk, so the K loop is only as fast as the number of rows in flight)
// warps 16-19: wgmma + epilogue   warp 20: TMA (B tiles)
#include "tfy_common.cuh"
#include "tfy_tma.cuh"
#include "tfy_wgmma.cuh"

namespace {

constexpr int PG_BM = 128, PG_BN = 256, PG_BK = 64, PG_STAGES = 2;
constexpr int PG_A_BYTES = PG_BM * PG_BK * 2, PG_B_BYTES = PG_BN * PG_BK * 2, PG_STAGE_BYTES = PG_A_BYTES + PG_B_BYTES;
constexpr int PG_PROD_WARPS = 16, PG_PROD_THREADS = PG_PROD_WARPS * 32;   // 4 threads per A-tile row
constexpr int PG_DEPTH = 3;                                                  // gathered chunks in flight per thread
constexpr int PG_MMA_WARP = PG_PROD_WARPS, PG_TMA_WARP = PG_PROD_WARPS + 4;
constexpr int PG_THREADS = (PG_PROD_WARPS + 5) * 32;                         // 672
constexpr int PG_ACC_BYTES = PG_BM * PG_BN * 4;                              // [8 pieces][32 values][128 threads]
constexpr size_t PG_SMEM = 1024 + (size_t)PG_STAGES * PG_STAGE_BYTES + PG_ACC_BYTES + 512;

}  // namespace

// tables: device array of T peer pointers to fp32 [V, 64] embedding tables; ids: int64 [T, B]; numeric: fp32 [B, n_num]
// (n_num <= 64); map_w: bf16 shadow [N, Kp] of the weights (peer address allowed); xbuf: bf16 [B, Kp] (written);
// y: bf16 [B, N] = x . W^T + bias.
__global__ void __launch_bounds__(PG_THREADS, 1)
tfy_ps_gather_gemm_kernel(const __grid_constant__ CUtensorMap map_w, const uint64_t* __restrict__ tables,
                          const long long* __restrict__ ids, const float* __restrict__ numeric,
                          const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ xbuf,
                          __nv_bfloat16* __restrict__ y, int B, int N, int T, int n_num, int Kp, long long V) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = tfy_align1024(smem_raw);
    uint8_t* ring = smem;
    float* acc_s = reinterpret_cast<float*>(ring + (size_t)PG_STAGES * PG_STAGE_BYTES);
    uint64_t* full_a = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_s) + PG_ACC_BYTES);
    uint64_t* full_b = full_a + PG_STAGES;
    uint64_t* empty = full_b + PG_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b0 = blockIdx.x * PG_BM, n0 = blockIdx.y * PG_BN;
    const int n_chunks = T + (n_num > 0 ? 1 : 0);
    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_w);
        for (int s = 0; s < PG_STAGES; ++s) {
            tfy_mbar_init(&full_a[s], PG_PROD_THREADS);
            tfy_mbar_init(&full_b[s], 1);
            tfy_mbar_init(&empty[s], 4);        // one arrival per MMA warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();

    if (warp == PG_TMA_WARP) {
        // ===== weights: the ps rank's bf16 shadow, two 128-row boxes per 64-column chunk =====
        if (tfy_elect_one()) {
            for (int c = 0; c < n_chunks; ++c) {
                const int s = c % PG_STAGES;
                if (c >= PG_STAGES) tfy_mbar_wait(&empty[s], ((c / PG_STAGES) - 1) & 1);
                uint8_t* b_dst = ring + (size_t)s * PG_STAGE_BYTES + PG_A_BYTES;
                tfy_mbar_expect_tx(&full_b[s], PG_B_BYTES);
                tfy_tma_load_2d(&map_w, &full_b[s], b_dst, c * PG_BK, n0);
                tfy_tma_load_2d(&map_w, &full_b[s], b_dst + PG_B_BYTES / 2, c * PG_BK, n0 + 128);
            }
        }
    } else if (warp >= PG_MMA_WARP) {
        // ===== wgmma: piece q = (64-row half q / 4, 64-column quarter q % 4); accumulator word (q, i) of thread t at
        // acc_s[(q * 32 + i) * 128 + t] =====
        const int t = (int)threadIdx.x - PG_MMA_WARP * 32;
        float* mine = acc_s + t;
        for (int i = 0; i < 8 * 32; ++i) mine[i * 128] = 0.f;
        for (int c = 0; c < n_chunks; ++c) {
            const int s = c % PG_STAGES;
            const uint32_t ph = (c / PG_STAGES) & 1;
            tfy_mbar_wait(&full_a[s], ph);
            tfy_mbar_wait(&full_b[s], ph);
            const uint32_t a_addr = tfy_smem_u32(ring + (size_t)s * PG_STAGE_BYTES), b_addr = a_addr + PG_A_BYTES;
#pragma unroll 1
            for (int q = 0; q < 8; ++q) {
                float d[32];
                const uint64_t adesc = tfy_wg_desc_sw128(a_addr + (q >> 2) * 64 * 128);
                const uint64_t bdesc = tfy_wg_desc_sw128(b_addr + (q & 3) * 64 * 128);
                tfy_wg_fence();
#pragma unroll
                for (int k = 0; k < PG_BK / 16; ++k)
                    tfy_wgmma_m64n64<0, 0>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
                tfy_wg_commit();
                tfy_wg_wait<0>();
                float* acc_q = mine + q * 32 * 128;
#pragma unroll
                for (int i = 0; i < 32; ++i) acc_q[i * 128] += d[i];
            }
            if (lane == 0) tfy_mbar_arrive(&empty[s]);
        }
        // ===== epilogue: bias, bf16 pairs (fragment layout: row 16 w + l / 4 (+8), column 8 j + 2 (l % 4)) =====
        const int w = t >> 5;
#pragma unroll 1
        for (int q = 0; q < 8; ++q) {
            const float* acc_q = mine + q * 32 * 128;
#pragma unroll 4
            for (int i = 0; i < 32; i += 2) {
                const int ob = b0 + (q >> 2) * 64 + 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);
                const int n = n0 + (q & 3) * 64 + 8 * (i >> 2) + 2 * (lane & 3);
                if (ob >= B || n >= N) continue;                 // N % 8 == 0: n < N covers n + 1
                float v0 = acc_q[i * 128], v1 = acc_q[(i + 1) * 128];
                if (bias) {
                    v0 += __bfloat162float(bias[n]);
                    v1 += __bfloat162float(bias[n + 1]);
                }
                *reinterpret_cast<__nv_bfloat162*>(y + (size_t)ob * N + n) = __floats2bfloat162_rn(v0, v1);
            }
        }
    } else {
        // ===== A-tile producers: 4 threads per sample; thread (r, p) owns columns [16 p, 16 p + 16) of every chunk =====
        const int pt = (int)threadIdx.x;
        const int r = pt >> 2, p = pt & 3;
        const int b = b0 + r;
        const bool live = b < B;
        auto issue = [&](int c, float4* dst) {
            const float* row = nullptr;
            if (live && c < T) {
                const long long id = ids[(size_t)c * B + b];
                if (id >= 0 && id < V) row = reinterpret_cast<const float*>(tables[c]) + (size_t)id * 64 + p * 16;
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) dst[q] = row ? tfy_ld_peer_f32x4(row + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        };
        float4 buf[PG_DEPTH][4];
#pragma unroll
        for (int j = 0; j < PG_DEPTH; ++j) issue(j, buf[j]);
        for (int c0 = 0; c0 < n_chunks; c0 += PG_DEPTH) {
#pragma unroll
            for (int j = 0; j < PG_DEPTH; ++j) {
                const int c = c0 + j;
                if (c < n_chunks) {
                    const int s = c % PG_STAGES;
                    uint4 pk[2];
                    if (c < T) {
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            pk[h].x = tfy_pack_bf16x2(buf[j][2 * h].x, buf[j][2 * h].y);
                            pk[h].y = tfy_pack_bf16x2(buf[j][2 * h].z, buf[j][2 * h].w);
                            pk[h].z = tfy_pack_bf16x2(buf[j][2 * h + 1].x, buf[j][2 * h + 1].y);
                            pk[h].w = tfy_pack_bf16x2(buf[j][2 * h + 1].z, buf[j][2 * h + 1].w);
                        }
                    } else {
                        float f[16];
#pragma unroll
                        for (int q = 0; q < 16; ++q)
                            f[q] = (live && p * 16 + q < n_num) ? numeric[(size_t)b * n_num + p * 16 + q] : 0.f;
                        pk[0] = TfyPack<__nv_bfloat16>::pack(f);
                        pk[1] = TfyPack<__nv_bfloat16>::pack(f + 8);
                    }
                    if (c >= PG_STAGES) tfy_mbar_wait(&empty[s], ((c / PG_STAGES) - 1) & 1);
                    uint8_t* a_row = ring + (size_t)s * PG_STAGE_BYTES + r * 128;
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        *reinterpret_cast<uint4*>(a_row + (((2 * p + h) ^ (r & 7)) << 4)) = pk[h];
                    tfy_fence_proxy_async();
                    tfy_mbar_arrive(&full_a[s]);
                    if (live) {                          // keep the activations for the backward (dW = dy^T x)
                        __nv_bfloat16* xr = xbuf + (size_t)b * Kp + c * 64 + p * 16;
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            if (c * 64 + p * 16 + h * 8 + 8 <= Kp) tfy_st16(xr + h * 8, pk[h]);
                    }
                    issue(c + PG_DEPTH, buf[j]);         // refill this slot (zeros beyond the last table)
                }
            }
        }
    }
}

namespace {
bool pg_attr_set = false;
}  // namespace

extern "C" {

// Requirements: every table is fp32 [V, 64]; n_num <= 64; N % 8 == 0; Kp % 8 == 0 and Kp >= 64 T + n_num; the weight
// shadow is bf16 [N, Kp] (row pitch Kp), 16-byte aligned; xbuf bf16 [B, Kp], y bf16 [B, N].
int tfy_ps_gather_gemm(const void* w_shadow, const uint64_t* tables, const void* ids, const void* numeric,
                       const void* bias, void* xbuf, void* y, int B, int N, int T, int n_num, int Kp, long long V,
                       cudaStream_t s) {
    if (B < 1 || N < 8 || (N & 7) || (Kp & 7) || n_num < 0 || n_num > 64 || T < 0 || Kp < 64 * T + n_num) return -2;
    if (((uintptr_t)w_shadow | (uintptr_t)xbuf | (uintptr_t)y) & 15) return -3;
    if (!tfy_tensor_map_encoder()) return -4;
    if (!pg_attr_set) {
        if (cudaFuncSetAttribute(tfy_ps_gather_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PG_SMEM) !=
            cudaSuccess)
            return -5;
        pg_attr_set = true;
    }
    CUtensorMap mw;
    if (!tfy_tensor_map_bf16_2d(&mw, w_shadow, N, Kp, Kp)) return -6;
    dim3 grid((B + PG_BM - 1) / PG_BM, (N + PG_BN - 1) / PG_BN);
    tfy_launch_pdl((tfy_ps_gather_gemm_kernel), grid, dim3(PG_THREADS), PG_SMEM, s, mw, tables, (const long long*)ids,
                   (const float*)numeric, (const __nv_bfloat16*)bias, (__nv_bfloat16*)xbuf, (__nv_bfloat16*)y, B, N, T,
                   n_num, Kp, V);
    return (int)cudaGetLastError();
}

}  // extern "C"
