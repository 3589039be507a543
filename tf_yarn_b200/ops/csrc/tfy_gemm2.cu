// Persistent Hopper GEMM for sm_90a:  C[M,N] = act(A[M,K] . B[N,K]^T + bias[N])   (bf16 in, fp32 accumulate)
//
// The large-shape companion of tfy_gemm.cu (one 128x128 tile per CTA, which re-reads both operands for every
// tile and runs one warpgroup).  Here one CTA per SM walks the output tiles of 128 x 256 (static round-robin):
//   * two consumer warpgroups, each issuing wgmma M64 N256 K16 on its 64-row half of the tile, share every
//     B byte staged in shared memory (256 x 64 per stage) -- twice the operand re-use of the 128x128 kernel;
//   * a 4-stage TMA ring (48 KB per stage) shared by all tiles of the CTA, so the loads of the next tile start
//     while the current one is drained;
//   * epilogue straight from the accumulator registers: bias / ReLU -> bf16 pairs -> global.
// Roles: warps 0-3 and 4-7 the two consumer warpgroups, warp 8 the TMA producer.
// The B operand may be a peer (NVLink) address, as in tfy_gemm.cu.
#include "tfy_common.cuh"
#include "tfy_tma.cuh"
#include "tfy_wgmma.cuh"

namespace {

constexpr int G2_BM = 128, G2_BN = 256, G2_BK = 64;      // output tile of a CTA
constexpr int G2_STAGES = 4;
constexpr int G2_A_BYTES = G2_BM * G2_BK * 2, G2_B_BYTES = G2_BN * G2_BK * 2;
constexpr int G2_STAGE_BYTES = G2_A_BYTES + G2_B_BYTES;                // 48 KB per stage
constexpr int G2_THREADS = 288;
constexpr size_t G2_SMEM = 1024 + (size_t)G2_STAGES * G2_STAGE_BYTES + 512;

}  // namespace

__global__ void __launch_bounds__(G2_THREADS, 1)
tfy_gemm2_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                      __nv_bfloat16* __restrict__ C, const __nv_bfloat16* __restrict__ bias, int M, int N, int K,
                      int ldc, int relu) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = tfy_align1024(smem_raw);
    uint8_t* ring = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)G2_STAGES * G2_STAGE_BYTES);
    uint64_t* empty = full + G2_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_m = (M + G2_BM - 1) / G2_BM, tiles_n = (N + G2_BN - 1) / G2_BN;
    const int n_tiles = tiles_m * tiles_n;
    const int k_blocks = (K + G2_BK - 1) / G2_BK;

    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_a);
        tfy_prefetch_tensormap(&map_b);
        for (int s = 0; s < G2_STAGES; ++s) {
            tfy_mbar_init(&full[s], 1);         // the producer's expect_tx + the TMA bytes
            tfy_mbar_init(&empty[s], 8);        // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();

    if (warp == 8) {
        // ===== TMA producer: 128 rows of A and 256 rows of B (two 128-row boxes) per stage =====
        if (tfy_elect_one()) {
            uint32_t it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int m0 = (t % tiles_m) * G2_BM, n0 = (t / tiles_m) * G2_BN;
                for (int kb = 0; kb < k_blocks; ++kb, ++it) {
                    const int s = it % G2_STAGES;
                    if (it >= G2_STAGES) tfy_mbar_wait(&empty[s], ((it / G2_STAGES) - 1) & 1);
                    uint8_t* a_dst = ring + (size_t)s * G2_STAGE_BYTES;
                    tfy_mbar_expect_tx(&full[s], G2_STAGE_BYTES);
                    tfy_tma_load_2d(&map_a, &full[s], a_dst, kb * G2_BK, m0);
                    tfy_tma_load_2d(&map_b, &full[s], a_dst + G2_A_BYTES, kb * G2_BK, n0);
                    tfy_tma_load_2d(&map_b, &full[s], a_dst + G2_A_BYTES + G2_B_BYTES / 2, kb * G2_BK, n0 + 128);
                }
            }
        }
        return;
    }
    // ===== consumers: warpgroup h owns rows [64 h, 64 h + 64) of every tile =====
    const int h = warp >> 2, w = warp & 3;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int m0 = (t % tiles_m) * G2_BM, n0 = (t / tiles_m) * G2_BN;
        float acc[G2_BN / 2];
        tfy_wg_zero<G2_BN>(acc);
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
            const int s = it % G2_STAGES;
            tfy_mbar_wait(&full[s], (it / G2_STAGES) & 1);
            tfy_wg_fence();
            const uint32_t a_addr = tfy_smem_u32(ring + (size_t)s * G2_STAGE_BYTES);
            const uint64_t adesc = tfy_wg_desc_sw128(a_addr + h * 64 * 128);
            const uint64_t bdesc = tfy_wg_desc_sw128(a_addr + G2_A_BYTES);
#pragma unroll
            for (int k = 0; k < G2_BK / 16; ++k)
                tfy_wgmma_m64n256<0, 0>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), 1u);
            tfy_wg_commit();
            tfy_wg_wait<1>();                            // the previous stage's wgmmas have retired
            if (kb > 0 && lane == 0) tfy_mbar_arrive(&empty[(it - 1) % G2_STAGES]);
        }
        tfy_wg_wait<0>();
        if (k_blocks > 0 && lane == 0) tfy_mbar_arrive(&empty[(it - 1) % G2_STAGES]);
        // fragment layout: value i of this thread is row 16 w + lane / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (lane % 4)
        const int r0 = m0 + h * 64 + 16 * w + (lane >> 2);
#pragma unroll
        for (int i = 0; i < G2_BN / 2; i += 2) {
            const int row = r0 + 8 * ((i >> 1) & 1), n = n0 + 8 * (i >> 2) + 2 * (lane & 3);
            if (row >= M || n >= N) continue;
            float v0 = acc[i], v1 = acc[i + 1];
            if (bias) {
                v0 += __bfloat162float(bias[n]);
                if (n + 1 < N) v1 += __bfloat162float(bias[n + 1]);
            }
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            __nv_bfloat16* dst = C + (size_t)row * ldc + n;
            if (n + 1 < N) *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
            else dst[0] = __float2bfloat16(v0);
        }
    }
}

namespace {

bool g2_attr_set = false;
int g2_sms = 0;

}  // namespace

extern "C" {

// C[M,N] (bf16, ld ldc) = act(A[M,K] (ld lda) . B[N,K]^T (ld ldb) + bias[N]); B may be a peer (NVLink) pointer.
// Requirements: K % 8 == 0, lda/ldb/ldc % 8 == 0, 16-byte aligned base pointers.
int tfy_gemm2_bf16(const void* A, const void* B, void* C, const void* bias, int M, int N, int K, int lda, int ldb,
                   int ldc, int relu, cudaStream_t s) {
    if ((K & 7) || (lda & 7) || (ldb & 7) || (ldc & 7)) return -2;
    if (((uintptr_t)A | (uintptr_t)B | (uintptr_t)C) & 15) return -3;
    if (!tfy_tensor_map_encoder()) return -4;
    if (!g2_attr_set) {
        if (cudaFuncSetAttribute(tfy_gemm2_bf16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G2_SMEM) !=
            cudaSuccess)
            return -5;
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&g2_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || g2_sms < 1) return -5;
        g2_attr_set = true;
    }
    CUtensorMap ma, mb;
    if (!tfy_tensor_map_bf16_2d(&ma, A, M, K, lda) || !tfy_tensor_map_bf16_2d(&mb, B, N, K, ldb)) return -6;
    const int n_tiles = ((M + G2_BM - 1) / G2_BM) * ((N + G2_BN - 1) / G2_BN);
    const int grid = n_tiles < g2_sms ? n_tiles : g2_sms;
    tfy_launch_pdl((tfy_gemm2_bf16_kernel), dim3(grid), dim3(G2_THREADS), G2_SMEM, s, ma, mb, (__nv_bfloat16*)C,
                   (const __nv_bfloat16*)bias, M, N, K, ldc, relu);
    return (int)cudaGetLastError();
}

}  // extern "C"
