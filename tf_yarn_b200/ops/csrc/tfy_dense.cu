// Dense-layer backward on the Hopper tensor core (sm_90a): BOTH products of a Linear layer's backward in one kernel.
//
//   dW[u, i] = sum_b dh[b, u] * x[b, i]        (M = units, N = in-features, K = batch)
//   dx[b, i] = sum_u dh[b, u] * W[u, i]        (M = batch, N = in-features, K = units)
//
// for the skinny-batch / wide-input layers of the mini-Keras fast path (the MNIST-CNN's 9216 -> 128 layer:
// batch <= 128, units <= 128, in-features = 9216).  The two GEMMs share the dh operand, have the same
// output width and a tiny K, so ONE CTA per 64-column slice of the in-features does both: dh (32 KB) and the
// slice's x and W tiles (16 KB each) arrive by TMA, one warpgroup per product issues wgmma M64 N64 K16 on both
// 64-row halves of its 128-row accumulator, and packs it to bf16 from registers into the B-operand tile it has
// finished reading, for a TMA store (dW straight into the flat gradient buffer the fused optimizer/collective step
// consumes).  At 65 KB of shared memory two CTAs fit per SM, so the 144 CTAs of the 9216-wide layer run in one
// wave.  No operand is transposed in memory: the SAME shared-memory bytes of dh serve as the K-major A operand of dx and, through the transpose flag
// of the wgmma, as the MN-major A operand of dW; x and W tiles are MN-major B operands as they sit in memory
// (in-features contiguous).  This replaces two cuBLAS GEMM launches of the round-1 step
// (reference path being replaced: the Dense backward of the Keras/Horovod worker, tf_yarn/tensorflow/tasks/
// gloo_allred_task.py:54 running TensorFlow's MatMul gradients).
//
// warps 0-3: dW wgmma + epilogue   warps 4-7: dx wgmma + epilogue   warp 8: TMA loads
#include "tfy_common.cuh"
#include "tfy_tma.cuh"
#include "tfy_wgmma.cuh"

namespace {

constexpr int DB_M = 128;             // MMA M: units (dW) / batch (dx), zero-filled by TMA beyond the real extent
constexpr int DB_N = 64;              // in-features per CTA = one 128-byte swizzle atom of bf16
constexpr int DB_K = 128;             // batch (dW) / units (dx)
constexpr int DB_THREADS = 288;
constexpr int DH_BYTES = DB_M * 128 * 2;          // two 64-column boxes of 128 rows x 128 B
constexpr int TILE_BYTES = 128 * 128;             // 128 rows x 64 bf16
constexpr size_t DB_SMEM = 1024 + DH_BYTES + 2 * TILE_BYTES /*x, w*/ + 256;

// Operands are 128-byte swizzled views (tfy_wg_desc_sw128), sbo = 8 rows of 128 B.  K-major: rows = M/N index (64
// K-elements each).  MN-major: rows = K index (64 M/N-elements each); one M64 / N64 operand is exactly one atom, so
// lbo is unused.
// dW = dh^T . x (A = dh MN-major: M = units, 64-unit halves TILE_BYTES apart; K = batch rows, 16 rows = 2048 B per
// MMA; B = x / W tile MN-major: N = 64 in-features in one atom)   -- TA = 1
// dx = dh . W   (A = dh K-major: M = batch rows, 64-row halves 8 KB apart; K = units: 4 x 32 B inside each 64-unit
// atom; B = W tile MN-major, K = unit rows, 2048 B per MMA)      -- TA = 0
template <int TA>
__device__ __forceinline__ void d_mma_chunk(float (&acc)[2][DB_N / 2], uint32_t dh0, uint32_t t0, bool first) {
#pragma unroll
    for (int k = 0; k < DB_K / 16; ++k) {
        const uint64_t bdesc = tfy_wg_desc_sw128(t0 + k * 2048);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t a = TA ? dh0 + h * TILE_BYTES + k * 2048 : dh0 + (k >> 2) * TILE_BYTES + (k & 3) * 32 + h * 8192;
            tfy_wgmma_m64n64<TA, 1>(acc[h], tfy_wg_desc_sw128(a), bdesc, (first && k == 0) ? 0u : 1u);
        }
    }
}

// Warpgroup epilogue: accumulator -> bf16, 128-byte-swizzled [128 rows][128 B] tile (stage) -> one TMA store.  Each
// thread packs its fragment's column pairs straight from registers (the rounding TfyPack<bf16> applies), so `stage`
// may be the B-operand tile the warpgroup's wgmma has just read.  `bar` is the named barrier of the warpgroup.
__device__ __forceinline__ void d_epilogue(float (&acc)[2][DB_N / 2], uint8_t* stage, int bar, const CUtensorMap* map,
                                           int c0, int c1) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");     // every warp's wgmma is done reading `stage`
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        // fragment rows 16 w + l / 4 and 8 below it; columns 8 j + 2 (l % 4) + {0, 1} = bytes 4 (l % 4) of 16-byte
        // chunk j, stored at chunk j XOR (row mod 8) (the 128-byte swizzle of the TMA store map; row mod 8 = l / 4)
        uint8_t* r0 = stage + (h * 64 + 16 * w + (l >> 2)) * 128 + 4 * (l & 3);
#pragma unroll
        for (int j = 0; j < DB_N / 8; ++j) {
            const int sw = (j ^ (l >> 2)) << 4;
            *reinterpret_cast<uint32_t*>(r0 + sw) = tfy_pack_bf16x2(acc[h][4 * j], acc[h][4 * j + 1]);
            *reinterpret_cast<uint32_t*>(r0 + 8 * 128 + sw) = tfy_pack_bf16x2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
    }
    tfy_fence_proxy_async();     // generic-proxy writes -> async proxy
    asm volatile("bar.sync %0, 128;" ::"r"(bar) : "memory");
    if ((threadIdx.x & 127) < 32 && tfy_elect_one()) {
        tfy_tma_store_2d(map, stage, c0, c1);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem must outlive the read
    }
}

}  // namespace

__global__ void __launch_bounds__(DB_THREADS, 2)
tfy_dense_bwd_kernel(const __grid_constant__ CUtensorMap map_dh, const __grid_constant__ CUtensorMap map_x,
                     const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_dw,
                     const __grid_constant__ CUtensorMap map_dx, int want_dx) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = tfy_align1024(smem_raw);
    uint8_t* s_dh = smem;                            // [2 boxes][128 rows (batch)][128 B (64 units)]  sw128
    uint8_t* s_x = s_dh + DH_BYTES;                  // [128 rows (batch)][128 B (64 in-features)]     sw128
    uint8_t* s_w = s_x + TILE_BYTES;                 // [128 rows (units)][128 B (64 in-features)]     sw128
    uint64_t* full = reinterpret_cast<uint64_t*>(s_w + TILE_BYTES);

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // warp-uniform role index
    const int n0 = blockIdx.x * DB_N;
    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_dh);
        tfy_prefetch_tensormap(&map_x);
        tfy_prefetch_tensormap(&map_w);
        tfy_prefetch_tensormap(&map_dw);
        tfy_prefetch_tensormap(&map_dx);
        tfy_mbar_init(full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();

    if (warp == 8) {
        if (tfy_elect_one()) {
            tfy_mbar_expect_tx(full, DH_BYTES + TILE_BYTES + (want_dx ? TILE_BYTES : 0));
            tfy_tma_load_2d(&map_dh, full, s_dh, 0, 0);
            tfy_tma_load_2d(&map_dh, full, s_dh + TILE_BYTES, 64, 0);
            tfy_tma_load_2d(&map_x, full, s_x, n0, 0);
            if (want_dx) tfy_tma_load_2d(&map_w, full, s_w, n0, 0);
        }
        return;
    }
    const int which = warp >> 2;                     // 0 -> dW (warps 0-3), 1 -> dx (warps 4-7)
    if (which == 1 && !want_dx) return;
    tfy_mbar_wait(full, 0);
    const uint32_t dh0 = tfy_smem_u32(s_dh);
    float acc[2][DB_N / 2];
    tfy_wg_fence();
    if (which == 0) d_mma_chunk<1>(acc, dh0, tfy_smem_u32(s_x), true);
    else d_mma_chunk<0>(acc, dh0, tfy_smem_u32(s_w), true);
    tfy_wg_commit();
    tfy_wg_wait<0>();
    // dW is staged in the x tile, dx in the W tile: each is read by its own warpgroup's wgmma only
    d_epilogue(acc, which == 0 ? s_x : s_w, 1 + which, which == 0 ? &map_dw : &map_dx, n0, 0);
}

// ---------------------------------------------------------------------------------------------------------
// General shapes (batch > 128 and / or units > 128): one CTA per (64-column slice of the in-features, job) where
// a job is either a 128-unit tile of dW -- K loop over the batch in chunks of 128 rows -- or a 128-row tile of
// dx -- K loop over the units in chunks of 128.  Same operand views and epilogue as the single-shot kernel, with
// a 3-stage TMA ring (48 KB per stage: the two 64-column boxes of the dh chunk + the x or W tile).
// warps 0-3: wgmma + epilogue   warp 4: TMA producer
// ---------------------------------------------------------------------------------------------------------
namespace {
constexpr int DT_STAGES = 3, DT_STAGE_BYTES = DH_BYTES + TILE_BYTES, DT_THREADS = 160;
constexpr size_t DT_SMEM = 1024 + (size_t)DT_STAGES * DT_STAGE_BYTES + TILE_BYTES + 256;
}  // namespace

__global__ void __launch_bounds__(DT_THREADS, 1)
tfy_dense_bwd_tiled_kernel(const __grid_constant__ CUtensorMap map_dh, const __grid_constant__ CUtensorMap map_x,
                           const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_dw,
                           const __grid_constant__ CUtensorMap map_dx, int n_u_tiles, int n_b_tiles, int want_dx) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = tfy_align1024(smem_raw);
    uint8_t* ring = smem;                                            // [3] { dh box0, dh box1, tile }
    uint8_t* s_out = ring + (size_t)DT_STAGES * DT_STAGE_BYTES;      // staging for the TMA store
    uint64_t* full = reinterpret_cast<uint64_t*>(s_out + TILE_BYTES);
    uint64_t* empty = full + DT_STAGES;

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    const int n0 = blockIdx.x * DB_N;
    const int job = blockIdx.y;
    const bool is_dw = job < n_u_tiles;
    const int m0 = (is_dw ? job : job - n_u_tiles) * DB_M;           // first unit (dW) / batch row (dx) of the tile
    const int n_chunks = is_dw ? n_b_tiles : n_u_tiles;              // K loop: batch chunks (dW) / unit chunks (dx)
    if (!is_dw && !want_dx) return;
    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_dh);
        tfy_prefetch_tensormap(is_dw ? &map_x : &map_w);
        for (int st = 0; st < DT_STAGES; ++st) { tfy_mbar_init(&full[st], 1); tfy_mbar_init(&empty[st], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();

    if (warp == 4) {
        if (tfy_elect_one()) {
            for (int i = 0; i < n_chunks; ++i) {
                const int st = i % DT_STAGES;
                if (i >= DT_STAGES) tfy_mbar_wait(&empty[st], ((i / DT_STAGES) - 1) & 1);
                uint8_t* dst = ring + (size_t)st * DT_STAGE_BYTES;
                tfy_mbar_expect_tx(&full[st], DT_STAGE_BYTES);
                const int k0 = i * DB_K;
                if (is_dw) {           // dh rows = batch chunk, columns = this tile's units; x rows = batch chunk
                    tfy_tma_load_2d(&map_dh, &full[st], dst, m0, k0);
                    tfy_tma_load_2d(&map_dh, &full[st], dst + TILE_BYTES, m0 + 64, k0);
                    tfy_tma_load_2d(&map_x, &full[st], dst + DH_BYTES, n0, k0);
                } else {               // dh rows = this tile's batch rows, columns = unit chunk; W rows = unit chunk
                    tfy_tma_load_2d(&map_dh, &full[st], dst, k0, m0);
                    tfy_tma_load_2d(&map_dh, &full[st], dst + TILE_BYTES, k0 + 64, m0);
                    tfy_tma_load_2d(&map_w, &full[st], dst + DH_BYTES, n0, k0);
                }
            }
        }
        return;
    }
    float acc[2][DB_N / 2];
    tfy_wg_zero<DB_N>(acc[0]);
    tfy_wg_zero<DB_N>(acc[1]);
    for (int i = 0; i < n_chunks; ++i) {
        const int st = i % DT_STAGES;
        tfy_mbar_wait(&full[st], (i / DT_STAGES) & 1);
        tfy_wg_fence();
        const uint32_t dh0 = tfy_smem_u32(ring + (size_t)st * DT_STAGE_BYTES), t0 = dh0 + DH_BYTES;
        if (is_dw) d_mma_chunk<1>(acc, dh0, t0, false);
        else d_mma_chunk<0>(acc, dh0, t0, false);
        tfy_wg_commit();
        tfy_wg_wait<0>();
        if (lane == 0) tfy_mbar_arrive(&empty[st]);
    }
    d_epilogue(acc, s_out, 1, is_dw ? &map_dw : &map_dx, n0, m0);
}

namespace {
bool d_attr_set = false, d_attr_set_tiled = false;
}  // namespace

extern "C" {

// dh: [B, U] bf16 (gradient wrt the layer's pre-activation), x: [B, I] bf16 (the layer's input), w: [U, I] bf16.
// dw: [U, I] bf16 (overwritten), dx: [B, I] bf16 (overwritten; nullptr = first layer, no data gradient).
// Requirements: U % 8 == 0, I % 8 == 0, 16-byte aligned pointers (-2 / -3 otherwise).  batch <= 128 and units <= 128
// take the single-shot kernel (one CTA per 64 in-features does both products); anything larger the tiled one.
int tfy_dense_bwd(const void* dh, const void* x, const void* w, void* dw, void* dx, int B, int U, int I,
                  cudaStream_t s) {
    if (B < 1 || U < 8 || (U & 7) || (I & 7) || I < 8) return -2;
    if (B > DB_M || U > DB_M) {
        if (((uintptr_t)dh | (uintptr_t)x | (uintptr_t)w | (uintptr_t)dw | (uintptr_t)dx) & 15) return -3;
        if (!tfy_tensor_map_encoder()) return -4;
        if (!d_attr_set_tiled) {
            if (cudaFuncSetAttribute(tfy_dense_bwd_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)DT_SMEM) != cudaSuccess)
                return -5;
            d_attr_set_tiled = true;
        }
        CUtensorMap mdh, mx, mw, mdw, mdx;
        if (!tfy_tensor_map_bf16_2d(&mdh, dh, B, U, U) || !tfy_tensor_map_bf16_2d(&mx, x, B, I, I) ||
            !tfy_tensor_map_bf16_2d(&mw, w, U, I, I) || !tfy_tensor_map_bf16_2d(&mdw, dw, U, I, I) ||
            !tfy_tensor_map_bf16_2d(&mdx, dx ? dx : dw, dx ? B : U, I, I))
            return -6;
        const int n_u = (U + DB_M - 1) / DB_M, n_b = (B + DB_M - 1) / DB_M;
        dim3 grid((I + DB_N - 1) / DB_N, n_u + (dx ? n_b : 0));
        tfy_launch_pdl((tfy_dense_bwd_tiled_kernel), grid, dim3(DT_THREADS), DT_SMEM, s, mdh, mx, mw, mdw, mdx, n_u, n_b,
                       dx != nullptr ? 1 : 0);
        return (int)cudaGetLastError();
    }
    if (((uintptr_t)dh | (uintptr_t)x | (uintptr_t)w | (uintptr_t)dw | (uintptr_t)dx) & 15) return -3;
    if (!tfy_tensor_map_encoder()) return -4;
    if (!d_attr_set) {
        if (cudaFuncSetAttribute(tfy_dense_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DB_SMEM) !=
            cudaSuccess)
            return -5;
        d_attr_set = true;
    }
    CUtensorMap mdh, mx, mw, mdw, mdx;
    if (!tfy_tensor_map_bf16_2d(&mdh, dh, B, U, U) || !tfy_tensor_map_bf16_2d(&mx, x, B, I, I) ||
        !tfy_tensor_map_bf16_2d(&mw, w, U, I, I) || !tfy_tensor_map_bf16_2d(&mdw, dw, U, I, I) ||
        !tfy_tensor_map_bf16_2d(&mdx, dx ? dx : dw, dx ? B : U, I, I))
        return -6;
    const int grid = (I + DB_N - 1) / DB_N;
    tfy_launch_pdl((tfy_dense_bwd_kernel), dim3(grid), dim3(DB_THREADS), DB_SMEM, s, mdh, mx, mw, mdw, mdx,
                   dx != nullptr ? 1 : 0);
    return (int)cudaGetLastError();
}

}  // extern "C"
