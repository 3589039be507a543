// Hopper GEMM for sm_90a:  C[M,N] = act(A[M,K] . B[N,K]^T + bias[N])   (bf16 in, fp32 accumulate)
//
// This is the compute half of K5, the parameter-server PULL fused with the consuming GEMM:
// B (the layer's weight matrix) is addressed through a TMA tensor map whose base pointer may be a
// PEER address -- the ps rank's HBM mapped over NVLink by the symmetric arena -- so the weight
// tiles stream from the parameter server's memory straight into this SM's shared memory and into
// the tensor core, with no staging copy of the shard on the worker (reference path being replaced:
// TF gRPC RecvTensor of every variable before the first consumer op, tf_yarn/tensorflow/cluster.py:
// 60-66).  With a local B it is also the dense-layer GEMM of the mini-Keras fast path.
//
// Structure (one 128x128 output tile per CTA, 160 threads):
//   warps 0-3: one warpgroup -- wgmma M64 N128 K16 (kind f32.bf16.bf16) on both 64-row halves of the tile,
//              accumulators in registers; then the epilogue: the fp32 tile goes through shared memory so that
//              each thread owns one row, bias + activation, bf16 stores; or fp32 red.add for split-K
//   warp 4   : TMA producer  -- cp.async.bulk.tensor.2d of a 128x64 A box and a 128x64 B box per
//              stage (128-byte swizzle), completion on an mbarrier (complete_tx)
// Pipeline: STAGES-deep ring of {A,B} tiles guarded by full/empty mbarriers.
//
// Sub-tiled split-K (slab output only): when tiles x K-slices leave most SMs idle, the FM x FN CTAs of a cluster share
// one tile -- CTA (cx, cy) owns rows [64 cx, 64 cx + 64) of it when FM = 2 and columns [64 cy, 64 cy + 64) when FN = 2.
// Each runs, for its rows and columns, the k16 chain the one-tile CTA runs (same wgmma shape along M, same K order,
// one accumulator from zero), so the slabs are the same bits.  The A rows a CTA needs are shared with the FN CTAs of
// its cluster row and the B rows with the FM CTAs of its column: each CTA loads 1/FN of its A box and 1/FM of its B
// box and multicasts them, and a stage is refilled only after the consumers of every CTA of the cluster released it.
#include "tfy_common.cuh"
#include "tfy_tma.cuh"
#include "tfy_wgmma.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 64, UMMA_K = 16;
constexpr int GEMM_THREADS = 160;
constexpr int RING_BYTES = 4 * (BM + BN) * BK * 2;   // four stages of the one-tile CTA

// The shape of one CTA's work when FM x FN CTAs share a 128 x 128 tile.
template <int FM, int FN>
struct GemmGeom {
    static constexpr int CLUSTER = FM * FN;
    static constexpr int SM = BM / FM, SN = BN / FN;                   // rows of A and of B this CTA multiplies
    static constexpr int A_BYTES = SM * BK * 2, B_BYTES = SN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = RING_BYTES / STAGE_BYTES;            // 4 (one tile), 5 (2 x 1), 8 (2 x 2)
    static constexpr int BOX_ROWS = 128 / CLUSTER;                     // rows of the A and B boxes one CTA loads
    static constexpr int ACC_LD = SN + 4;     // fp32 row pitch of the staged accumulator (conflict-free row reads)
    static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + (size_t)SM * ACC_LD * 4 + 1024 /*align slack*/ +
                                   256 /*barriers*/;
    static_assert(2 * STAGES * 8 <= 256, "ring barriers overflow their shared-memory slot");
    static_assert(A_BYTES % 1024 == 0 && (SM / FN) * 128 % 1024 == 0 && (SN / FM) * 128 % 1024 == 0,
                  "boxes must land on 128-byte-swizzle atoms");
};

// Optional per-CTA event timeline (tests/gpu/gemm_timeline.py): 16 slots per CTA, slot 0 the CTA's start on the
// global timer (ns), the others SM-clock deltas from it.  CTA index: x + gridDim.x * (y + gridDim.y * z).
__device__ long long* g_timeline = nullptr;
#define G_MARK(k)                                                                                         \
    do {                                                                                                  \
        if (g_tl) g_tl[(size_t)(blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)) * 16 + (k)] = \
            clock64() - g_t0;                                                                             \
    } while (0)

}  // namespace

// Split-K partial sums are never added with atomics: K-slice z stores its fp32 partial tile into slab z of the
// workspace (slab stride M * ldc) and the slabs are summed in slice order afterwards, so the result is the same
// bit for bit on every run.
// Fused split-K epilogue (out_mode 2): what runs after the partial sums of ALL K-slices of a tile are stored.
// The K-slice CTAs of the tile share the work: each sums a part of the tile over the slabs, applies bias + ReLU +
// dropout and writes the bf16 activations and the gradient-gate mask -- the work of the separate
// tfy_bias_act_drop_fwd_f32 launch (same element indexing, same random numbers).
struct TfySplitKEpilogue {
    uint32_t* counters;      // two per output tile (arrive, finish), zero on entry, left zero
    __nv_bfloat16* y;        // [M, N] bf16 activations (row pitch ldy)
    uint8_t* mask;           // [M, N] bytes: 1 = gradient flows (optional)
    const TfyOptHyper* hp;   // dropout step counter
    float drop_rate;
    uint32_t seed;
    int ldy;
};

// out_mode 0: C (bf16) = act(acc + bias)      out_mode 1: slab blockIdx.z of C32 (fp32) = acc   (split-K partials)
// out_mode 2: as 1, then the K-slice CTAs of every tile run the fused epilogue above (one CTA per tile only)
// FM x FN > 1: a cluster of FM x FN CTAs shares each tile (out_mode 1 only); the grid is (tiles_m FM, tiles_n FN, splits).
template <int FM, int FN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
tfy_gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     __nv_bfloat16* __restrict__ C, float* __restrict__ C32, const __nv_bfloat16* __restrict__ bias,
                     int M, int N, int K, int ldc, int relu, int out_mode, int k_tiles_per_split, TfySplitKEpilogue ep) {
    using Geom = GemmGeom<FM, FN>;
    constexpr int STAGES = Geom::STAGES, A_BYTES = Geom::A_BYTES, STAGE_BYTES = Geom::STAGE_BYTES, ACC_LD = Geom::ACC_LD;
    extern __shared__ uint8_t smem_raw[];
    long long* const g_tl = g_timeline;
    const long long g_t0 = clock64();
    if (g_tl && threadIdx.x == 0) {
        unsigned long long ns;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
        g_tl[(size_t)(blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)) * 16] = (long long)ns;
    }
    uint8_t* smem = tfy_align1024(smem_raw);
    uint8_t* tiles = smem;
    float* acc_s = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE_BYTES);     // [Geom::SM][ACC_LD]
    uint64_t* full = reinterpret_cast<uint64_t*>(acc_s + (size_t)Geom::SM * ACC_LD);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // this CTA's coordinates in its cluster (cluster rank cx + FM cy) and the first row of A and of B it multiplies
    const int cx = (int)blockIdx.x % FM, cy = (int)blockIdx.y % FN;
    const int m0 = (int)blockIdx.x * Geom::SM, n0 = (int)blockIdx.y * Geom::SN;
    const int total_k_tiles = (K + BK - 1) / BK;
    const int kt0 = blockIdx.z * k_tiles_per_split;
    int kt1 = kt0 + k_tiles_per_split;
    if (kt1 > total_k_tiles) kt1 = total_k_tiles;
    const int n_kt = kt1 - kt0;

    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_a);
        tfy_prefetch_tensormap(&map_b);
        for (int s = 0; s < STAGES; ++s) {
            tfy_mbar_init(&full[s], 1);
            tfy_mbar_init(&empty[s], 4 * Geom::CLUSTER);   // one arrival per MMA warp of every CTA the stage feeds
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if constexpr (Geom::CLUSTER > 1)
        tfy_cluster_sync<true>();        // the peers' barriers are initialised before anything lands on them
    else
        __syncthreads();
    tfy_pdl_sync();                      // upstream grids complete; our dependents may start launching
    if (threadIdx.x == 0) G_MARK(1);

    if (warp == 4) {
        if (tfy_elect_one()) {
            for (int i = 0; i < n_kt; ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (i / STAGES) & 1;
                tfy_mbar_wait(&empty[s], ph ^ 1);
                uint8_t* a_dst = tiles + (size_t)s * STAGE_BYTES;
                uint8_t* b_dst = a_dst + A_BYTES;
                tfy_mbar_expect_tx(&full[s], STAGE_BYTES);   // including the boxes the peers multicast to us
                const int k0 = (kt0 + i) * BK;
                if constexpr (FN == 1) {
                    tfy_tma_load_2d(&map_a, &full[s], a_dst, k0, m0);
                } else {                 // our share of the A rows, to every CTA of our cluster row
                    constexpr int rows = Geom::SM / FN;
                    uint16_t mask = 0;
                    for (int y = 0; y < FN; ++y) mask |= (uint16_t)(1u << (cx + FM * y));
                    tfy_tma_load_2d_multicast(&map_a, &full[s], a_dst + cy * rows * 128, k0, m0 + cy * rows, mask);
                }
                if constexpr (FM == 1) {
                    tfy_tma_load_2d(&map_b, &full[s], b_dst, k0, n0);
                } else {                 // our share of the B rows, to every CTA of our cluster column
                    constexpr int rows = Geom::SN / FM;
                    const uint16_t mask = (uint16_t)(((1u << FM) - 1u) << (FM * cy));
                    tfy_tma_load_2d_multicast(&map_b, &full[s], b_dst + cx * rows * 128, k0, n0 + cx * rows, mask);
                }
            }
        }
        if constexpr (Geom::CLUSTER > 1) {
            __syncwarp();
            tfy_cluster_sync();          // the peers stop arriving on our barriers before this CTA exits
        }
        return;
    }
    {
        // ---- MMA: the warpgroup accumulates its 64-row halves; a stage is released once the wgmmas of the
        // NEXT stage are issued and the older group has retired (one group in flight behind the TMA ring)
        constexpr int HALVES = Geom::SM / 64;
        float acc[HALVES][Geom::SN / 2];
#pragma unroll
        for (int h = 0; h < HALVES; ++h) tfy_wg_zero<Geom::SN>(acc[h]);
        for (int i = 0; i < n_kt; ++i) {
            const int s = i % STAGES;
            tfy_mbar_wait(&full[s], (i / STAGES) & 1);
            if (i == 0 && threadIdx.x == 0) G_MARK(2);
            tfy_wg_fence();
            const uint32_t a_addr = tfy_smem_u32(tiles + (size_t)s * STAGE_BYTES);
            const uint64_t bdesc = tfy_wg_desc_sw128(a_addr + A_BYTES);
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
                // advance 16 bf16 = 32 B along K inside the 128 B swizzle atom: +2 in 16-byte units
#pragma unroll
                for (int h = 0; h < HALVES; ++h) {
                    const uint64_t adesc = tfy_wg_desc_sw128(a_addr + h * 64 * 128) + (uint64_t)(2 * k);
                    if constexpr (Geom::SN == 128)
                        tfy_wgmma_m64n128<0, 0>(acc[h], adesc, bdesc + (uint64_t)(2 * k), 1u);
                    else
                        tfy_wgmma_m64n64<0, 0>(acc[h], adesc, bdesc + (uint64_t)(2 * k), 1u);
                }
            }
            tfy_wg_commit();
            tfy_wg_wait<1>();
            if constexpr (Geom::CLUSTER > 1) {   // lane r releases the stage to cluster CTA r
                if (i > 0 && lane < Geom::CLUSTER) tfy_mbar_arrive_cluster(&empty[(i - 1) % STAGES], lane);
            } else {
                if (i > 0 && lane == 0) tfy_mbar_arrive(&empty[(i - 1) % STAGES]);
            }
        }
        tfy_wg_wait<0>();
        if (threadIdx.x == 0) G_MARK(3);
#pragma unroll
        for (int h = 0; h < HALVES; ++h) tfy_wg_store_rows<Geom::SN>(acc_s, ACC_LD, acc[h], 64 * h);
        asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    {
        // epilogue: FM threads per row of the CTA's tile (one when it is the whole 128-row tile), each storing
        // Geom::SN / FM consecutive columns
        constexpr int COLS = Geom::SN / FM;
        const int r = threadIdx.x / FM, c0 = (threadIdx.x % FM) * COLS;
        const int row = m0 + r;
        const bool row_ok = row < M;
        const float* acc_row = acc_s + (size_t)r * ACC_LD;
#pragma unroll 1
        for (int c = c0; c < c0 + COLS; c += 16) {
            const int n = n0 + c;
            if (!row_ok || n >= N || n_kt <= 0) continue;
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(v + j) = *reinterpret_cast<const float4*>(acc_row + c + j);
            if (Geom::CLUSTER > 1 || out_mode >= 1) {
                float* dst = C32 + (size_t)blockIdx.z * M * ldc + (size_t)row * ldc + n;
                if (n + 16 <= N && (ldc & 3) == 0 && (n & 3) == 0) {
#pragma unroll
                    for (int j = 0; j < 16; j += 4) __stcg(reinterpret_cast<float4*>(dst + j), *reinterpret_cast<float4*>(v + j));
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (n + j < N) __stcg(dst + j, v[j]);
                }
            } else {
                if (bias) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (n + j < N) v[j] += __bfloat162float(bias[n + j]);
                }
                if (relu) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                __nv_bfloat16* dst = C + (size_t)row * ldc + n;
                if (n + 16 <= N && (ldc & 7) == 0 && (n & 7) == 0) {
                    tfy_st16(dst, TfyPack<__nv_bfloat16>::pack(v));
                    tfy_st16(dst + 8, TfyPack<__nv_bfloat16>::pack(v + 8));
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (n + j < N) dst[j] = __float2bfloat16(v[j]);
                }
            }
        }
        if (g_tl) {                                  // every thread of the tile has issued its stores
            asm volatile("bar.sync 1, 128;" ::: "memory");
            if (threadIdx.x == 0) G_MARK(4);
        }
    }
    if constexpr (Geom::CLUSTER > 1) tfy_cluster_sync();
    if (Geom::CLUSTER == 1 && out_mode == 2) {
        // ---- fused split-K epilogue, spread over ALL K-slice CTAs of the tile ----
        // Every CTA arrives on the tile's counter after its slab stores, waits until all gridDim.z slices have arrived
        // (they are co-resident: the host only selects this mode when the whole grid fits the SMs) and then finishes
        // 1/gridDim.z of the tile: one 8-element group per thread, i.e. ONE L2 round trip.  (A first version let the
        // last-arriving CTA finish the whole 128x128 tile alone: 16 dependent L2 round trips per thread, +9 us.)
        uint32_t* cnt = ep.counters + 2 * (blockIdx.y * gridDim.x + blockIdx.x);
        asm volatile("bar.sync 1, 128;" ::: "memory");                 // this CTA's slab stores are all issued
        if (threadIdx.x == 0) {
            __threadfence();
            atomicAdd(cnt, 1u);
            while (*reinterpret_cast<volatile uint32_t*>(cnt) < gridDim.z) {
            }
            __threadfence();
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        {
            const uint32_t step = ep.hp ? (uint32_t)ep.hp->step : 0u;
            const float keep_scale = ep.drop_rate > 0.f ? 1.f / (1.f - ep.drop_rate) : 1.f;
            const int t = threadIdx.x;                                 // 0..127
            const int G = N / 8;                                       // 8-element groups per row (N % 8 == 0)
            constexpr int tile_g = BN / 8, tile_groups = BM * tile_g;
            const int per = (tile_groups + (int)gridDim.z - 1) / (int)gridDim.z;
            const int lo = (int)blockIdx.z * per, hi = min(lo + per, tile_groups);
            for (int i = lo + t; i < hi; i += 128) {
                const int r = i / tile_g, gq = i % tile_g;
                const int row = m0 + r, n = n0 + gq * 8;
                if (row >= M || n >= N) continue;
                float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
                for (int z = 0; z < (int)gridDim.z; ++z) {             // slice order: the same sum on every run
                    const float4* zp = reinterpret_cast<const float4*>(C32 + (size_t)z * M * ldc + (size_t)row * ldc + n);
                    const float4 a = __ldcg(zp), b = __ldcg(zp + 1);
                    v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w;
                    v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
                }
                if (bias) {
                    float bv[8];
                    TfyPack<__nv_bfloat16>::unpack(tfy_ld16(bias + n), bv);
#pragma unroll
                    for (int k = 0; k < 8; ++k) v[k] += bv[k];
                }
                const size_t idx = (size_t)row * G + n / 8;            // group index of the un-fused kernel
                uint32_t m_lo = 0, m_hi = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    bool on = true;
                    if (relu) { on = v[k] > 0.f; v[k] = on ? v[k] : 0.f; }
                    if (ep.drop_rate > 0.f) {
                        const bool keep = tfy_uniform(ep.seed, step, idx * 8 + k) >= ep.drop_rate;
                        v[k] = keep ? v[k] * keep_scale : 0.f;
                        on = on && keep;
                    }
                    if (k < 4) m_lo |= (on ? 1u : 0u) << (8 * k);
                    else m_hi |= (on ? 1u : 0u) << (8 * (k - 4));
                }
                tfy_st16(ep.y + (size_t)row * ep.ldy + n, TfyPack<__nv_bfloat16>::pack(v));
                if (ep.mask) *reinterpret_cast<uint2*>(ep.mask + (size_t)row * N + n) = make_uint2(m_lo, m_hi);
            }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (threadIdx.x == 0) {                                       // the CTA that finishes last re-arms both counters
            __threadfence();
            if (atomicAdd(cnt + 1, 1u) == gridDim.z - 1) {
                cnt[0] = 0u;
                cnt[1] = 0u;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
namespace {
// the operand maps are tfy_tensor_map_bf16_2d: one box is BK columns x GemmGeom::BOX_ROWS rows
static_assert(BK == 64 && BM == 128 && BN == 128, "tile shape must match the tensor-map box");

int sm_count() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return sms;
}

// Launches tfy_gemm_bf16_kernel<FM, FN> on (tiles_m, tiles_n, splits) tiles; the tensor maps are built here because
// their box depends on the split of the tile.
template <int FM, int FN>
int launch_gemm(const void* A, const void* B, __nv_bfloat16* C, float* C32, const __nv_bfloat16* bias, int M, int N,
                int K, int lda, int ldb, int ldc, int relu, int out_mode, int per, int splits, TfySplitKEpilogue ep,
                cudaStream_t s) {
    using Geom = GemmGeom<FM, FN>;
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(tfy_gemm_bf16_kernel<FM, FN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)Geom::SMEM) != cudaSuccess)
            return -5;
        attr_set = true;
    }
    CUtensorMap ma, mb;
    if (!tfy_tensor_map_bf16_2d(&ma, A, M, K, lda, Geom::BOX_ROWS) ||
        !tfy_tensor_map_bf16_2d(&mb, B, N, K, ldb, Geom::BOX_ROWS))
        return -6;
    const dim3 grid(((M + BM - 1) / BM) * FM, ((N + BN - 1) / BN) * FN, splits);
    tfy_launch_pdl((tfy_gemm_bf16_kernel<FM, FN>), grid, dim3(FM, FN, 1), dim3(GEMM_THREADS), Geom::SMEM, s, ma, mb, C,
                   C32, bias, M, N, K, ldc, relu, out_mode, per, ep);
    return (int)cudaGetLastError();
}
}  // namespace

__global__ void __launch_bounds__(256) tfy_splitk_sum_f32_kernel(const float* __restrict__ slabs, float* __restrict__ out,
                                                                int splits, size_t slab, size_t n4) {
    tfy_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = __ldcg(reinterpret_cast<const float4*>(slabs) + i);
#pragma unroll 8
        for (int z = 1; z < splits; ++z) {
            const float4 b = __ldcg(reinterpret_cast<const float4*>(slabs + (size_t)z * slab) + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        reinterpret_cast<float4*>(out)[i] = a;
    }
}

extern "C" {

// debug: device buffer of 16 x int64 per CTA receiving the event timeline of the next launches (nullptr = off)
int tfy_gemm_set_timeline(long long* buf) { return (int)cudaMemcpyToSymbol(g_timeline, &buf, sizeof(buf)); }

// Number of K-slices (= workspace slabs) tfy_gemm_bf16 / tfy_gemm_bf16_splitk_fused run for a requested split_k.
int tfy_gemm_bf16_splitk_slabs(int K, int split_k) {
    const int k_tiles = (K + BK - 1) / BK;
    if (split_k < 1) split_k = 1;
    if (split_k > k_tiles) split_k = k_tiles;
    if (split_k < 1) return 1;
    const int per = (k_tiles + split_k - 1) / split_k;
    return (k_tiles + per - 1) / per;
}

// out[i] = sum over z in order of slabs[z * slab + i], i < n (n % 4 == 0, 16-byte aligned): the split-K reduction.
int tfy_splitk_sum_f32(const float* slabs, float* out, int splits, size_t slab, size_t n, cudaStream_t s) {
    if (splits < 1 || (n & 3) || (slab & 3) || (((uintptr_t)slabs | (uintptr_t)out) & 15)) return -2;
    const size_t n4 = n / 4;
    int grid = (int)((n4 + 255) / 256);
    if (grid > TFY_NUM_SMS * 4) grid = TFY_NUM_SMS * 4;
    if (grid < 1) grid = 1;
    tfy_launch_pdl(tfy_splitk_sum_f32_kernel, dim3(grid), dim3(256), 0, s, slabs, out, splits, slab, n4);
    return (int)cudaGetLastError();
}

// C[M,N] (bf16, ld ldc) = act(A[M,K] (ld lda) . B[N,K]^T (ld ldb) + bias[N]);  B may be a peer (NVLink) pointer.
// split_k > 1 (or C == nullptr): C32 is a workspace of tfy_gemm_bf16_splitk_slabs(K, split_k) x M x ldc floats; slab z
// (C32 + z * M * ldc) receives the partial product of K-slice z, to be summed in slab order (tfy_splitk_sum_f32,
// tfy_bias_act_drop_fwd_f32).
// Requirements: K % 8 == 0, lda % 8 == 0, ldb % 8 == 0 (-2), 16-byte aligned A, B, and C (when ldc % 8 == 0) or C32
// (when ldc % 4 == 0) as soon as N >= 16 (-3).
int tfy_gemm_bf16(const void* A, const void* B, void* C, float* C32, const void* bias, int M, int N, int K, int lda,
                  int ldb, int ldc, int relu, int split_k, cudaStream_t s) {
    if ((K & 7) || (lda & 7) || (ldb & 7)) return -2;
    if (((uintptr_t)A & 15) || ((uintptr_t)B & 15)) return -3;
    if (!tfy_tensor_map_encoder()) return -4;
    const int k_tiles = (K + BK - 1) / BK;
    if (split_k < 1) split_k = 1;
    if (split_k > k_tiles) split_k = k_tiles;
    const int per = (k_tiles + split_k - 1) / split_k;
    split_k = (k_tiles + per - 1) / per;
    const int out_mode = (split_k > 1 || (C == nullptr && C32 != nullptr)) ? 1 : 0;
    if (out_mode == 1 && C32 == nullptr) return -7;
    // the epilogue stores 16 bytes at a time (8 bf16 / 4 floats) whenever the row pitch allows it and a row has 16 columns
    if (N >= 16 && (out_mode == 0 ? ((ldc & 7) == 0 && ((uintptr_t)C & 15)) : ((ldc & 3) == 0 && ((uintptr_t)C32 & 15))))
        return -3;
    // slabs of a grid that leaves SMs idle: share each tile among the CTAs of a cluster, as many as still fit one wave
    const int ctas = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * split_k;
    const int sub = out_mode == 1 ? (4 * ctas <= sm_count() ? 4 : 2 * ctas <= sm_count() ? 2 : 1) : 1;
    const TfySplitKEpilogue ep{};
    if (sub == 4)
        return launch_gemm<2, 2>(A, B, nullptr, C32, nullptr, M, N, K, lda, ldb, ldc, 0, 1, per, split_k, ep, s);
    if (sub == 2)
        return launch_gemm<2, 1>(A, B, nullptr, C32, nullptr, M, N, K, lda, ldb, ldc, 0, 1, per, split_k, ep, s);
    return launch_gemm<1, 1>(A, B, (__nv_bfloat16*)C, C32, (const __nv_bfloat16*)bias, M, N, K, lda, ldb, ldc, relu,
                             out_mode, per, split_k, ep, s);
}

// Split-K GEMM with the fused epilogue: y[M,N] (bf16) = dropout(act(A . B^T + bias)), mask[M,N] (optional bytes).
// acc32: fp32 scratch of tfy_gemm_bf16_splitk_slabs(K, split_k) x M x N floats (slabs of row pitch N); counters: two uint32 per
// 128x128 output tile, zero on entry, left zero.  N % 8 == 0 (-2); A, B, y, acc32 and bias 16-byte aligned, mask 8-byte
// aligned (-3).  The K-slice CTAs of a tile meet on a counter, so the
// whole grid must be co-resident: returns -8 when tiles x split_k exceeds the SM count (use the two-launch path).
int tfy_gemm_bf16_splitk_fused(const void* A, const void* B, float* acc32, uint32_t* counters, const void* bias, void* y,
                               void* mask, int M, int N, int K, int lda, int ldb, int relu, float drop_rate, uint32_t seed,
                               const TfyOptHyper* hp, int split_k, cudaStream_t s) {
    if ((K & 7) || (lda & 7) || (ldb & 7) || (N & 7)) return -2;
    if (((uintptr_t)A & 15) || ((uintptr_t)B & 15) || ((uintptr_t)y & 15)) return -3;
    // the epilogue reads acc32 and bias 16 bytes at a time and writes the mask 8 bytes at a time
    if (((uintptr_t)acc32 & 15) || ((uintptr_t)bias & 15) || ((uintptr_t)mask & 7)) return -3;
    if (!tfy_tensor_map_encoder()) return -4;
    const int k_tiles = (K + BK - 1) / BK;
    if (split_k < 1) split_k = 1;
    if (split_k > k_tiles) split_k = k_tiles;
    const int per = (k_tiles + split_k - 1) / split_k;
    split_k = (k_tiles + per - 1) / per;
    TfySplitKEpilogue ep;
    ep.counters = counters; ep.y = (__nv_bfloat16*)y; ep.mask = (uint8_t*)mask; ep.hp = hp;
    ep.drop_rate = drop_rate; ep.seed = seed; ep.ldy = N;
    if (((M + BM - 1) / BM) * ((N + BN - 1) / BN) * split_k > sm_count()) return -8;
    return launch_gemm<1, 1>(A, B, nullptr, acc32, (const __nv_bfloat16*)bias, M, N, K, lda, ldb, N, relu, 2, per,
                             split_k, ep, s);
}

}  // extern "C"
