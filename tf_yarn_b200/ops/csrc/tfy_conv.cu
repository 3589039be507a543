// Hopper (wgmma) implicit-GEMM 3x3 convolution kernels (C_in = 32 -> C_out = 64, stride 1, VALID) for sm_90a:
// the second convolution of the MNIST-CNN, forward (fused with bias + ReLU + 2x2 max-pool + dropout),
// data gradient (fused with the ReLU gate of the previous layer) and weight gradient.
//
// Shared-memory operand format (all three kernels).  A work item is an 8 x 8 pixel patch of an image
// PAIR; TMA stores the (haloed) patch as
//        [h][image n][w][all channels of the pixel]         one pixel = one 64- or 128-byte row,
// with the 64B / 128B hardware swizzle.  The wgmma operand fetch XORs the 16-byte chunk index with ABSOLUTE
// shared-memory address bits (base_offset = 0), as TMA does when it writes the tile, whatever the descriptor's
// start address and stride between 8-row groups are.  So a filter tap (kh, kw) is just a
// different START ADDRESS into the same halo patch (+kh rows, +kw pixels) and the stride between 8-pixel
// groups is the 10-pixel halo row: the halo is loaded ONCE per patch by ONE TMA and the nine im2col views
// never materialise, neither in HBM nor in shared memory.  The pixel dimension is GEMM-M for fprop / dgrad
// (K-major A operand) and GEMM-K for wgrad (MN-major operands: the SAME bytes, other major-ness).
//
//   fprop : D[pix, o]  = sum_{t,c} a[pix + t, c] W[o, t, c]     M=128 N=64 K=9x32   (A: K-major, B: K-major)
//   dgrad : D[pix, c]  = sum_{t,o} dz[pix - t, o] W[o, t, c]    M=128 N=32 K=9x64   (A: K-major, B: MN-major)
//   wgrad : D[o, (t,c)] = sum_pix dz[pix, o] a[pix + t, c]      M=64  N=32 K=128/patch, 9 accumulators
//                                                               (A: MN-major, B: MN-major)
// Weights ([O][3][3][C] bf16) are loaded by one TMA as [tap][o][32 c] (64-byte rows): K-major for fprop
// and, read with the MN-major flag, the transposed operand dgrad needs -- no transpose kernel.
//
// All three are persistent (one CTA per SM walking the patch list) and warp-specialised: one TMA thread,
// one MMA warpgroup (wgmma M64 on each 64-row half of the tile, accumulators in registers), epilogue warps
// overlapped with the next patch through a double-buffered fp32 accumulator tile in shared memory.
//
// Operand layout: whole-pixel rows (64/128 B) + swizzle, so a patch is 200 TMA rows instead of the
// 800-1600 16-byte rows of an un-swizzled [pixel][16 B] layout.
#include "tfy_common.cuh"
#include "tfy_fused_step.cuh"
#include "tfy_tma.cuh"
#include "tfy_wgmma.cuh"

namespace {

constexpr int CIN = 32, COUT = 64, TAPS = 9;
constexpr int HALO = 10;                               // 8 + 2
constexpr int A_PIX_B = CIN * 2;                       // 64  : one input pixel  (SWIZZLE_64B rows)
constexpr int Z_PIX_B = COUT * 2;                      // 128 : one output pixel (SWIZZLE_128B rows)
constexpr int A_ROW_B = HALO * A_PIX_B;                // 640  : one (h, n) row of an input halo patch
constexpr int Z_ROW_B = HALO * Z_PIX_B;                // 1280 : one (h, n) row of an output halo patch
constexpr int A_HALO_B = HALO * 2 * A_ROW_B;           // 12800
constexpr int A_HALO_PAD = 13312;                      // stage stride: keeps every TMA destination 1024-aligned
constexpr int Z_HALO_B = HALO * 2 * Z_ROW_B;           // 25600 (= 25 x 1024)
constexpr int Z_PATCH_B = 8 * 2 * 8 * Z_PIX_B;         // 16384
constexpr int W_TAP_B = COUT * A_PIX_B;                // 4096 : [64 o][32 c]
constexpr int W_BYTES = TAPS * W_TAP_B;                // 36864

// double-buffered fp32 accumulator tiles [2][128 rows][N + 4] (the pad keeps row-per-thread reads conflict-free)
constexpr int FP_ACC_LD = COUT + 4, DG_ACC_LD = CIN + 4;
// 416 threads: the launch bound leaves the MMA warpgroup room for both halves' accumulators (2 x 32 fp32) in flight
constexpr int FP_STAGES = 3, FP_EPI_WARPS = 8, FP_THREADS = (FP_EPI_WARPS + 4 + 1) * 32;    // 416
constexpr size_t FP_SMEM = (size_t)FP_STAGES * A_HALO_PAD + W_BYTES + 2 * 128 * FP_ACC_LD * 4 + 1024 + 256;
// 512 threads: + 4 un-pool producer warps, + 3 warps that reduce deferred weight-gradient partials with the TMA warp
constexpr int DG_STAGES = 3, DG_EPI_WARPS = 4, DG_RED_WARPS = 4;
constexpr int DG_THREADS = (DG_EPI_WARPS + 4 + 1 + 4 + DG_RED_WARPS - 1) * 32;
// + the part sums of the deferred weight-gradient reduction (c_wg_reduce): 37 float4 outputs x 16 parts per CTA at
// batch 128 fit in one chunk
constexpr int DG_RED_B = 32 * 1024;
constexpr size_t DG_SMEM =
    (size_t)DG_STAGES * Z_HALO_B + W_BYTES + 2 * 128 * DG_ACC_LD * 4 + DG_RED_B + 1024 + 256;
static_assert(DG_SMEM <= 232448, "dgrad shared memory exceeds the sm_90 opt-in limit per block");
// The ring holds every patch of a CTA at batch 128 (5 of them), so all of them load during the prologue; the MMA
// warpgroup still takes patches WG_GROUP at a time (one wgmma chain per tap and group), which fixes the fp32
// summation order of the partial tile whatever the ring depth.
constexpr int WG_RING = 5, WG_GROUP = 4, WG_STAGE_B = Z_PATCH_B + A_HALO_PAD;              // 29696
constexpr int WG_WORK_WARPS = 16, WG_THREADS = (WG_WORK_WARPS + 4 + 1) * 32;               // 672
constexpr int WG_OUT = COUT * TAPS * CIN;                                                 // 18432
constexpr int WG_PART = WG_OUT + COUT;                 // per-CTA partial: dW tile + db (un-pool variant)
constexpr int WG_ACC_B = TAPS * 16 * 128 * 4;          // 9 taps x 64 x 32 fp32 in fragment order [tap][16][128 threads]
constexpr size_t WG_SMEM = (size_t)WG_RING * WG_STAGE_B + 1024 + 512 + WG_WORK_WARPS * COUT * 4 + WG_ACC_B;
static_assert(WG_SMEM <= 232448, "wgrad shared memory exceeds the sm_90 opt-in limit per block");
static_assert(2 * WG_RING * 8 <= 512, "wgrad ring barriers overflow their shared-memory slot");

constexpr uint32_t SW128 = TFY_WG_SW128, SW64 = TFY_WG_SW64;

// Optional per-CTA event timeline (tests/gpu/conv_check.py): 16 slots of SM-clock deltas per CTA.
__device__ long long* c_timeline = nullptr;
#define C_MARK(k)                                                                  \
    do {                                                                           \
        if (c_tl) c_tl[(size_t)blockIdx.x * 16 + (k)] = clock64() - c_t0;          \
    } while (0)
#define C_TIMELINE_BEGIN()                 \
    long long* const c_tl = c_timeline;    \
    const long long c_t0 = clock64();      \
    if (c_tl && threadIdx.x == 0) {        \
        unsigned long long ns;             \
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns)); \
        c_tl[(size_t)blockIdx.x * 16] = (long long)ns;          \
    }

#include "tfy_conv_index.cuh"

// Un-pooling producer task: the gradient dp of ONE pooled pixel (8 channels of group g) becomes the 2x2 window
// of dz rows it came from, written straight into a swizzled [pixel rows][128 B] operand tile:
//   dz[2py+dy, 2px+dx, o] = (code[o] & 4) && (code[o] & 3) == dy*2+dx ? dp[o] * scale : 0
// (code byte of the forward kernel: argmax position + gate).  The fused pool/dropout/ReLU backward never
// writes the 4x larger dz tensor to memory.  row0 = tile row of the window's top-left pixel, row_dy = rows per
// image row of the tile (2 images interleaved: 2 * pixels per row).  Returns the gated values for db.
struct CUnpoolIn {
    uint4 v;
    uint2 cd;
};
__device__ __forceinline__ CUnpoolIn c_unpool_load(const __nv_bfloat16* __restrict__ dp,
                                                   const uint8_t* __restrict__ code, bool valid, size_t pidx, int g) {
    CUnpoolIn in;
    in.v = make_uint4(0, 0, 0, 0);
    in.cd = make_uint2(0, 0);
    if (valid) {
        in.v = tfy_ld16(dp + pidx * COUT + g * 8);
        in.cd = *reinterpret_cast<const uint2*>(code + pidx * COUT + g * 8);
    }
    return in;
}
__device__ __forceinline__ void c_unpool_emit(uint8_t* tile, const CUnpoolIn& in, float scale, int g, int row0,
                                              int row_dy, float* gated) {
    float f[8];
    TfyPack<__nv_bfloat16>::unpack(in.v, f);
    uint32_t c[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        c[k] = ((k < 4 ? in.cd.x >> (8 * k) : in.cd.y >> (8 * (k - 4)))) & 0xffu;
        f[k] = (c[k] & 4u) ? f[k] * scale : 0.f;
        gated[k] = f[k];
    }
#pragma unroll
    for (int pos = 0; pos < 4; ++pos) {
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = ((c[k] & 3u) == (uint32_t)pos) ? f[k] : 0.f;
        const int row = row0 + (pos >> 1) * row_dy + (pos & 1);
        *reinterpret_cast<uint4*>(tile + (size_t)row * Z_PIX_B + ((uint32_t)(g ^ (row & 7)) << 4)) =
            TfyPack<__nv_bfloat16>::pack(o);
    }
}

// Deferred reduction of the weight gradient's per-CTA partials (DG_RED_WARPS warps, rt = 0 .. 32 DG_RED_WARPS - 1):
// float4 outputs [f0, f1) of the dW tile + db, each summed over the n_part partials in the order c_wg_slice gives the
// wgrad CTA that owns it, then converted to bf16.  As in that CTA, part p of an output sums partials p, p + parts, ...
// (8 loads in flight per thread); the part sums of the outputs are one task each for all reduction threads, so the
// ~70 KB a CTA reads are in flight at once, and go to buf (DG_RED_B bytes, `stride` per output) to be added in order.
__device__ __forceinline__ void c_wg_reduce(const float* __restrict__ partials, int n_part, int f0, int f1,
                                            __nv_bfloat16* __restrict__ dw, __nv_bfloat16* __restrict__ db,
                                            float4* buf, int rt) {
    constexpr int TOTAL4 = WG_PART / 4, STRIDE4 = WG_PART / 4, NT = DG_RED_WARPS * 32;
    if (f0 >= f1) return;                                            // the same for every reduction thread
    const int per = c_wg_per(TOTAL4, n_part);
    auto parts_of = [&](int f) { return c_wg_slice(TOTAL4, n_part, f / per, WG_THREADS).parts; };
    // every owner but the last has the same slice length: the ends of [f0, f1) bound the part sums per output
    const int stride = max(min(parts_of(f0), n_part), min(parts_of(f1 - 1), n_part));
    const int chunk = DG_RED_B / (16 * stride);                     // float4 outputs per round
    const float4* src = reinterpret_cast<const float4*>(partials);
    for (int c0 = f0; c0 < f1; c0 += chunk) {
        const int cn = min(chunk, f1 - c0);
        for (int k = rt; k < cn * stride; k += NT) {
            const int j = k / stride, p = k - j * stride, parts = parts_of(c0 + j);
            if (p >= parts || p >= n_part) continue;
            const float4* col = src + c0 + j;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int q0 = p; q0 < n_part; q0 += 8 * parts) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (q0 + u * parts < n_part) v[u] = __ldcg(col + (size_t)(q0 + u * parts) * STRIDE4);
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (q0 + u * parts < n_part) { s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w; }
            }
            buf[k] = s;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(NT) : "memory");
        for (int j = rt; j < cn; j += NT) {
            const int parts = parts_of(c0 + j);
            const float4* ps = buf + j * stride;
            float4 tot = ps[0];
            for (int p = 1; p < parts && p < n_part; ++p) {
                tot.x += ps[p].x; tot.y += ps[p].y; tot.z += ps[p].z; tot.w += ps[p].w;
            }
            if (parts > n_part) { tot.x += 0.f; tot.y += 0.f; tot.z += 0.f; tot.w += 0.f; }   // the empty parts
            __nv_bfloat162 l2 = __floats2bfloat162_rn(tot.x, tot.y), h2 = __floats2bfloat162_rn(tot.z, tot.w);
            uint2 packed;
            packed.x = *reinterpret_cast<uint32_t*>(&l2);
            packed.y = *reinterpret_cast<uint32_t*>(&h2);
            const int e = (c0 + j) * 4;                              // outputs [0, WG_OUT) = dW, then db
            if (e < WG_OUT) *reinterpret_cast<uint2*>(dw + e) = packed;
            else *reinterpret_cast<uint2*>(db + (e - WG_OUT)) = packed;
        }
        asm volatile("bar.sync 1, %0;" ::"r"(NT) : "memory");       // buf is reused by the next round
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// forward: pooled = dropout(maxpool2x2(relu(conv(a, W) + bias))), code byte per pooled element
// (bits 0-1 = argmax position dy*2+dx inside the 2x2 window, bit 2 = gradient flows).
// warps 0..7 epilogue (row quadrant = warp & 3, 16-column slices warp >> 2 and (warp >> 2) + 2), warps 8..11 MMA,
// warp 12 TMA
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FP_THREADS, 1)
tfy_conv3x3_fprop_pool_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                              const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ pooled,
                              uint8_t* __restrict__ code, int H, int W, int tiles_x, int tiles_y, int n_patches,
                              float drop_rate, uint32_t seed, const TfyOptHyper* __restrict__ hp) {
    extern __shared__ uint8_t smem_raw[];
    C_TIMELINE_BEGIN();
    uint8_t* stages = tfy_align1024(smem_raw);                      // [3][10 h][2 n][10 w][64 B], 64B swizzle
    uint8_t* w_tile = stages + (size_t)FP_STAGES * A_HALO_PAD;    // [9][64 o][64 B], 64B swizzle
    float* acc_s = reinterpret_cast<float*>(w_tile + W_BYTES);    // [2][128][FP_ACC_LD]
    uint64_t* full = reinterpret_cast<uint64_t*>(acc_s + 2 * 128 * FP_ACC_LD);
    uint64_t* empty = full + FP_STAGES;
    uint64_t* tfull = empty + FP_STAGES;
    uint64_t* tempty = tfull + 2;
    uint64_t* wfull = tempty + 2;

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_a);
        tfy_prefetch_tensormap(&map_w);
        for (int s = 0; s < FP_STAGES; ++s) { tfy_mbar_init(&full[s], 1); tfy_mbar_init(&empty[s], 4); }
        for (int b = 0; b < 2; ++b) { tfy_mbar_init(&tfull[b], 128); tfy_mbar_init(&tempty[b], FP_EPI_WARPS * 32); }
        tfy_mbar_init(wfull, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();                      // upstream grids complete; our dependents may start launching
    if (threadIdx.x == 0) C_MARK(1);
    const int my_patches = ((int)blockIdx.x < n_patches) ? (n_patches - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (warp == FP_EPI_WARPS + 4) {
        // ---------------- TMA producer
        if (tfy_elect_one()) {
            tfy_mbar_expect_tx(wfull, W_BYTES);
            tfy_tma_load_3d(&map_w, wfull, w_tile, 0, 0, 0);
            CPatchIter it(tiles_x, tiles_y);
            for (int i = 0; i < my_patches; ++i, it.next()) {
                const int s = i % FP_STAGES;
                if (i >= FP_STAGES) tfy_mbar_wait(&empty[s], ((i / FP_STAGES) - 1) & 1);
                tfy_mbar_expect_tx(&full[s], A_HALO_B);
                tfy_tma_load_4d(&map_a, &full[s], stages + (size_t)s * A_HALO_PAD, 0, it.tx * 8, it.bz * 2, it.ty * 8);
                if (i == 0) C_MARK(2);
            }
        }
    } else if (warp >= FP_EPI_WARPS) {
        // ---------------- MMA warpgroup: the two 64-pixel halves of the patch (8 (h, n) rows of the halo apart) are
        // two chains, each its own commit group; half 0's accumulators are stored while the tensor core runs half 1.
        // Each chain is fully unrolled and keeps the (tap, k-step) order, so no wgmma waits on another one's
        // registers and the result is the same bit for bit as one interleaved chain.
        const uint32_t w0 = tfy_smem_u32(w_tile);
        float acc[2][COUT / 2];
        auto issue = [&](float (&d)[COUT / 2], uint32_t a0) {
            tfy_wg_fence();
#pragma unroll
            for (int t = 0; t < TAPS; ++t) {
                const int kh = t / 3, kw = t - kh * 3;
#pragma unroll
                for (int ks = 0; ks < CIN / 16; ++ks) {
                    // B rows = output channels (64 B apart), 8-row groups 512 B apart
                    const uint64_t bdesc = tfy_wg_desc(w0 + t * W_TAP_B + ks * 32, 16, 8 * A_PIX_B, SW64);
                    // A rows = pixels: 8 consecutive w (64 B apart), next group = next (h, n) row of the halo
                    const uint64_t adesc =
                        tfy_wg_desc(a0 + kh * 2 * A_ROW_B + kw * A_PIX_B + ks * 32, 16, A_ROW_B, SW64);
                    tfy_wgmma_m64n64<0, 0>(d, adesc, bdesc, (t > 0 || ks > 0) ? 1u : 0u);
                }
            }
            tfy_wg_commit();
        };
        tfy_mbar_wait(wfull, 0);
        for (int i = 0; i < my_patches; ++i) {
            const int s = i % FP_STAGES, b = i & 1;
            float* tile = acc_s + b * 128 * FP_ACC_LD;
            tfy_mbar_wait(&full[s], (i / FP_STAGES) & 1);
            if (i == 0 && threadIdx.x == FP_EPI_WARPS * 32) C_MARK(4);
            const uint32_t a0 = tfy_smem_u32(stages + (size_t)s * A_HALO_PAD);
            issue(acc[0], a0);
            issue(acc[1], a0 + 4 * 2 * A_ROW_B);
            if (i >= 2) tfy_mbar_wait(&tempty[b], ((i >> 1) - 1) & 1);
            tfy_wg_wait<1>();                                     // half 0 is complete
            tfy_wg_store_rows<COUT>(tile, FP_ACC_LD, acc[0], 0);
            tfy_wg_wait<0>();
            if (lane == 0) tfy_mbar_arrive(&empty[s]);
            tfy_wg_store_rows<COUT>(tile, FP_ACC_LD, acc[1], 64);
            tfy_mbar_arrive(&tfull[b]);
            if (threadIdx.x == FP_EPI_WARPS * 32) { if (i == 0) C_MARK(5); if (i == my_patches - 1) C_MARK(11); }
        }
    } else {
        // ---------------- epilogue: accumulator row r = (h, n, w) = (r/16, (r/8)&1, r%8) is row r of the staged tile
        const int quad = warp & 3, cq0 = warp >> 2;                // column slices cq0 and cq0 + 2
        const int r = quad * 32 + lane;
        const int h = r >> 4, n = (r >> 3) & 1, w = r & 7;
        const int dx = lane & 1, dy = (lane >> 4) & 1;            // position inside the 2x2 pooling window
        const uint32_t tag = (uint32_t)(dy * 2 + dx);
        const int OH = H - 2, OW = W - 2, PH = OH / 2, PW = OW / 2;
        const uint32_t step = hp ? (uint32_t)hp->step : 0u;
        // dropout decisions come 4 to a hash (one byte each): the rate is quantised to 1/256
        const uint32_t thr = drop_rate > 0.f ? (uint32_t)(drop_rate * 256.f + 0.5f) : 0u;
        const float keep_scale = 256.f / (256.f - (float)thr);
        const uint32_t salt = seed ^ tfy_hash32(step * 0x9E3779B9U + 0x85ebca6bU);
        // after the two exchanges below lane (dy, dx) owns columns [8 dx + 4 dy, +4) of each of the warp's slices
        float bv[2][4];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint2 braw = *reinterpret_cast<const uint2*>(bias + (cq0 + 2 * k) * 16 + dx * 8 + dy * 4);
            bv[k][0] = tfy_bf16lo(braw.x); bv[k][1] = tfy_bf16hi(braw.x);
            bv[k][2] = tfy_bf16lo(braw.y); bv[k][3] = tfy_bf16hi(braw.y);
        }
        CPatchIter it(tiles_x, tiles_y);
        for (int i = 0; i < my_patches; ++i, it.next()) {
            const int b = i & 1;
            tfy_mbar_wait(&tfull[b], (i >> 1) & 1);
            if (threadIdx.x == 0) { if (i == 0) C_MARK(6); if (i == my_patches - 1) C_MARK(8); }
            uint32_t accs[2][16];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float* src = acc_s + (size_t)(b * 128 + r) * FP_ACC_LD + (cq0 + 2 * k) * 16;
#pragma unroll
                for (int j = 0; j < 16; j += 4)
                    *reinterpret_cast<uint4*>(accs[k] + j) = *reinterpret_cast<const uint4*>(src + j);
            }
            tfy_mbar_arrive(&tempty[b]);                             // the MMA warps may overwrite this buffer now
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int col = (cq0 + 2 * k) * 16 + dx * 8 + dy * 4;
                const uint32_t prow = (uint32_t)((((it.bz * 2 + n) * PH + ((it.ty * 8 + h) >> 1)) * PW +
                                                  ((it.tx * 8 + w) >> 1)) * COUT + col);
                const uint32_t* acc = accs[k];
                // tag every value with its window position in the 2 low mantissa bits, then reduce-scatter the
                // max over the window (lane ^ 1: other column, lane ^ 16: other row)
                float v[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] = __uint_as_float((acc[j] & ~3u) | tag);
                float m8[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float send = dx ? v[j] : v[8 + j];
                    const float keep = dx ? v[8 + j] : v[j];
                    m8[j] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, 1));
                }
                float m4[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float send = dy ? m8[j] : m8[4 + j];
                    const float keep = dy ? m8[4 + j] : m8[j];
                    m4[j] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, 16));
                }
                const uint32_t rnd =
                    thr ? tfy_hash32(salt ^ tfy_hash32((prow >> 2) * 0xC2B2AE35U + 0x27d4eb2fU)) : 0xffffffffu;
                float o[4];
                uint32_t codes = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t pos = __float_as_uint(m4[j]) & 3u;
                    float x = m4[j] + bv[k][j];
                    const bool on = x > 0.f && ((rnd >> (8 * j)) & 0xffu) >= thr;
                    x = on ? x * keep_scale : 0.f;
                    o[j] = x;
                    codes |= (pos | (on ? 4u : 0u)) << (8 * j);
                }
                __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], o[3]);
                uint2 packed;
                packed.x = *reinterpret_cast<uint32_t*>(&lo);
                packed.y = *reinterpret_cast<uint32_t*>(&hi);
                *reinterpret_cast<uint2*>(pooled + prow) = packed;
                *reinterpret_cast<uint32_t*>(code + prow) = codes;
                if (threadIdx.x == 0) { if (i == 0) C_MARK(7); if (i == my_patches - 1) C_MARK(9); }
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) C_MARK(10);
}

// ------------------------------------------------------------------------------------------------
// data gradient: dx[b, y, x, c] = sum_{kh,kw,o} dz[b, y-kh, x-kw, o] W[o, kh, kw, c], optionally gated by
// the previous layer's ReLU (gate = that layer's output: dx is zeroed where gate <= 0).
// dz: [B, H-2, W-2, 64]; dx: [B, H, W, 32].  warps 0..3 epilogue, warps 4..7 MMA, warp 8 TMA (zero-fills the halo)
// ------------------------------------------------------------------------------------------------
// UNPOOL: the A operand is not loaded from a materialised dz but rebuilt by warps 9..12 from the pooled gradient
// dp [B, (H-2)/2, (W-2)/2, 64] and the forward kernel's code bytes (c_unpool_task).  With `partials` (UNPOOL only)
// warp 8, idle once it has issued the weight load, and warps 13..15 reduce a slice of the n_part weight-gradient
// partials a deferred tfy_conv3x3_wgrad_kernel<true> left behind into bf16 dw / db (c_wg_reduce), behind the main
// loop.
template <bool UNPOOL>
__global__ void __launch_bounds__(DG_THREADS, 1)
tfy_conv3x3_dgrad_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_w,
                         const __nv_bfloat16* __restrict__ gate, __nv_bfloat16* __restrict__ dx, int H, int W,
                         int tiles_x, int tiles_y, int n_patches, const __nv_bfloat16* __restrict__ dp,
                         const uint8_t* __restrict__ code, float scale, const float* __restrict__ partials,
                         int n_part, __nv_bfloat16* __restrict__ dw, __nv_bfloat16* __restrict__ db) {
    extern __shared__ uint8_t smem_raw[];
    C_TIMELINE_BEGIN();
    uint8_t* stages = tfy_align1024(smem_raw);                      // [3][10 h][2 n][10 w][128 B], 128B swizzle
    uint8_t* w_tile = stages + (size_t)DG_STAGES * Z_HALO_B;      // [9][64 o][64 B], 64B swizzle
    float* acc_s = reinterpret_cast<float*>(w_tile + W_BYTES);    // [2][128][DG_ACC_LD]
    float4* red_buf = reinterpret_cast<float4*>(acc_s + 2 * 128 * DG_ACC_LD);   // DG_RED_B: part sums (c_wg_reduce)
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(red_buf) + DG_RED_B);
    uint64_t* empty = full + DG_STAGES;
    uint64_t* tfull = empty + DG_STAGES;
    uint64_t* tempty = tfull + 2;
    uint64_t* wfull = tempty + 2;

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    if (threadIdx.x == 0) {
        if (!UNPOOL) tfy_prefetch_tensormap(&map_dz);
        tfy_prefetch_tensormap(&map_w);
        for (int s = 0; s < DG_STAGES; ++s) { tfy_mbar_init(&full[s], UNPOOL ? 128 : 1); tfy_mbar_init(&empty[s], 4); }
        for (int b = 0; b < 2; ++b) { tfy_mbar_init(&tfull[b], 128); tfy_mbar_init(&tempty[b], DG_EPI_WARPS * 32); }
        tfy_mbar_init(wfull, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();                      // upstream grids complete; our dependents may start launching
    if (threadIdx.x == 0) C_MARK(1);
    const int my_patches = ((int)blockIdx.x < n_patches) ? (n_patches - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (warp == DG_EPI_WARPS + 4) {
        if (tfy_elect_one()) {
            tfy_mbar_expect_tx(wfull, W_BYTES);
            tfy_tma_load_3d(&map_w, wfull, w_tile, 0, 0, 0);
            CPatchIter it(tiles_x, tiles_y);
            for (int i = 0; !UNPOOL && i < my_patches; ++i, it.next()) {
                const int s = i % DG_STAGES;
                if (i >= DG_STAGES) tfy_mbar_wait(&empty[s], ((i / DG_STAGES) - 1) & 1);
                tfy_mbar_expect_tx(&full[s], Z_HALO_B);
                // halo origin (y0-2, x0-2) of the dz image: pixels outside it are zero-filled by TMA
                tfy_tma_load_4d(&map_dz, &full[s], stages + (size_t)s * Z_HALO_B, 0, it.tx * 8 - 2, it.bz * 2,
                                it.ty * 8 - 2);
                if (i == 0) C_MARK(2);
            }
        }
        __syncwarp();
    } else if (warp > DG_EPI_WARPS + 8) {
        // reduction warps (below)
    } else if (warp >= DG_EPI_WARPS && warp < DG_EPI_WARPS + 4) {
        // ---------------- MMA warpgroup: both 64-pixel halves of the patch (4 h rows of the halo apart)
        const uint32_t w0 = tfy_smem_u32(w_tile);
        tfy_mbar_wait(wfull, 0);
        for (int i = 0; i < my_patches; ++i) {
            const int s = i % DG_STAGES, b = i & 1;
            tfy_mbar_wait(&full[s], (i / DG_STAGES) & 1);
            if (UNPOOL) tfy_fence_proxy_async();
            if (i == 0 && threadIdx.x == DG_EPI_WARPS * 32) C_MARK(4);
            const uint32_t a0 = tfy_smem_u32(stages + (size_t)s * Z_HALO_B);
            float acc[2][CIN / 2];
            tfy_wg_fence();
#pragma unroll 1
            for (int t = 0; t < TAPS; ++t) {
                const int kh = t / 3, kw = t - kh * 3;
#pragma unroll
                for (int ks = 0; ks < COUT / 16; ++ks) {
                    // W tap [o][32 c]: K = o (rows of 64 B, 8-row groups 512 B apart), N = c inside the row (MN-major)
                    const uint64_t bdesc = tfy_wg_desc(w0 + t * W_TAP_B + ks * 16 * A_PIX_B, 16, 8 * A_PIX_B, SW64);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        // dz[y-kh, x-kw] sits (2-kh, 2-kw) into the halo patch; rows = pixels of 128 B
                        const uint64_t adesc = tfy_wg_desc(
                            a0 + (2 - kh + 4 * h) * 2 * Z_ROW_B + (2 - kw) * Z_PIX_B + ks * 32, 16, Z_ROW_B, SW128);
                        tfy_wgmma_m64n32<0, 1>(acc[h], adesc, bdesc, (t > 0 || ks > 0) ? 1u : 0u);
                    }
                }
            }
            tfy_wg_commit();
            tfy_wg_wait<0>();
            if (lane == 0) tfy_mbar_arrive(&empty[s]);
            if (i >= 2) tfy_mbar_wait(&tempty[b], ((i >> 1) - 1) & 1);
            tfy_wg_store_rows<CIN>(acc_s + b * 128 * DG_ACC_LD, DG_ACC_LD, acc[0], 0);
            tfy_wg_store_rows<CIN>(acc_s + b * 128 * DG_ACC_LD, DG_ACC_LD, acc[1], 64);
            tfy_mbar_arrive(&tfull[b]);
            if (threadIdx.x == DG_EPI_WARPS * 32) { if (i == 0) C_MARK(5); if (i == my_patches - 1) C_MARK(11); }
        }
    } else if (warp > DG_EPI_WARPS + 4) {
        // ---------------- un-pool producers (UNPOOL only): 5 x 5 pooled pixels x 2 images x 8 channel groups
        if (UNPOOL) {
            const int ptid = threadIdx.x - (DG_EPI_WARPS + 5) * 32;           // 0..127
            const int PH = (H - 2) / 2, PWp = (W - 2) / 2;
            CPatchIter it(tiles_x, tiles_y);
            for (int i = 0; i < my_patches; ++i, it.next()) {
                const int s = i % DG_STAGES;
                if (i >= DG_STAGES) tfy_mbar_wait(&empty[s], ((i / DG_STAGES) - 1) & 1);
                uint8_t* tile = stages + (size_t)s * Z_HALO_B;
                // 400 tasks per patch, 4 slots per thread: all loads are issued before the first is consumed
                // (one L2 round trip per patch instead of four)
                CUnpoolIn in[4];
                int row0[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = ptid + u * 128;
                    const int g = t & 7, n = (t >> 3) & 1, pp = min(t >> 4, 24);
                    const int ppy = pp / 5, ppx = pp - ppy * 5;
                    const int py = it.ty * 4 - 1 + ppy, px = it.tx * 4 - 1 + ppx;
                    const bool valid = t < 400 && (unsigned)py < (unsigned)PH && (unsigned)px < (unsigned)PWp;
                    const size_t pidx = ((size_t)(it.bz * 2 + n) * PH + (valid ? py : 0)) * PWp + (valid ? px : 0);
                    in[u] = c_unpool_load(dp, code, valid, pidx, g);
                    row0[u] = (ppy * 2 * 2 + n) * HALO + ppx * 2;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = ptid + u * 128;
                    float gated[8];
                    if (t < 400) c_unpool_emit(tile, in[u], scale, t & 7, row0[u], 2 * HALO, gated);
                }
                tfy_fence_proxy_async();
                tfy_mbar_arrive(&full[s]);
            }
        }
    } else {
        const int quad = warp & 3;
        const int r = quad * 32 + lane;
        const int h = r >> 4, n = (r >> 3) & 1, w = r & 7;
        CPatchIter it(tiles_x, tiles_y);
        for (int i = 0; i < my_patches; ++i, it.next()) {
            const int b = i & 1;
            const int y = it.ty * 8 + h, x = it.tx * 8 + w;
            const bool valid = y < H && x < W;
            const size_t off = (((size_t)(it.bz * 2 + n) * H + y) * W + x) * CIN;
            uint4 g0, g1, g2, g3;
            if (gate && valid) {                                   // issued before the accumulator wait
                g0 = tfy_ld16(gate + off); g1 = tfy_ld16(gate + off + 8);
                g2 = tfy_ld16(gate + off + 16); g3 = tfy_ld16(gate + off + 24);
            }
            tfy_mbar_wait(&tfull[b], (i >> 1) & 1);
            if (threadIdx.x == 0) { if (i == 0) C_MARK(6); if (i == my_patches - 1) C_MARK(8); }
            uint32_t acc[2][16];
            const float* src = acc_s + (size_t)(b * 128 + r) * DG_ACC_LD;
#pragma unroll
            for (int j = 0; j < 32; j += 4) *reinterpret_cast<uint4*>(&acc[j >> 4][j & 15]) = *reinterpret_cast<const uint4*>(src + j);
            tfy_mbar_arrive(&tempty[b]);
            if (valid) {
                float v[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(acc[j >> 4][j & 15]);
                if (gate) {
                    float g[32];
                    TfyPack<__nv_bfloat16>::unpack(g0, g);
                    TfyPack<__nv_bfloat16>::unpack(g1, g + 8);
                    TfyPack<__nv_bfloat16>::unpack(g2, g + 16);
                    TfyPack<__nv_bfloat16>::unpack(g3, g + 24);
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = g[j] > 0.f ? v[j] : 0.f;
                }
#pragma unroll
                for (int j = 0; j < 32; j += 8) tfy_st16(dx + off + j, TfyPack<__nv_bfloat16>::pack(v + j));
            }
        }
    }
    if (UNPOOL && partials != nullptr && (warp == DG_EPI_WARPS + 4 || warp > DG_EPI_WARPS + 8)) {
        const int rt = warp == DG_EPI_WARPS + 4 ? lane : (warp - (DG_EPI_WARPS + 8)) * 32 + lane;
        constexpr int TOTAL4 = WG_PART / 4;
        const int per = (TOTAL4 + (int)gridDim.x - 1) / (int)gridDim.x;
        const int f0 = min((int)blockIdx.x * per, TOTAL4), f1 = min(f0 + per, TOTAL4);
        c_wg_reduce(partials, n_part, f0, f1, dw, db, red_buf, rt);
        if (rt == 0) C_MARK(3);
    }
    __syncthreads();
    if (threadIdx.x == 0) C_MARK(10);
}

// ------------------------------------------------------------------------------------------------
// weight gradient: dW[o, t, c] = sum_{b,y,x} dz[b, y, x, o] a[b, y+kh, x+kw, c].  The pixel patches are the
// GEMM K dimension: every CTA accumulates nine 64x32 tiles (one per tap) over its share of the patches -- each
// group of staged patches is one wgmma chain per tap in registers, added into fp32 tiles in shared memory --
// and writes the fp32 partial tile to `partials[blockIdx.x]` (L2 resident); after a grid-wide arrive/release it
// reduces a slice of the 18432 outputs over all partials in a fixed order (deterministic, no atomics) and writes
// bf16 dW.
// warps 0..15 un-pool producers (UNPOOL) + final reduction, warps 16..19 MMA + partial tile, warp 20 TMA.
// sync: 1024 uint32, zero-initialised once (generation + two levels of arrival counters, see below).  sync ==
// nullptr (UNPOOL only): no grid barrier and no reduction -- the compute CTAs store their partials and exit, and
// the un-pool dgrad kernel that follows reduces them (tfy_conv3x3_dgrad_kernel<true>, c_wg_reduce).
// ------------------------------------------------------------------------------------------------
// UNPOOL: dz tiles are rebuilt by warps 0..3 from the pooled gradient dp and the forward kernel's code bytes
// (c_unpool_task) and the bias gradient db = sum of the gated dp rides along as 64 more outputs.
template <bool UNPOOL>
__global__ void __launch_bounds__(WG_THREADS, 1)
tfy_conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap map_dz, const __grid_constant__ CUtensorMap map_a,
                         float* __restrict__ partials, __nv_bfloat16* __restrict__ dw, uint32_t* __restrict__ sync,
                         int tiles_x, int tiles_y, int n_patches, const __nv_bfloat16* __restrict__ dp,
                         const uint8_t* __restrict__ code, float scale, __nv_bfloat16* __restrict__ db, int PH,
                         int PWp, const __grid_constant__ TfyOverlapStep ov) {
    // The last ov.n_cta CTAs of the grid are COMMUNICATION CTAs: they run the fused reduce-scatter -> optimizer ->
    // all-gather step of the parameters whose gradients were final before this kernel started (tfy_fused_step.cuh)
    // over NVLink while the compute CTAs below run the weight gradient.  One CTA per SM and grid <= #SMs, so both
    // roles are co-resident by construction.
    const int n_cmp = (int)gridDim.x - ov.n_cta;                     // compute CTAs (share patches, grid barrier)
    if ((int)blockIdx.x >= n_cmp) {
        extern __shared__ uint8_t smem_role[];
        tfy_pdl_sync();
        tfy_overlap_role<WG_THREADS>(ov, (int)blockIdx.x - n_cmp, tfy_align1024(smem_role));
        return;
    }
    extern __shared__ uint8_t smem_raw[];
    C_TIMELINE_BEGIN();
    uint8_t* stages = tfy_align1024(smem_raw);    // [5] { dz [8 h][2 n][8 w][128 B] sw128 ; a [10 h][2 n][10 w][64 B] sw64 }
    uint64_t* full = reinterpret_cast<uint64_t*>(stages + (size_t)WG_RING * WG_STAGE_B);
    uint64_t* empty = full + WG_RING;
    float* s_db = reinterpret_cast<float*>(empty + WG_RING);        // [16 warps][64] bias-gradient partials (UNPOOL)
    float* acc_s = s_db + WG_WORK_WARPS * COUT;                      // [9 taps][16][128 threads] fp32

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    if (threadIdx.x == 0) {
        if (!UNPOOL) tfy_prefetch_tensormap(&map_dz);
        tfy_prefetch_tensormap(&map_a);
        for (int s = 0; s < WG_RING; ++s) { tfy_mbar_init(&full[s], UNPOOL ? 257 : 1); tfy_mbar_init(&empty[s], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    tfy_pdl_sync();                      // upstream grids complete; our dependents may start launching
    if (threadIdx.x == 0) C_MARK(1);
    const uint32_t gen0 = (threadIdx.x == 0 && sync) ? *reinterpret_cast<volatile uint32_t*>(sync) : 0u;
    const int my_patches = ((int)blockIdx.x < n_patches) ? (n_patches - 1 - (int)blockIdx.x) / n_cmp + 1 : 0;

    if (warp == WG_WORK_WARPS + 4) {
        if (tfy_elect_one()) {
            CPatchIter it(tiles_x, tiles_y, n_cmp);
            for (int i = 0; i < my_patches; ++i, it.next()) {
                const int s = i % WG_RING;
                if (i >= WG_RING) tfy_mbar_wait(&empty[s], ((i / WG_RING) - 1) & 1);
                uint8_t* st = stages + (size_t)s * WG_STAGE_B;
                tfy_mbar_expect_tx(&full[s], (UNPOOL ? 0 : Z_PATCH_B) + A_HALO_B);
                if (!UNPOOL) tfy_tma_load_4d(&map_dz, &full[s], st, 0, it.tx * 8, it.bz * 2, it.ty * 8);
                tfy_tma_load_4d(&map_a, &full[s], st + Z_PATCH_B, 0, it.tx * 8, it.bz * 2, it.ty * 8);
                if (i == 0) C_MARK(2);
            }
        }
    } else if (warp >= WG_WORK_WARPS) {
        // Patches are taken WG_GROUP at a time; per group and tap, one wgmma chain over the group's pixels in
        // registers, then added into the tap's fp32 tile (fragment order: thread t owns words [tap][i][t]).
        // Patch i sits in ring stage i % WG_RING.
        const int tid = (int)threadIdx.x - WG_WORK_WARPS * 32;
        float* mine = acc_s + tid;
        for (int i = 0; i < TAPS * 16; ++i) mine[i * 128] = 0.f;
        const int n_groups = (my_patches + WG_GROUP - 1) / WG_GROUP;
        for (int g = 0; g < n_groups; ++g) {
            const int i0 = g * WG_GROUP, cnt = min(WG_GROUP, my_patches - i0);
            for (int q = 0; q < cnt; ++q) tfy_mbar_wait(&full[(i0 + q) % WG_RING], ((i0 + q) / WG_RING) & 1);
            if (UNPOOL) tfy_fence_proxy_async();
            if (g == 0 && tid == 0) C_MARK(4);
            const uint32_t st0 = tfy_smem_u32(stages);
#pragma unroll 1
            for (int t = 0; t < TAPS; ++t) {
                const int kh = t / 3, kw = t - kh * 3;
                float d[16];
                tfy_wg_fence();
#pragma unroll 1
                for (int q = 0; q < cnt; ++q) {
                    const uint32_t dz0 = st0 + ((i0 + q) % WG_RING) * WG_STAGE_B, a0 = dz0 + Z_PATCH_B;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {      // 16 pixels (one h row of both images) per MMA
                        // A = dz^T: M = 64 o inside the 128 B pixel row; K = pixels, 8-pixel groups 1024 B apart
                        const uint64_t adesc = tfy_wg_desc(dz0 + j * 2 * 8 * Z_PIX_B, 16, 8 * Z_PIX_B, SW128);
                        // B = a (tap shifted): N = 32 c inside the 64 B pixel row; K = pixels, groups = (h, n) rows
                        const uint64_t bdesc =
                            tfy_wg_desc(a0 + (j + kh) * 2 * A_ROW_B + kw * A_PIX_B, 16, A_ROW_B, SW64);
                        tfy_wgmma_m64n32<1, 1>(d, adesc, bdesc, (q > 0 || j > 0) ? 1u : 0u);
                    }
                }
                tfy_wg_commit();
                tfy_wg_wait<0>();
#pragma unroll
                for (int i = 0; i < 16; ++i) mine[(t * 16 + i) * 128] += d[i];
            }
            if (lane == 0)
                for (int q = 0; q < cnt; ++q) tfy_mbar_arrive(&empty[(i0 + q) % WG_RING]);     // stages reusable
        }
        if (tid == 0) C_MARK(5);
        // partial tile rows o = (o, tap) rows of 128 B: value i of this thread is o = 16 w + lane / 4 + 8 ((i / 2) % 2),
        // c = 8 (i / 4) + 2 (lane % 4) + i % 2
        float* part = partials + (size_t)blockIdx.x * WG_PART;
        const int w = tid >> 5;
#pragma unroll 1
        for (int t = 0; t < TAPS; ++t) {
#pragma unroll
            for (int i = 0; i < 16; i += 2) {
                const int o = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (lane & 3);
                __stcg(reinterpret_cast<float2*>(part + (size_t)o * (TAPS * CIN) + t * CIN + c),
                       make_float2(mine[(t * 16 + i) * 128], mine[(t * 16 + i + 1) * 128]));
            }
        }
        if (sync) __threadfence();     // the grid barrier follows (deferred: the kernel boundary orders the stores)
        if (tid == 0) C_MARK(6);
    } else if (my_patches > 0) {
        if (UNPOOL) {
            // ---------------- un-pool producers (all 16 worker warps): a patch needs 4 x 4 pooled pixels x 2 images
            // x 8 channel groups = 256 tasks; thread t serves task t & 255 of patches (t >> 8), (t >> 8) + 2, ...
            // and always the same channel group, so db accumulates in registers.  Loads of two patches are in
            // flight together.
            const int t = threadIdx.x, task = t & 255, g = task & 7, n = (task >> 3) & 1, pp = task >> 4;
            const int ppy = pp >> 2, ppx = pp & 3;
            const int row0 = (ppy * 2 * 2 + n) * 8 + ppx * 2;
            float colacc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            CPatchIter it(tiles_x, tiles_y, n_cmp);
            if (t >> 8) it.next();
            for (int i = (t >> 8); i < my_patches; i += 4) {
                // patches i and i + 2 (if any)
                CPatchIter it2 = it;
                it2.next(); it2.next();
                const bool two = i + 2 < my_patches;
                const size_t p0 = ((size_t)(it.bz * 2 + n) * PH + it.ty * 4 + ppy) * PWp + it.tx * 4 + ppx;
                const size_t p1 = ((size_t)(it2.bz * 2 + n) * PH + it2.ty * 4 + ppy) * PWp + it2.tx * 4 + ppx;
                const CUnpoolIn in0 = c_unpool_load(dp, code, true, p0, g);
                const CUnpoolIn in1 = c_unpool_load(dp, code, two, two ? p1 : p0, g);
                float gated[8];
                {
                    const int s = i % WG_RING;
                    if (i >= WG_RING) tfy_mbar_wait(&empty[s], ((i / WG_RING) - 1) & 1);
                    c_unpool_emit(stages + (size_t)s * WG_STAGE_B, in0, scale, g, row0, 16, gated);
#pragma unroll
                    for (int k = 0; k < 8; ++k) colacc[k] += gated[k];
                    tfy_fence_proxy_async();
                    tfy_mbar_arrive(&full[s]);
                }
                if (two) {
                    const int i2 = i + 2, s = i2 % WG_RING;
                    if (i2 >= WG_RING) tfy_mbar_wait(&empty[s], ((i2 / WG_RING) - 1) & 1);
                    c_unpool_emit(stages + (size_t)s * WG_STAGE_B, in1, scale, g, row0, 16, gated);
#pragma unroll
                    for (int k = 0; k < 8; ++k) colacc[k] += gated[k];
                    tfy_fence_proxy_async();
                    tfy_mbar_arrive(&full[s]);
                }
                it.next(); it.next(); it.next(); it.next();
            }
            // lanes l, l+8, l+16, l+24 serve the same channel group: reduce them, one plain store per warp
            // (shared-memory float atomics are CAS loops: 512 threads on 64 addresses cost microseconds)
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                colacc[k] += __shfl_xor_sync(0xffffffffu, colacc[k], 8);
                colacc[k] += __shfl_xor_sync(0xffffffffu, colacc[k], 16);
            }
            if (lane < 8) {
#pragma unroll
                for (int k = 0; k < 8; ++k) s_db[warp * COUT + g * 8 + k] = colacc[k];
            }
        }
        if (UNPOOL) {
            asm volatile("bar.sync 1, %0;" ::"r"(WG_WORK_WARPS * 32) : "memory");     // all producers added their db
            if (threadIdx.x < COUT) {
                float a = 0.f;
#pragma unroll
                for (int q = 0; q < WG_WORK_WARPS; ++q) a += s_db[q * COUT + threadIdx.x];
                __stcg(partials + (size_t)blockIdx.x * WG_PART + WG_OUT + threadIdx.x, a);
            }
        }
        if (sync) __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) C_MARK(7);
    if (sync == nullptr) return;                                    // deferred: the dgrad kernel reduces

    // Grid-wide arrive / release (all CTAs are co-resident: grid <= #SMs, one CTA per SM).  Same-sector atomics
    // serialise at ~20-30 cycles each and every returning atomic in a chain costs an L2 round trip, so: arrivals
    // are fire-and-forget `red`s spread over 16 counters (one per 128-byte line, sync[32 + 32 k]); CTA 0 polls
    // them, clears them and bumps the generation word sync[0] that everybody else polls.
    if (threadIdx.x == 0) {
        __threadfence();
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(sync + 32 + 32 * (blockIdx.x & 15u)) : "memory");
    }
    if (blockIdx.x == 0 && warp == 0) {
        if (lane < 16 && lane < n_cmp) {
            const uint32_t expect = ((uint32_t)n_cmp - (uint32_t)lane + 15u) / 16u;
            volatile uint32_t* cnt = sync + 32 + 32 * lane;
            while (*cnt != expect) __nanosleep(20);
            *cnt = 0u;
        }
        __syncwarp();
        if (lane == 0) {
            __threadfence();
            *reinterpret_cast<volatile uint32_t*>(sync) = gen0 + 1;
        }
    }
    if (threadIdx.x == 0) {
        while (*reinterpret_cast<volatile uint32_t*>(sync) == gen0) __nanosleep(32);
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) C_MARK(8);
    // slice of the outputs owned by this CTA (float4 units), summed over the partials in a fixed order (c_wg_slice)
    constexpr int TOTAL4 = (UNPOOL ? WG_PART : WG_OUT) / 4, STRIDE4 = WG_PART / 4;
    const CWgSlice sl = c_wg_slice(TOTAL4, n_cmp, (int)blockIdx.x, WG_THREADS);
    const int lo = sl.lo, len = sl.len;
    const int n_part = n_cmp;                                       // every CTA wrote a partial
    const float4* src = reinterpret_cast<const float4*>(partials) + lo;
    auto store = [&](int f, const float4& s4) {
        __nv_bfloat162 l2 = __floats2bfloat162_rn(s4.x, s4.y), h2 = __floats2bfloat162_rn(s4.z, s4.w);
        uint2 packed;
        packed.x = *reinterpret_cast<uint32_t*>(&l2);
        packed.y = *reinterpret_cast<uint32_t*>(&h2);
        const int e = (lo + f) * 4;                                  // outputs [0, WG_OUT) = dW, then db
        if (e < WG_OUT) *reinterpret_cast<uint2*>(dw + e) = packed;
        else *reinterpret_cast<uint2*>(db + (e - WG_OUT)) = packed;
    };
    if (len > 0 && sl.parts > 1) {
        // few outputs per CTA (the usual case: 32): `parts` thread groups split the list of partials
        float4* red = reinterpret_cast<float4*>(stages);             // the ring is idle now
        const int parts = sl.parts;
        const int f = (int)threadIdx.x % len, part = (int)threadIdx.x / len;
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (part < parts) {
#pragma unroll 8
            for (int q = part; q < n_part; q += parts) {
                const float4 v = __ldcg(src + (size_t)q * STRIDE4 + f);
                s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
            }
        }
        red[threadIdx.x] = s4;
        __syncthreads();
        if (part == 0) {
            for (int q = 1; q < parts; ++q) {
                const float4 v = red[q * len + f];
                s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
            }
            store(f, s4);
        }
    } else {
        for (int f = (int)threadIdx.x; f < len; f += WG_THREADS) {
            float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
            for (int q = 0; q < n_part; ++q) {
                const float4 v = __ldcg(src + (size_t)q * STRIDE4 + f);
                s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
            }
            store(f, s4);
        }
    }
    if (threadIdx.x == 0) C_MARK(10);
}

// ------------------------------------------------------------------------------------------------
// First-layer weight + bias gradient (C_in = 1, 32 filters) on the tensor core:
//   D[n, o] = sum_pix X~[pix, n] dz[pix, o],   X~[pix, 0..8] = x[pix + tap], X~[pix, 9] = 1 (bias), rest 0
// M = 64 (n, padded), N = 32 (o), K = pixels.  dz rows (64 B) arrive by TMA exactly as they sit in memory
// (MN-major B, 64B swizzle); the im2col operand X~ (128-byte rows, 128B swizzle, MN-major A) is built in
// shared memory by 128 threads from the tiny single-channel input.  Replaces the CUDA-core wgrad kernel and the
// separate bias-gradient column sum of the first layer.
// warps 0..3 build X~, warps 4..7 MMA (warp 4, which holds rows 0..15 of D, also runs the epilogue), warp 8 TMA.
// acc: one partial [10 n][32 o] of 320 floats per CTA (plain stores, no float atomics); the last CTA to finish sums
// them in CTA order, so dW / db are the same bit for bit on every run.  counter: one uint32, zero on entry, left zero.
// ------------------------------------------------------------------------------------------------
constexpr int C1_O = 32, C1_STAGES = 4, C1_PIX = 128, C1_MAX_CTAS = 160;
constexpr int C1_A_B = C1_PIX * 128, C1_B_B = C1_PIX * 64, C1_STAGE_B = C1_A_B + C1_B_B;   // 16 KB + 8 KB
constexpr int C1_THREADS = 288;
constexpr size_t C1_SMEM = (size_t)C1_STAGES * C1_STAGE_B + 1024 + 256;

template <typename XT>
__global__ void __launch_bounds__(C1_THREADS, 1)
tfy_conv3x3_c1_wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dz, const XT* __restrict__ x,
                               float* __restrict__ acc, uint32_t* __restrict__ counter,
                               __nv_bfloat16* __restrict__ dw, __nv_bfloat16* __restrict__ dbias, int H, int W,
                               int n_pix, int n_chunks) {
    extern __shared__ uint8_t smem_raw[];
    C_TIMELINE_BEGIN();
    uint8_t* stages = tfy_align1024(smem_raw);        // [4] { X~ [128 pix][128 B] sw128 ; dz [128 pix][64 B] sw64 }
    uint64_t* full_a = reinterpret_cast<uint64_t*>(stages + (size_t)C1_STAGES * C1_STAGE_B);
    uint64_t* full_b = full_a + C1_STAGES;
    uint64_t* empty = full_b + C1_STAGES;
    __shared__ uint32_t s_last;

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    if (threadIdx.x == 0) {
        tfy_prefetch_tensormap(&map_dz);
        for (int s = 0; s < C1_STAGES; ++s) {
            tfy_mbar_init(&full_a[s], 128);
            tfy_mbar_init(&full_b[s], 1);
            tfy_mbar_init(&empty[s], 4);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // the padding columns of X~ (n >= 16) stay zero for the whole kernel
    for (int i = threadIdx.x; i < C1_STAGES * C1_A_B / 16; i += C1_THREADS) {
        const int s = i / (C1_A_B / 16), r = i - s * (C1_A_B / 16);
        *reinterpret_cast<uint4*>(stages + (size_t)s * C1_STAGE_B + (size_t)r * 16) = make_uint4(0, 0, 0, 0);
    }
    tfy_fence_proxy_async();
    __syncthreads();
    tfy_pdl_sync();                      // upstream grids complete; our dependents may start launching
    if (threadIdx.x == 0) C_MARK(1);
    const int my_chunks = ((int)blockIdx.x < n_chunks) ? (n_chunks - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int OH = H - 2, OW = W - 2;

    if (warp == 8) {
        if (tfy_elect_one()) {
            for (int i = 0; i < my_chunks; ++i) {
                const int s = i % C1_STAGES;
                if (i >= C1_STAGES) tfy_mbar_wait(&empty[s], ((i / C1_STAGES) - 1) & 1);
                const int chunk = (int)blockIdx.x + i * (int)gridDim.x;
                tfy_mbar_expect_tx(&full_b[s], C1_B_B);
                tfy_tma_load_2d(&map_dz, &full_b[s], stages + (size_t)s * C1_STAGE_B + C1_A_B, 0, chunk * C1_PIX);
            }
        }
    } else if (warp >= 4) {
        float d[16];
        tfy_wg_zero<C1_O>(d);
        for (int i = 0; i < my_chunks; ++i) {
            const int s = i % C1_STAGES;
            tfy_mbar_wait(&full_a[s], (i / C1_STAGES) & 1);
            tfy_mbar_wait(&full_b[s], (i / C1_STAGES) & 1);
            if (i == 0 && threadIdx.x == 128) C_MARK(4);
            const uint32_t a0 = tfy_smem_u32(stages + (size_t)s * C1_STAGE_B), b0 = a0 + C1_A_B;
            tfy_wg_fence();
#pragma unroll
            for (int j = 0; j < C1_PIX / 16; ++j) {
                // A = X~^T: M = 64 n inside the 128 B pixel row; B = dz: N = 32 o inside the 64 B pixel row
                const uint64_t adesc = tfy_wg_desc(a0 + j * 16 * 128, 16, 8 * 128, SW128);
                const uint64_t bdesc = tfy_wg_desc(b0 + j * 16 * 64, 16, 8 * 64, SW64);
                tfy_wgmma_m64n32<1, 1>(d, adesc, bdesc, 1u);
            }
            tfy_wg_commit();
            tfy_wg_wait<0>();
            if (lane == 0) tfy_mbar_arrive(&empty[s]);
        }
        if (threadIdx.x == 128) C_MARK(5);
        if (warp == 4) {
            // D rows 0..8 = taps, row 9 = bias; value i of this thread: row lane / 4 + 8 ((i / 2) % 2),
            // column 8 (i / 4) + 2 (lane % 4) + i % 2
            float* part = acc + (size_t)blockIdx.x * (10 * C1_O);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int n = (lane >> 2) + 8 * ((i >> 1) & 1), o = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
                if (n < 10) __stcg(part + n * C1_O + o, d[i]);
            }
            __threadfence();
            if (lane == 0) C_MARK(7);
        }
    } else {
        // ---------------- im2col builders: one pixel per thread per chunk; the next chunk's inputs are gathered
        // before this chunk is packed and stored (one exposed L2 round trip instead of one per chunk)
        const int r = threadIdx.x;                                  // row of the stage, 0..127
        const uint32_t sw = (uint32_t)(r & 7);
        auto gather = [&](int chunk, float* v) -> bool {
            const int p = chunk * C1_PIX + r;
            const bool ok = p < n_pix;
            if (ok) {
                const int b = p / (OH * OW), rem = p - b * (OH * OW), y = rem / OW, xx = rem - y * OW;
                const XT* src = x + ((size_t)b * H + y) * W + xx;
#pragma unroll
                for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw) v[kh * 3 + kw] = (float)src[kh * W + kw];
            } else {
#pragma unroll
                for (int t = 0; t < 9; ++t) v[t] = 0.f;
            }
            return ok;
        };
        float v[9];
        bool ok = my_chunks > 0 ? gather((int)blockIdx.x, v) : false;
        for (int i = 0; i < my_chunks; ++i) {
            const int s = i % C1_STAGES;
            float c1[8] = {v[8], ok ? 1.f : 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            const uint4 q0 = TfyPack<__nv_bfloat16>::pack(v), q1 = TfyPack<__nv_bfloat16>::pack(c1);
            if (i + 1 < my_chunks) ok = gather((int)blockIdx.x + (i + 1) * (int)gridDim.x, v);
            if (i >= C1_STAGES) tfy_mbar_wait(&empty[s], ((i / C1_STAGES) - 1) & 1);
            uint8_t* rowp = stages + (size_t)s * C1_STAGE_B + (size_t)r * 128;
            *reinterpret_cast<uint4*>(rowp + ((0u ^ sw) << 4)) = q0;    // 128B swizzle: chunk ^= row & 7
            *reinterpret_cast<uint4*>(rowp + ((1u ^ sw) << 4)) = q1;
            tfy_fence_proxy_async();
            tfy_mbar_arrive(&full_a[s]);
            if (threadIdx.x == 0) { if (i == 0) C_MARK(2); if (i == my_chunks - 1) C_MARK(3); }
        }
    }
    __syncthreads();
    // the last CTA to finish sums the per-CTA partials in CTA order and converts them
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = (atomicAdd(counter, 1u) == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (threadIdx.x == 0) C_MARK(8);
    if (s_last) {
        __threadfence();
        // PARTS thread groups each sum every PARTS-th partial (float4 columns), then the groups are added in order
        constexpr int F4 = 10 * C1_O / 4, PARTS = C1_THREADS / F4;
        __shared__ float4 s_part[PARTS * F4];
        const int f = (int)threadIdx.x % F4, part = (int)threadIdx.x / F4;
        if (part < PARTS) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            const float4* src = reinterpret_cast<const float4*>(acc);
#pragma unroll 8
            for (int g = part; g < (int)gridDim.x; g += PARTS) {
                const float4 v = __ldcg(src + (size_t)g * F4 + f);
                a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
            }
            s_part[part * F4 + f] = a;
        }
        __syncthreads();
        if ((int)threadIdx.x < F4) {
            float4 a = s_part[f];
            for (int q = 1; q < PARTS; ++q) {
                const float4 v = s_part[q * F4 + f];
                a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
            }
            const float vals[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = f * 4 + e, n = i / C1_O, o = i - n * C1_O;
                if (n < 9) dw[o * 9 + n] = __float2bfloat16(vals[e]);
                else dbias[o] = __float2bfloat16(vals[e]);
            }
        }
        if (threadIdx.x == 0) *counter = 0u;
    }
    if (threadIdx.x == 0) C_MARK(10);
}

// ------------------------------------------------------------------------------------------------
// First-layer forward (C_in = 1, 32 filters) on the tensor core:
//   y[pix, o] = relu( sum_k X~[pix, k] W~[o, k] ),  X~[pix, 0..8] = x[pix + tap], X~[pix, 9] = 1,  W~[o, 9] = bias[o]
// Two wgmma M64 N32 K16 per 128 pixels; both operands are built in shared memory in the un-swizzled K-major
// core-matrix layout ([k half][row][16 B]: lbo = distance between the halves, sbo = 128).  The CUDA-core
// version spends its time on 288 shared-memory weight loads + FMAs per pixel; here a thread gathers 9 inputs and
// stores 2 x 16 B, and the MMA warpgroup writes ReLU'd bf16 pairs straight from its accumulator registers.
// warps 0..3 build X~, warps 4..7 MMA + epilogue.
// ------------------------------------------------------------------------------------------------
constexpr int F1_STAGES = 4, F1_PIX = 128, F1_A_B = 2 * F1_PIX * 16;      // 4 KB per stage
constexpr int F1_W_B = 2 * C1_O * 16;                                     // 1 KB
constexpr int F1_THREADS = 8 * 32;
constexpr size_t F1_SMEM = (size_t)F1_STAGES * F1_A_B + F1_W_B + 128 + 256;

template <typename XT>
__global__ void __launch_bounds__(F1_THREADS, 2)
tfy_conv3x3_c1_fwd_tc_kernel(const XT* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                             const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int H, int W,
                             int n_pix, int n_chunks) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* stages = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    uint8_t* w_tile = stages + (size_t)F1_STAGES * F1_A_B;          // [2 k halves][32 o][16 B]
    uint64_t* full = reinterpret_cast<uint64_t*>(w_tile + F1_W_B);
    uint64_t* empty = full + F1_STAGES;

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
    if (threadIdx.x == 0) {
        for (int s = 0; s < F1_STAGES; ++s) { tfy_mbar_init(&full[s], 128); tfy_mbar_init(&empty[s], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    tfy_pdl_sync();                      // (the weights below are produced by the previous step's optimizer kernel)
    if (threadIdx.x < C1_O) {
        // W~ row o: taps 0..7 | tap 8, bias, 0 x 6
        const int o = threadIdx.x;
        float k0[8], k1[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int t = 0; t < 8; ++t) k0[t] = __bfloat162float(w[o * 9 + t]);
        k1[0] = __bfloat162float(w[o * 9 + 8]);
        k1[1] = __bfloat162float(bias[o]);
        *reinterpret_cast<uint4*>(w_tile + o * 16) = TfyPack<__nv_bfloat16>::pack(k0);
        *reinterpret_cast<uint4*>(w_tile + C1_O * 16 + o * 16) = TfyPack<__nv_bfloat16>::pack(k1);
    }
    tfy_fence_proxy_async();
    __syncthreads();
    const int my_chunks = ((int)blockIdx.x < n_chunks) ? (n_chunks - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int OH = H - 2, OW = W - 2;

    if (warp >= 4) {
        const uint64_t bdesc = tfy_wg_desc(tfy_smem_u32(w_tile), C1_O * 16, 128, TFY_WG_NOSWIZZLE);
        const int w = warp & 3;
        for (int i = 0; i < my_chunks; ++i) {
            const int s = i % F1_STAGES;
            const int chunk = (int)blockIdx.x + i * (int)gridDim.x;
            tfy_mbar_wait(&full[s], (i / F1_STAGES) & 1);
            tfy_fence_proxy_async();
            float acc[2][C1_O / 2];
            tfy_wg_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h)       // pixels [64 h, 64 h + 64): 8 core-matrix rows of 128 B further
                tfy_wgmma_m64n32<0, 0>(acc[h], tfy_wg_desc(tfy_smem_u32(stages + (size_t)s * F1_A_B + h * 64 * 16),
                                                           F1_PIX * 16, 128, TFY_WG_NOSWIZZLE), bdesc, 0u);
            tfy_wg_commit();
            tfy_wg_wait<0>();
            if (lane == 0) tfy_mbar_arrive(&empty[s]);
            // value i of this thread: pixel row 64 h + 16 w + lane / 4 + 8 ((i / 2) % 2), channel 8 (i / 4) + 2 (lane % 4)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int i2 = 0; i2 < C1_O / 2; i2 += 2) {
                    const int p = chunk * F1_PIX + 64 * h + 16 * w + (lane >> 2) + 8 * ((i2 >> 1) & 1);
                    const int o = 8 * (i2 >> 2) + 2 * (lane & 3);
                    if (p < n_pix)
                        *reinterpret_cast<__nv_bfloat162*>(y + (size_t)p * C1_O + o) =
                            __floats2bfloat162_rn(fmaxf(acc[h][i2], 0.f), fmaxf(acc[h][i2 + 1], 0.f));
                }
            }
        }
    } else {
        // ---------------- im2col builders: one pixel per thread per chunk; the next chunk's inputs are loaded
        // before this chunk's stage is waited for
        const int r = threadIdx.x;
        auto gather = [&](int chunk, float* v) -> bool {
            const int p = chunk * F1_PIX + r;
            const bool ok = p < n_pix;
            if (ok) {
                const int b = p / (OH * OW), rem = p - b * (OH * OW), yy = rem / OW, xx = rem - yy * OW;
                const XT* src = x + ((size_t)b * H + yy) * W + xx;
#pragma unroll
                for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw) v[kh * 3 + kw] = (float)src[kh * W + kw];
            } else {
#pragma unroll
                for (int t = 0; t < 9; ++t) v[t] = 0.f;
            }
            return ok;
        };
        float v[9];
        bool ok = my_chunks > 0 ? gather((int)blockIdx.x, v) : false;
        for (int i = 0; i < my_chunks; ++i) {
            const int s = i % F1_STAGES;
            float c1[8] = {v[8], ok ? 1.f : 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            const uint4 q0 = TfyPack<__nv_bfloat16>::pack(v), q1 = TfyPack<__nv_bfloat16>::pack(c1);
            if (i + 1 < my_chunks) ok = gather((int)blockIdx.x + (i + 1) * (int)gridDim.x, v);
            if (i >= F1_STAGES) tfy_mbar_wait(&empty[s], ((i / F1_STAGES) - 1) & 1);
            uint8_t* st = stages + (size_t)s * F1_A_B;
            *reinterpret_cast<uint4*>(st + r * 16) = q0;
            *reinterpret_cast<uint4*>(st + F1_PIX * 16 + r * 16) = q1;
            tfy_fence_proxy_async();
            tfy_mbar_arrive(&full[s]);
        }
    }
}

namespace {
bool c_attr_set = false;
int c_sms = 0;
bool c_init() {
    if (!tfy_tensor_map_encoder()) return false;
    if (!c_attr_set) {
        if (cudaFuncSetAttribute(tfy_conv3x3_fprop_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)FP_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(tfy_conv3x3_dgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)DG_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(tfy_conv3x3_dgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)DG_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(tfy_conv3x3_wgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)WG_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(tfy_conv3x3_wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)WG_SMEM) != cudaSuccess)
            return false;
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&c_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || c_sms <= 0)
            return false;
        c_attr_set = true;
    }
    return true;
}
// persistent grid: one CTA per SM, trimmed so that the patches divide as evenly as possible
int c_grid(int n_patches) {
    if (n_patches <= c_sms) return n_patches;
    const int waves = (n_patches + c_sms - 1) / c_sms;
    return (n_patches + waves - 1) / waves;
}
// NHWC bf16 tensor [B, H, W, C] seen as {C, W, B, H}; box = {C, bw, 2, bh}: one pixel per shared-memory row
bool c_map_nhwc(CUtensorMap* m, const void* p, int B, int H, int W, int C, int bw, int bh) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)B, (cuuint64_t)H};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)H * W * C * 2, (cuuint64_t)W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)C, (cuuint32_t)bw, 2, (cuuint32_t)bh};
    return tfy_tensor_map_bf16(m, p, 4, dims, strides, box,
                               C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
// weights [O][9][C] bf16 seen as {C, O, 9}; one box = everything, stored [tap][o][32 c] with 64-byte rows
bool c_map_w(CUtensorMap* m, const void* p) {
    cuuint64_t dims[3] = {(cuuint64_t)CIN, (cuuint64_t)COUT, (cuuint64_t)TAPS};
    cuuint64_t strides[2] = {(cuuint64_t)TAPS * CIN * 2, (cuuint64_t)CIN * 2};
    cuuint32_t box[3] = {(cuuint32_t)CIN, (cuuint32_t)COUT, (cuuint32_t)TAPS};
    return tfy_tensor_map_bf16(m, p, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}
}  // namespace

extern "C" {

// debug: device buffer of 16 x int64 per CTA receiving the event timeline of the next launches (nullptr = off)
int tfy_conv_set_timeline(long long* buf) {
    return (int)cudaMemcpyToSymbol(c_timeline, &buf, sizeof(buf));
}

// number of fp32 elements of the `partials` scratch buffer tfy_conv3x3_c32_wgrad needs
size_t tfy_conv3x3_c32_wgrad_scratch_elems() { return (size_t)160 * WG_PART; }

// a: [B, H, W, 32] bf16 (NHWC), w: [64, 3, 3, 32] bf16, bias: [64] bf16
// pooled / code: [B, (H-2)/2, (W-2)/2, 64].  Requires (H-2) % 8 == 0, (W-2) % 8 == 0, B % 2 == 0.
int tfy_conv3x3_c32_pool_fwd(const void* a, const void* w, const void* bias, void* pooled, void* code, int B, int H,
                             int W, float drop_rate, uint32_t seed, const TfyOptHyper* hp, cudaStream_t s) {
    const int OH = H - 2, OW = W - 2;
    if ((OH % 8) || (OW % 8) || (B % 2) || drop_rate < 0.f || drop_rate >= 1.f) return -2;
    if ((size_t)B * (OH / 2) * (OW / 2) * COUT >= (1ull << 32)) return -3;
    if (!c_init()) return -4;
    CUtensorMap ma, mw;
    if (!c_map_nhwc(&ma, a, B, H, W, CIN, HALO, HALO) || !c_map_w(&mw, w)) return -6;
    const int tiles_x = OW / 8, tiles_y = OH / 8, n_patches = tiles_x * tiles_y * (B / 2);
    tfy_launch_pdl((tfy_conv3x3_fprop_pool_kernel), dim3(c_grid(n_patches)), dim3(FP_THREADS), FP_SMEM, s, 
        ma, mw, (const __nv_bfloat16*)bias, (__nv_bfloat16*)pooled, (uint8_t*)code, H, W, tiles_x, tiles_y, n_patches,
        drop_rate, seed, hp);
    return (int)cudaGetLastError();
}

// dz: [B, H-2, W-2, 64] bf16, w: [64, 3, 3, 32], gate (optional): [B, H, W, 32], dx: [B, H, W, 32].  B % 2 == 0.
int tfy_conv3x3_c32_dgrad(const void* dz, const void* w, const void* gate, void* dx, int B, int H, int W,
                          cudaStream_t s) {
    if (B % 2) return -2;
    if (!c_init()) return -4;
    CUtensorMap mz, mw;
    if (!c_map_nhwc(&mz, dz, B, H - 2, W - 2, COUT, HALO, HALO) || !c_map_w(&mw, w)) return -6;
    const int tiles_x = (W + 7) / 8, tiles_y = (H + 7) / 8, n_patches = tiles_x * tiles_y * (B / 2);
    tfy_launch_pdl((tfy_conv3x3_dgrad_kernel<false>), dim3(c_grid(n_patches)), dim3(DG_THREADS), DG_SMEM, s,
        mz, mw, (const __nv_bfloat16*)gate, (__nv_bfloat16*)dx, H, W, tiles_x, tiles_y, n_patches, (const __nv_bfloat16*)nullptr, (const uint8_t*)nullptr, 1.0f,
        (const float*)nullptr, 0, (__nv_bfloat16*)nullptr, (__nv_bfloat16*)nullptr);
    return (int)cudaGetLastError();
}

// a: [B, H, W, 32], dz: [B, H-2, W-2, 64], dw: [64, 3, 3, 32] bf16 (overwritten).
// partials: tfy_conv3x3_c32_wgrad_scratch_elems() floats of scratch; sync: 1024 x uint32, zeroed once at allocation.
int tfy_conv3x3_c32_wgrad(const void* a, const void* dz, float* partials, void* dw, uint32_t* sync, int B, int H, int W,
                          cudaStream_t s) {
    const int OH = H - 2, OW = W - 2;
    if ((OH % 8) || (OW % 8) || (B % 2)) return -2;
    if (!c_init() || c_sms > 160) return -4;
    CUtensorMap mz, ma;
    if (!c_map_nhwc(&mz, dz, B, OH, OW, COUT, 8, 8) || !c_map_nhwc(&ma, a, B, H, W, CIN, HALO, HALO)) return -6;
    const int tiles_x = OW / 8, tiles_y = OH / 8, n_patches = tiles_x * tiles_y * (B / 2);
    tfy_launch_pdl((tfy_conv3x3_wgrad_kernel<false>), dim3(c_grid(n_patches)), dim3(WG_THREADS), WG_SMEM, s, mz, ma,
                   partials, (__nv_bfloat16*)dw, sync, tiles_x, tiles_y, n_patches, (const __nv_bfloat16*)nullptr,
                   (const uint8_t*)nullptr, 1.0f, (__nv_bfloat16*)nullptr, 0, 0, TfyOverlapStep{});
    return (int)cudaGetLastError();
}

// Fused pool/dropout/ReLU backward variants: instead of a materialised dz they take the pooled gradient
// dp [B, (H-2)/2, (W-2)/2, 64] bf16, the forward kernel's code bytes (same shape) and the dropout scale.
// With `partials`, the kernel also reduces the n_part weight-gradient partials that
// tfy_conv3x3_c32_wgrad_unpool_deferred left there into dw [64, 3, 3, 32] and db [64] (bf16): the same bits as
// tfy_conv3x3_c32_wgrad_unpool gives.  partials == nullptr: no reduction (tfy_conv3x3_c32_dgrad_unpool).
int tfy_conv3x3_c32_dgrad_unpool_reduce(const void* dp, const void* code, float scale, const void* w,
                                        const void* gate, void* dx, int B, int H, int W, const float* partials,
                                        int n_part, void* dw, void* db, cudaStream_t s) {
    if ((B % 2) || ((H - 2) % 8) || ((W - 2) % 8)) return -2;
    if (partials != nullptr && (n_part <= 0 || n_part > 160 || dw == nullptr || db == nullptr)) return -2;
    if (!c_init()) return -4;
    CUtensorMap mw;
    if (!c_map_w(&mw, w)) return -6;
    const int tiles_x = (W + 7) / 8, tiles_y = (H + 7) / 8, n_patches = tiles_x * tiles_y * (B / 2);
    tfy_launch_pdl((tfy_conv3x3_dgrad_kernel<true>), dim3(c_grid(n_patches)), dim3(DG_THREADS), DG_SMEM, s, mw, mw,
                   (const __nv_bfloat16*)gate, (__nv_bfloat16*)dx, H, W, tiles_x, tiles_y, n_patches,
                   (const __nv_bfloat16*)dp, (const uint8_t*)code, scale, partials, n_part, (__nv_bfloat16*)dw,
                   (__nv_bfloat16*)db);
    return (int)cudaGetLastError();
}

int tfy_conv3x3_c32_dgrad_unpool(const void* dp, const void* code, float scale, const void* w, const void* gate,
                                 void* dx, int B, int H, int W, cudaStream_t s) {
    return tfy_conv3x3_c32_dgrad_unpool_reduce(dp, code, scale, w, gate, dx, B, H, W, nullptr, 0, nullptr, nullptr, s);
}

}  // extern "C"

namespace {
// sync == nullptr: deferred reduction (see tfy_conv3x3_wgrad_kernel); *n_part receives the number of partials
int c_wgrad_unpool(const void* a, const void* dp, const void* code, float scale, float* partials, void* dw, void* db,
                   uint32_t* sync, int B, int H, int W, const TfyOverlapStep* ov, int* n_part, cudaStream_t s) {
    const int OH = H - 2, OW = W - 2;
    if ((OH % 8) || (OW % 8) || (B % 2)) return -2;
    if (!c_init() || c_sms > 160) return -4;
    CUtensorMap ma;
    if (!c_map_nhwc(&ma, a, B, H, W, CIN, HALO, HALO)) return -6;
    const int tiles_x = OW / 8, tiles_y = OH / 8, n_patches = tiles_x * tiles_y * (B / 2);
    const int n_cmp = c_grid(n_patches);
    TfyOverlapStep o{};
    if (ov != nullptr && ov->n_cta > 0) {
        o = *ov;
        if (o.n_cta > c_sms - n_cmp) return -7;       // the role must not displace a compute CTA
        if (o.slot0 < 0 || o.slot0 + o.n_cta > TFY_MAX_BLOCKS) return -8;
    }
    if (n_part != nullptr) *n_part = n_cmp;
    tfy_launch_pdl((tfy_conv3x3_wgrad_kernel<true>), dim3(n_cmp + o.n_cta), dim3(WG_THREADS), WG_SMEM, s, ma, ma,
                   partials, (__nv_bfloat16*)dw, sync, tiles_x, tiles_y, n_patches, (const __nv_bfloat16*)dp,
                   (const uint8_t*)code, scale, (__nv_bfloat16*)db, OH / 2, OW / 2, o);
    return (int)cudaGetLastError();
}
}  // namespace

extern "C" {

// also writes db [64] = sum over batch and positions of the gated pooled gradient.
// ov (optional): a fused gradient-exchange/optimizer step to run on SPARE SMs next to the weight gradient
// (tfy_overlap_role).  ov->n_cta is clamped to the SMs the compute grid leaves free (576 patches -> 116 compute
// CTAs of 5 patches on a 132-SM H100 -> up to 16 communication CTAs); tfy_conv3x3_c32_wgrad_spare_ctas() tells
// the caller how many that is so that it can size the overlapped range.
int tfy_conv3x3_c32_wgrad_unpool_ov(const void* a, const void* dp, const void* code, float scale, float* partials,
                                    void* dw, void* db, uint32_t* sync, int B, int H, int W, const TfyOverlapStep* ov,
                                    cudaStream_t s) {
    return c_wgrad_unpool(a, dp, code, scale, partials, dw, db, sync, B, H, W, ov, nullptr, s);
}

// Deferred variant: the compute CTAs only store their fp32 partials (dW tile + db) in `partials` -- no grid barrier,
// no reduction -- and *n_part receives their number.  tfy_conv3x3_c32_dgrad_unpool_reduce, the next launch on the
// stream, turns them into dw / db.
int tfy_conv3x3_c32_wgrad_unpool_deferred(const void* a, const void* dp, const void* code, float scale,
                                          float* partials, int B, int H, int W, const TfyOverlapStep* ov,
                                          int* n_part, cudaStream_t s) {
    if (n_part == nullptr) return -2;
    return c_wgrad_unpool(a, dp, code, scale, partials, nullptr, nullptr, nullptr, B, H, W, ov, n_part, s);
}

int tfy_conv3x3_c32_wgrad_unpool(const void* a, const void* dp, const void* code, float scale, float* partials,
                                 void* dw, void* db, uint32_t* sync, int B, int H, int W, cudaStream_t s) {
    return tfy_conv3x3_c32_wgrad_unpool_ov(a, dp, code, scale, partials, dw, db, sync, B, H, W, nullptr, s);
}

// SMs the weight-gradient grid leaves idle for B images of H x W (0 when the patches fill every SM)
int tfy_conv3x3_c32_wgrad_spare_ctas(int B, int H, int W) {
    if (!c_init()) return 0;
    const int n_patches = ((W - 2) / 8) * ((H - 2) / 8) * (B / 2);
    const int spare = c_sms - c_grid(n_patches);
    return spare > 0 ? spare : 0;
}

// First-layer (C_in = 1, 32 filters) forward with bias + ReLU.  x: [B, H, W, 1] fp32 or bf16, w: [32, 3, 3, 1] bf16,
// bias: [32] bf16, y: [B, H-2, W-2, 32] bf16.
int tfy_conv3x3_c1_fwd_tc(const void* x, int x_is_f32, const void* w, const void* bias, void* y, int B, int H, int W,
                          cudaStream_t s) {
    if (!c_init()) return -4;
    const long long n_pix_ll = (long long)B * (H - 2) * (W - 2);
    if (n_pix_ll >= (1ll << 31) - F1_PIX) return -3;
    const int n_pix = (int)n_pix_ll, n_chunks = (n_pix + F1_PIX - 1) / F1_PIX;
    const int grid = n_chunks < 2 * c_sms ? n_chunks : 2 * c_sms;
    if (x_is_f32)
        tfy_launch_pdl((tfy_conv3x3_c1_fwd_tc_kernel<float>), dim3(grid), dim3(F1_THREADS), F1_SMEM, s, (const float*)x,
                       (const __nv_bfloat16*)w, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y, H, W, n_pix, n_chunks);
    else
        tfy_launch_pdl((tfy_conv3x3_c1_fwd_tc_kernel<__nv_bfloat16>), dim3(grid), dim3(F1_THREADS), F1_SMEM, s,
                       (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y,
                       H, W, n_pix, n_chunks);
    return (int)cudaGetLastError();
}

// First-layer (C_in = 1, 32 filters) weight + bias gradient.  x: [B, H, W, 1] fp32 or bf16, dz: [B, H-2, W-2, 32] bf16
// (already gated by the layer's ReLU), dw: [32, 3, 3, 1] bf16, dbias: [32] bf16.  acc: 160 x 320 floats of scratch
// (one partial per CTA) and counter: one uint32, zero on entry (and left zero).
int tfy_conv3x3_c1_wgrad_tc(const void* x, int x_is_f32, const void* dz, float* acc, uint32_t* counter, void* dw,
                            void* dbias, int B, int H, int W, cudaStream_t s) {
    if (!c_init() || c_sms > C1_MAX_CTAS) return -4;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(tfy_conv3x3_c1_wgrad_tc_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)C1_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(tfy_conv3x3_c1_wgrad_tc_kernel<__nv_bfloat16>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C1_SMEM) != cudaSuccess)
            return -5;
        attr = true;
    }
    const long long n_pix_ll = (long long)B * (H - 2) * (W - 2);
    if (n_pix_ll >= (1ll << 31) - C1_PIX) return -3;
    const int n_pix = (int)n_pix_ll, n_chunks = (n_pix + C1_PIX - 1) / C1_PIX;
    CUtensorMap mz;
    {
        cuuint64_t dims[2] = {(cuuint64_t)C1_O, (cuuint64_t)n_pix};
        cuuint64_t strides[1] = {(cuuint64_t)C1_O * 2};
        cuuint32_t box[2] = {(cuuint32_t)C1_O, (cuuint32_t)C1_PIX};
        if (!tfy_tensor_map_bf16(&mz, dz, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
            return -6;
    }
    const int grid = c_grid(n_chunks);
    if (x_is_f32)
        tfy_launch_pdl((tfy_conv3x3_c1_wgrad_tc_kernel<float>), dim3(grid), dim3(C1_THREADS), C1_SMEM, s, 
            mz, (const float*)x, acc, counter, (__nv_bfloat16*)dw, (__nv_bfloat16*)dbias, H, W, n_pix, n_chunks);
    else
        tfy_launch_pdl((tfy_conv3x3_c1_wgrad_tc_kernel<__nv_bfloat16>), dim3(grid), dim3(C1_THREADS), C1_SMEM, s, 
            mz, (const __nv_bfloat16*)x, acc, counter, (__nv_bfloat16*)dw, (__nv_bfloat16*)dbias, H, W, n_pix,
            n_chunks);
    return (int)cudaGetLastError();
}

}  // extern "C"
