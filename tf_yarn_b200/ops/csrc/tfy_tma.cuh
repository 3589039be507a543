// Hopper (sm_90a) asynchronous-copy helpers shared by the TMA kernels: shared-memory mbarriers, TMA tensor loads
// and stores, and the host-side encoding of bf16 tensor maps.
//
// Every kernel that stages operands through TMA uses the same protocol: one elected thread arms an mbarrier with
// the byte count it expects (expect_tx), issues the bulk tensor copies that complete on that barrier, and the
// consumers wait on its phase parity.  Threads that write a tile with ordinary stores for the tensor core (or a
// TMA store) to read fence the generic proxy against the async proxy first.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ uint32_t tfy_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// TMA destinations with a 128-byte swizzle (and the wgmma descriptors that read them) need 1024-byte alignment.
__device__ __forceinline__ uint8_t* tfy_align1024(uint8_t* p) {
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

__device__ __forceinline__ void tfy_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tfy_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void tfy_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tfy_smem_u32(bar)) : "memory");
}
// Arrival on the mbarrier at bar's offset in the shared memory of cluster CTA `rank` (this CTA's own included).  It
// releases at CTA scope only: it signals that this thread's async-proxy reads of a stage (wgmma) have retired, and a
// cluster-scope release would wait for every earlier store of the thread to become visible to the cluster.
__device__ __forceinline__ void tfy_mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
        ::"r"(tfy_smem_u32(bar)), "r"(rank)
        : "memory");
}
// Every thread of every CTA of the cluster.  RELAXED: the arrival orders none of the thread's earlier accesses (enough
// after fence.mbarrier_init, which releases the barrier initialisation itself); otherwise it releases them.
template <bool RELAXED = false>
__device__ __forceinline__ void tfy_cluster_sync() {
    if constexpr (RELAXED)
        asm volatile("barrier.cluster.arrive.relaxed;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
    else
        asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
__device__ __forceinline__ void tfy_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tfy_smem_u32(bar)), "r"(bytes)
                 : "memory");
}
// PTX scopes the labels to the braces, so every inlined copy of this loop may use the same names.
__device__ __forceinline__ void tfy_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(tfy_smem_u32(bar)), "r"(parity) : "memory");
}

// Tensor loads: the box at coordinates (c0 = innermost, ...) of `map` into dst; completion is counted on bar.
__device__ __forceinline__ void tfy_tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(tfy_smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(tfy_smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// The same box written at dst's offset in the shared memory of every CTA of the cluster whose rank is set in cta_mask,
// completion counted on the mbarrier at bar's offset in each of them.
__device__ __forceinline__ void tfy_tma_load_2d_multicast(const CUtensorMap* map, uint64_t* bar, void* dst, int c0,
                                                          int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%4, %5}], [%2], %3;"
        ::"r"(tfy_smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(tfy_smem_u32(bar)), "h"(cta_mask),
          "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tfy_tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1,
                                                int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(tfy_smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(tfy_smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tfy_tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1,
                                                int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(tfy_smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(tfy_smem_u32(bar)), "r"(c0),
        "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// Tensor store of the box at (c0, c1) from src; the caller commits and waits on the bulk group.
__device__ __forceinline__ void tfy_tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(tfy_smem_u32(src)), "r"(c0), "r"(c1)
                 : "memory");
}

__device__ __forceinline__ void tfy_prefetch_tensormap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// Makes this thread's generic-proxy shared-memory writes visible to the async proxy (wgmma operand reads, TMA stores).
__device__ __forceinline__ void tfy_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One lane of a CONVERGED warp: the compiler knows the guarded region runs on exactly one thread and keeps the TMA
// operands in uniform registers.
__device__ __forceinline__ bool tfy_elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
using TfyTensorMapEncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                          const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                          CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                          CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled from the driver the runtime uses (the library does not link libcuda); nullptr when it cannot
// be resolved, in which case the next call tries again.
inline TfyTensorMapEncodeFn tfy_tensor_map_encoder() {
    static TfyTensorMapEncodeFn encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult st;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &st) == cudaSuccess &&
            st == cudaDriverEntryPointSuccess && fn)
            encode = reinterpret_cast<TfyTensorMapEncodeFn>(fn);
    }
    return encode;
}

// bf16 tensor of `rank` dimensions (dims and box innermost first, strides_bytes for dimensions 1 .. rank-1), dense
// elements, no interleave; out-of-bounds box elements read as zeros and are not written by stores.
inline bool tfy_tensor_map_bf16(CUtensorMap* map, const void* ptr, cuuint32_t rank, const cuuint64_t* dims,
                                const cuuint64_t* strides_bytes, const cuuint32_t* box, CUtensorMapSwizzle swizzle,
                                CUtensorMapL2promotion l2_promotion) {
    const TfyTensorMapEncodeFn encode = tfy_tensor_map_encoder();
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    return encode && encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides_bytes,
                            box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2_promotion,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Row-major [rows, cols] bf16 matrix with leading dimension ld (elements): the K-major GEMM operand map.  One box is
// 64 columns (one 128-byte swizzle atom) x box_rows rows.
inline bool tfy_tensor_map_bf16_2d(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld,
                                   uint32_t box_rows = 128) {
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {ld * 2};
    const cuuint32_t box[2] = {64, box_rows};
    return tfy_tensor_map_bf16(map, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}
