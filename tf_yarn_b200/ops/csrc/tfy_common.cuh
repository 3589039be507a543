// Shared device helpers for the tf_yarn_b200 sm_90a kernels.
//
// Everything in ops/csrc is written for ONE target: Hopper H100
// (-gencode arch=compute_90a,code=sm_90a).  There is no fallback path for
// other architectures.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "tfy_lr_schedule.cuh"

#define TFY_NUM_SMS 132               // H100 SXM: sizes the grid caps of the streaming kernels
#define TFY_MAX_RANKS 16
#define TFY_MAX_BLOCKS 1024            // barrier slots (one per CTA index)
#define TFY_FLAGS_BYTES (TFY_MAX_BLOCKS * TFY_MAX_RANKS * 4)

// Per-process view of the symmetric arena.  Passed BY VALUE to kernels (it is
// 160 bytes, well inside the 4 KB kernel parameter space) so that a CUDA graph
// captures the peer addresses together with the launch.
struct TfyCommCtx {
    uint64_t peer_base[TFY_MAX_RANKS];  // VA (in THIS process) of every rank's arena
    uint64_t mc_base;                   // multicast VA of the arena, 0 if NVLS is unavailable
    uint32_t* epoch;                    // local (non-shared) [TFY_MAX_BLOCKS][TFY_MAX_RANKS] counters
    int32_t rank;
    int32_t world;
};

// Device-resident optimizer hyper-parameters.  They live in HBM (not in kernel
// arguments) so that a captured CUDA graph sees learning-rate schedule changes
// and the step counter advancing without being re-captured.
struct TfyOptHyper {
    float lr;
    float p1;            // Adadelta: rho   | Adam, Adamax, Nadam: beta1 | SGD: momentum | Adagrad: initial acc (unused in kernel) | RMSprop: rho
    float p2;            // Adam, Adamax, Nadam: beta2 | SGD: dampening | RMSprop: momentum
    float eps;
    float weight_decay;
    float grad_scale;    // multiplied into the (already averaged) gradient, e.g. 1/loss_scale
    int32_t step;        // completed optimizer steps
    int32_t flags;       // bit0: nesterov (SGD) / decoupled weight decay (Adam) / centered (RMSprop)
    uint32_t done;       // CTA completion counter used to advance `step` exactly once per launch
    uint32_t pad;
};

// The hyper block of a fused step launched with TFY_OPT_LR_SCHEDULE: the schedule follows the hyper-parameters, and
// the step stores hp.lr = schedule(hp.step) whenever it advances hp.step (tfy_lr_schedule.cuh).
struct TfyHyperBlock {
    TfyOptHyper hp;
    TfyLrSchedule sched;
};

// Nadam's hyper block: TfyHyperBlock's layout followed by the running product of its momentum schedule,
// mu_product = mu_1 * ... * mu_t after t updates (1 before the first).  It depends on the history of the step counter
// and device and host pow differ, so it is kept on the device in float64 rather than rebuilt from t: every CTA of a
// step reads it with lr, and the thread that advances hp.step writes the next one (tfy_nadam_advance).
struct TfyNadamHyperBlock {
    TfyOptHyper hp;
    TfyLrSchedule sched;
    double mu_product;
};
static_assert(offsetof(TfyNadamHyperBlock, sched) == offsetof(TfyHyperBlock, sched) &&
                  sizeof(TfyHyperBlock) == offsetof(TfyNadamHyperBlock, mu_product),
              "a Nadam hyper block starts with a TfyHyperBlock");

// Called by the one thread that advances the step counter of a scheduled step, after every CTA of the step has read
// hp->lr.
__device__ __forceinline__ void tfy_advance_scheduled_step(TfyOptHyper* hp, int step) {
    hp->step = step + 1;
    hp->lr = tfy_lr_schedule_eval(reinterpret_cast<const TfyHyperBlock*>(hp)->sched, (int64_t)step + 1);
}

enum TfyDtype { TFY_BF16 = 0, TFY_F32 = 1 };
enum TfyAlgo { TFY_ALGO_ONESHOT = 0, TFY_ALGO_TWOSHOT = 1, TFY_ALGO_NVLS = 2 };
enum TfyOpt { TFY_OPT_SGD = 0, TFY_OPT_ADADELTA = 1, TFY_OPT_ADAM = 2, TFY_OPT_ADAGRAD = 3, TFY_OPT_FTRL = 4,
               TFY_OPT_RMSPROP = 5, TFY_OPT_ADAMAX = 6, TFY_OPT_NADAM = 7 };
// Or-ed into the `opt` code of a fused-step launch: `hp` heads a TfyHyperBlock and the step evaluates its schedule.
// The bit selects separate instantiations, so the kernels of a constant learning rate carry no schedule code.
#define TFY_OPT_LR_SCHEDULE 0x100
enum TfyMode { TFY_MODE_LOCAL = 0, TFY_MODE_P2P = 1, TFY_MODE_NVLS = 2 };

// ---------------------------------------------------------------------------
// system-scope flag primitives (cross-GPU barrier on the signal pad)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tfy_red_release_sys_inc(uint32_t* addr) {
    asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(addr) : "memory");
}
__device__ __forceinline__ uint32_t tfy_ld_acquire_sys(const uint32_t* addr) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
    return v;
}

// K8 — device-side barrier between the CTAs with the same blockIdx.x on every
// rank.  Monotonic counters: a rank adds 1 to flags[slot][me] on every peer
// (fire-and-forget `red.release.sys`, so the signal costs one one-way NVLink
// hop, not a CAS round trip) and then spins with `ld.acquire.sys` on its own
// pad until every peer's counter reached the local epoch.  The epoch lives in
// local HBM, so the protocol is replay-safe inside CUDA graphs.
__device__ __forceinline__ void tfy_block_barrier(const TfyCommCtx& c) {
    __syncthreads();
    if ((int)threadIdx.x < c.world) {
        const int peer = threadIdx.x;
        const uint32_t slot = blockIdx.x;
        uint32_t* ep = c.epoch + slot * TFY_MAX_RANKS + peer;
        const uint32_t e = *ep + 1u;
        uint32_t* remote = reinterpret_cast<uint32_t*>(c.peer_base[peer]) + slot * TFY_MAX_RANKS + c.rank;
        tfy_red_release_sys_inc(remote);
        const uint32_t* mine =
            reinterpret_cast<const uint32_t*>(c.peer_base[c.rank]) + slot * TFY_MAX_RANKS + peer;
        while ((int32_t)(tfy_ld_acquire_sys(mine) - e) < 0) {
        }
        *ep = e;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------
// Grid-level cross-GPU barriers (K2/K3/K4).  A kernel that only runs tfy_block_barrier pays, in every CTA, its
// own system-scope release and its own NVLink hop, so its cost grows with the grid, and the fused step ran two
// of them.  What the collectives need is weaker:
//   entry: "every rank has STARTED this kernel" (its inputs are complete by stream order).  ONE signal per rank
//          pair, sent by CTA 0; every CTA polls the LOCAL pad.
//   exit : "every rank's stores have landed".  Each CTA fences its own stores and arrives on a local counter;
//          the LAST CTA signals the peers once and waits for their signals, so the grid cannot complete before
//          the data of all peers is in place.  Other CTAs leave at once (or also wait, `all_wait`, when they
//          go on to overwrite inputs the peers were reading).
// Epochs: one monotonic counter per slot in local memory, bumped by the CTA that finishes last (CUDA-graph
// replay safe).  Grids need not be co-resident.
// ---------------------------------------------------------------------------
#define TFY_SLOT_GRID_ENTRY 1008u
#define TFY_SLOT_GRID_EXIT 1009u
#define TFY_SLOT_GRID_SCRATCH 1010u     // epoch words used as local counters: [0] arrive, [1] finish

__device__ __forceinline__ uint32_t tfy_grid_epoch(const TfyCommCtx& c) {
    return *reinterpret_cast<volatile uint32_t*>(c.epoch + TFY_SLOT_GRID_ENTRY * TFY_MAX_RANKS) + 1u;
}

__device__ __forceinline__ void tfy_grid_poll(const TfyCommCtx& c, uint32_t slot, uint32_t e) {
    if ((int)threadIdx.x < c.world) {
        const uint32_t* mine =
            reinterpret_cast<const uint32_t*>(c.peer_base[c.rank]) + slot * TFY_MAX_RANKS + threadIdx.x;
        while ((int32_t)(tfy_ld_acquire_sys(mine) - e) < 0) {
        }
    }
    __syncthreads();
}

__device__ __forceinline__ void tfy_grid_signal(const TfyCommCtx& c, uint32_t slot) {
    if ((int)threadIdx.x < c.world) {
        uint32_t* remote =
            reinterpret_cast<uint32_t*>(c.peer_base[threadIdx.x]) + slot * TFY_MAX_RANKS + c.rank;
        tfy_red_release_sys_inc(remote);
    }
}

// all threads of all CTAs; e = tfy_grid_epoch(c) read at kernel start
__device__ __forceinline__ void tfy_grid_entry(const TfyCommCtx& c, uint32_t e) {
    if (blockIdx.x == 0) tfy_grid_signal(c, TFY_SLOT_GRID_ENTRY);
    tfy_grid_poll(c, TFY_SLOT_GRID_ENTRY, e);
}

__device__ __forceinline__ void tfy_grid_exit(const TfyCommCtx& c, uint32_t e, bool all_wait) {
    __shared__ uint32_t s_last;
    __syncthreads();                                   // every thread of the CTA has issued its stores
    if (threadIdx.x == 0) {
        __threadfence_system();                        // ... and they are performed (peer replicas included)
        uint32_t prev;
        uint32_t* cnt = c.epoch + TFY_SLOT_GRID_SCRATCH * TFY_MAX_RANKS;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(cnt) : "memory");
        s_last = (prev == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last) tfy_grid_signal(c, TFY_SLOT_GRID_EXIT);
    if (s_last || all_wait) tfy_grid_poll(c, TFY_SLOT_GRID_EXIT, e);
}

// last statement of the kernel (all CTAs): the CTA that finishes last bumps the epochs and clears the counters
__device__ __forceinline__ bool tfy_grid_finish(const TfyCommCtx& c, uint32_t e) {
    __shared__ uint32_t s_fin;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        uint32_t* scratch = c.epoch + TFY_SLOT_GRID_SCRATCH * TFY_MAX_RANKS;
        const uint32_t prev = atomicAdd(scratch + 1, 1u);
        s_fin = (prev == gridDim.x - 1) ? 1u : 0u;
        if (s_fin) {
            c.epoch[TFY_SLOT_GRID_ENTRY * TFY_MAX_RANKS] = e;
            c.epoch[TFY_SLOT_GRID_EXIT * TFY_MAX_RANKS] = e;
            scratch[0] = 0u;
            scratch[1] = 0u;
        }
    }
    __syncthreads();
    return s_fin != 0u;
}

// ---------------------------------------------------------------------------
// 16-byte vector helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint4 tfy_ld16(const void* p) {
    uint4 v;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
// streaming (peer) load: do not allocate in L1, data is used once
__device__ __forceinline__ uint4 tfy_ld16_stream(const void* p) {
    uint4 v;
    asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
// the same load as fp32 lanes: rows of a parameter server's master tables, possibly on a peer GPU
__device__ __forceinline__ float4 tfy_ld_peer_f32x4(const void* p) {
    float4 v;
    asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void tfy_st16(void* p, uint4 v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void tfy_st16_sys(void* p, uint4 v) {
    asm volatile("st.global.relaxed.sys.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

// NVLS: in-switch reduction of the 16 bytes at the same offset of every
// replica bound to the multicast object.  bf16 inputs are accumulated in fp32
// inside the switch (.acc::f32) and rounded once on the way out.
__device__ __forceinline__ uint4 tfy_mc_ld_reduce_bf16x8(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
__device__ __forceinline__ uint4 tfy_mc_ld_reduce_f32x4(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
// NVLS: one store, replicated by the switch into every rank's HBM.
__device__ __forceinline__ void tfy_mc_st16(void* mc, uint4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}

__device__ __forceinline__ float tfy_bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float tfy_bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t tfy_pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

// Counter-based dropout randomness shared by every kernel that draws a mask: hash(seed, layer salt, optimizer step,
// element); the step is read from the device-resident TfyOptHyper, so a replayed CUDA graph draws fresh masks.
__device__ __forceinline__ uint32_t tfy_hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
// uniform in [0,1) for (seed, step, index)
__device__ __forceinline__ float tfy_uniform(uint32_t seed, uint32_t step, uint64_t idx) {
    uint32_t h = tfy_hash32(seed ^ tfy_hash32(step * 0x9E3779B9U + 0x85ebca6bU) ^
                            tfy_hash32((uint32_t)idx * 0xC2B2AE35U + (uint32_t)(idx >> 32) + 0x27d4eb2fU));
    return (float)(h >> 8) * (1.0f / 16777216.0f);
}
// The conv2 forward's draws (tfy_conv3x3_fprop_pool_kernel): a per-step salt, then one raw hash per group of 4 pooled
// elements, one byte per element.  For group indices below 2^32 the raw hash is the one tfy_uniform keeps the top 24
// bits of.  (A macro: as an inline function it changes the forward kernel's instruction schedule.)
__device__ __forceinline__ uint32_t tfy_drop_salt(uint32_t seed, uint32_t step) {
    return seed ^ tfy_hash32(step * 0x9E3779B9U + 0x85ebca6bU);
}
#define TFY_DROP_HASH(salt, group) tfy_hash32((salt) ^ tfy_hash32((uint32_t)(group) * 0xC2B2AE35U + 0x27d4eb2fU))

template <typename T>
struct TfyPack;  // 16-byte pack of T

template <>
struct TfyPack<__nv_bfloat16> {
    static constexpr int N = 8;
    __device__ static __forceinline__ void unpack(const uint4& v, float* f) {
        f[0] = tfy_bf16lo(v.x); f[1] = tfy_bf16hi(v.x);
        f[2] = tfy_bf16lo(v.y); f[3] = tfy_bf16hi(v.y);
        f[4] = tfy_bf16lo(v.z); f[5] = tfy_bf16hi(v.z);
        f[6] = tfy_bf16lo(v.w); f[7] = tfy_bf16hi(v.w);
    }
    __device__ static __forceinline__ void accum(const uint4& v, float* f) {
        f[0] += tfy_bf16lo(v.x); f[1] += tfy_bf16hi(v.x);
        f[2] += tfy_bf16lo(v.y); f[3] += tfy_bf16hi(v.y);
        f[4] += tfy_bf16lo(v.z); f[5] += tfy_bf16hi(v.z);
        f[6] += tfy_bf16lo(v.w); f[7] += tfy_bf16hi(v.w);
    }
    __device__ static __forceinline__ uint4 pack(const float* f) {
        uint4 v;
        v.x = tfy_pack_bf16x2(f[0], f[1]); v.y = tfy_pack_bf16x2(f[2], f[3]);
        v.z = tfy_pack_bf16x2(f[4], f[5]); v.w = tfy_pack_bf16x2(f[6], f[7]);
        return v;
    }
    __device__ static __forceinline__ uint4 mc_ld_reduce(const void* mc) { return tfy_mc_ld_reduce_bf16x8(mc); }
};

template <>
struct TfyPack<float> {
    static constexpr int N = 4;
    __device__ static __forceinline__ void unpack(const uint4& v, float* f) {
        f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
        f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    }
    __device__ static __forceinline__ void accum(const uint4& v, float* f) {
        f[0] += __uint_as_float(v.x); f[1] += __uint_as_float(v.y);
        f[2] += __uint_as_float(v.z); f[3] += __uint_as_float(v.w);
    }
    __device__ static __forceinline__ uint4 pack(const float* f) {
        uint4 v;
        v.x = __float_as_uint(f[0]); v.y = __float_as_uint(f[1]);
        v.z = __float_as_uint(f[2]); v.w = __float_as_uint(f[3]);
        return v;
    }
    __device__ static __forceinline__ uint4 mc_ld_reduce(const void* mc) { return tfy_mc_ld_reduce_f32x4(mc); }
};


// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch.  Every hot-path kernel is launched with the programmatic stream
// serialisation attribute and starts with tfy_pdl_sync(): it lets ITS dependents start launching at once
// (all our grids are a single wave, so early dependents never take a slot a primary CTA still needs) and
// then waits for the grids it depends on to complete and flush.  Under stream capture these become
// programmatic edges of the CUDA graph: launch latency and each kernel's prologue (barrier init, tensor-map
// prefetch) overlap the tail of the previous kernel.  Opt-in (TFY_PDL=1); the default is off.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void tfy_pdl_sync() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
#endif

static inline bool tfy_pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("TFY_PDL");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v != 0;
}

// Per-kernel opt-in (TFY_PDL_K4=1): only the fused step is launched with programmatic stream serialisation, so its
// launch latency and the prefetch of its optimizer state overlap the tail of the last backward kernel.
static inline bool tfy_pdl_k4_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("TFY_PDL_K4");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v != 0;
}

#ifdef __CUDACC__
__device__ __forceinline__ void tfy_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void tfy_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

template <typename... KArgs, typename... Args>
static inline cudaError_t tfy_launch_pdl_if(bool enable, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                            cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = enable ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// The same launch for a kernel whose CTAs run in clusters of cluster.x x cluster.y x cluster.z (the grid a multiple of
// it); a 1 x 1 x 1 cluster launches without the cluster attribute.
template <typename... KArgs, typename... Args>
static inline cudaError_t tfy_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 cluster, dim3 block, size_t smem,
                                         cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = tfy_pdl_enabled() ? 1 : 0;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster.x;
    attr[1].val.clusterDim.y = cluster.y;
    attr[1].val.clusterDim.z = cluster.z;
    cfg.attrs = attr;
    cfg.numAttrs = (cluster.x * cluster.y * cluster.z > 1) ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
static inline cudaError_t tfy_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                         Args... args) {
    return tfy_launch_pdl(kernel, grid, dim3(1, 1, 1), block, smem, s, args...);
}
