// Communication kernels over NVLink / NVSwitch peer memory (sm_90a).
//
//   K1  one-shot all-reduce     every rank reads every peer's buffer (latency-optimal, small)
//   K2  two-shot all-reduce     P2P reduce-scatter + P2P all-gather in ONE kernel
//   K3  NVLS all-reduce         multimem.ld_reduce (in-switch sum) + multimem.st (in-switch bcast)
//   K4  fused gradient step     reduce-scatter -> bf16->fp32 cast, 1/N scale -> optimizer update on the
//                               owned fp32 master shard -> all-gather of the updated (bf16|fp32) params,
//                               all inside one kernel; optimizer state is sharded 1/N per rank
//   K7  broadcast               root multicasts (NVLS) or peers pull (P2P)
//   K8  barrier                 see tfy_block_barrier in tfy_common.cuh
//       all-gather              pull-based, used to materialise sharded optimizer state for checkpoints
//
// These replace what the reference delegates to Horovod/gloo, torch-DDP/NCCL
// (reference: tf_yarn/tensorflow/tasks/gloo_allred_task.py:54,72-75,89 and
// tf_yarn/pytorch/tasks/worker.py:101-107).  No NCCL call is made on this path.
#include "tfy_common.cuh"
#include "tfy_fused_step.cuh"

// ---------------------------------------------------------------------------
// reduction of one 16-byte pack across ranks
// ---------------------------------------------------------------------------
template <typename T, int MODE>
__device__ __forceinline__ void tfy_reduce_pack(const TfyCommCtx& c, uint64_t byte_off, float* f) {
    tfy_reduce_pack_rt<T, MODE>(c, MODE, byte_off, f);
}

template <int MODE>
__device__ __forceinline__ void tfy_bcast_pack(const TfyCommCtx& c, uint64_t byte_off, uint4 v) {
    tfy_bcast_pack_rt<MODE>(c, MODE, byte_off, v);
}

// ---------------------------------------------------------------------------
// K1 / K2 / K3   all-reduce
// ---------------------------------------------------------------------------
// `off` is the byte offset of the buffer inside the symmetric arena, identical
// on every rank.  n_packs = number of 16-byte packs (for two-shot / NVLS it must
// be a multiple of world).  Two-shot and NVLS work in place; one-shot writes to
// `out` (a local buffer) because peers may still be reading the input.
// U packs are in flight per thread: every load of a batch is issued before the first store (the asm loads carry
// a memory clobber, so the compiler never overlaps iterations by itself; with one pack in flight per thread a
// full grid holds 1.2 MB, i.e. ~400 GB/s at the ~3 us NVLink round trip -- measured 323 GB/s in round 1).
template <typename T, int ALGO, int U>
__global__ void __launch_bounds__(512) tfy_allreduce_kernel(TfyCommCtx c, uint64_t off, size_t n_packs, float scale,
                                                            uint4* __restrict__ out) {
    using P = TfyPack<T>;
    const uint32_t ep = tfy_grid_epoch(c);
    tfy_grid_entry(c, ep);  // every rank has started this kernel: its input is complete (stream order)
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    if (ALGO == TFY_ALGO_ONESHOT) {
        for (size_t i = tid; i < n_packs; i += nthreads) {
            float f[P::N];
            tfy_reduce_pack<T, TFY_MODE_P2P>(c, off + i * 16, f);
#pragma unroll
            for (int k = 0; k < P::N; ++k) f[k] *= scale;
            out[i] = P::pack(f);
        }
    } else {
        const size_t shard = n_packs / c.world;
        const size_t base = shard * c.rank;
        constexpr int MODE = (ALGO == TFY_ALGO_NVLS) ? TFY_MODE_NVLS : TFY_MODE_P2P;
        const bool unit = (scale == 1.0f);
        for (size_t i0 = tid; i0 < shard; i0 += nthreads * U) {
            if (MODE == TFY_MODE_NVLS) {
                uint4 v[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const size_t i = i0 + (size_t)u * nthreads;
                    if (i < shard) v[u] = P::mc_ld_reduce(reinterpret_cast<const void*>(c.mc_base + off + (base + i) * 16));
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const size_t i = i0 + (size_t)u * nthreads;
                    if (i >= shard) continue;
                    if (!unit) {
                        float f[P::N];
                        P::unpack(v[u], f);
#pragma unroll
                        for (int k = 0; k < P::N; ++k) f[k] *= scale;
                        v[u] = P::pack(f);
                    }
                    tfy_mc_st16(reinterpret_cast<void*>(c.mc_base + off + (base + i) * 16), v[u]);
                }
            } else {
                float f[U][P::N];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const size_t i = i0 + (size_t)u * nthreads;
                    if (i < shard) tfy_reduce_pack<T, MODE>(c, off + (base + i) * 16, f[u]);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const size_t i = i0 + (size_t)u * nthreads;
                    if (i >= shard) continue;
#pragma unroll
                    for (int k = 0; k < P::N; ++k) f[u][k] *= scale;
                    tfy_bcast_pack<MODE>(c, off + (base + i) * 16, P::pack(f[u]));
                }
            }
        }
    }
    tfy_grid_exit(c, ep, false);  // results landed everywhere / every peer is done reading my input
    tfy_grid_finish(c, ep);
}

// ---------------------------------------------------------------------------
// K7 broadcast / all-gather
// ---------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(512) tfy_broadcast_kernel(TfyCommCtx c, uint64_t off, size_t n_packs, int root) {
    tfy_block_barrier(c);
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    if (MODE == TFY_MODE_NVLS) {
        if (c.rank == root)
            for (size_t i = tid; i < n_packs; i += nthreads) {
                uint4 v = tfy_ld16(reinterpret_cast<const void*>(c.peer_base[root] + off + i * 16));
                tfy_mc_st16(reinterpret_cast<void*>(c.mc_base + off + i * 16), v);
            }
    } else {
        if (c.rank != root)
            for (size_t i = tid; i < n_packs; i += nthreads) {
                uint4 v = tfy_ld16_stream(reinterpret_cast<const void*>(c.peer_base[root] + off + i * 16));
                tfy_st16(reinterpret_cast<void*>(c.peer_base[c.rank] + off + i * 16), v);
            }
    }
    tfy_block_barrier(c);
}

// buffer layout [world][shard_packs]; rank r owns slice r of its own replica
__global__ void __launch_bounds__(512) tfy_allgather_kernel(TfyCommCtx c, uint64_t off, size_t shard_packs) {
    tfy_block_barrier(c);
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    for (int rr = 1; rr < c.world; ++rr) {
        int r = c.rank + rr;
        if (r >= c.world) r -= c.world;
        const uint64_t bo = off + (uint64_t)r * shard_packs * 16;
        for (size_t i = tid; i < shard_packs; i += nthreads) {
            uint4 v = tfy_ld16_stream(reinterpret_cast<const void*>(c.peer_base[r] + bo + i * 16));
            tfy_st16(reinterpret_cast<void*>(c.peer_base[c.rank] + bo + i * 16), v);
        }
    }
    tfy_block_barrier(c);
}

__global__ void tfy_barrier_kernel(TfyCommCtx c) { tfy_block_barrier(c); }

// ---------------------------------------------------------------------------
// K4  fused reduce-scatter -> optimizer -> all-gather
// ---------------------------------------------------------------------------
// GT: gradient dtype in the symmetric grad buffer, PT: dtype of the replicated
// compute parameters.  master/s1/s2: local fp32 arrays of shard_n elements
// (rank r owns elements [r*shard_n, (r+1)*shard_n) of the flat buffers); RMSprop's s2 holds up to two states
// back to back (tfy_rmsprop_states).  For Nadam, hp heads a TfyNadamHyperBlock.
// [g_lo, g_hi): shard-relative groups of 8 elements this launch handles (the whole shard for the classic single
// launch).  Splitting a step into ranges lets the engine run the update of gradients that are final early (the
// big Dense kernel) inside the convolution-backward kernel (tfy_overlap_role) while this launch only handles the
// rest; `advance` is set on the last launch of a step only, so every range of the step sees the same step counter.
// Minimum resident CTAs per SM of an instantiation (__launch_bounds__): 0 (none) for the constant-rate kernels, whose
// code is as before.  The scheduled ones are held to the occupancy of their constant-rate twins, which the schedule's
// tail would otherwise lower: 3 CTAs of 128 threads (at most 80 registers) in LOCAL mode, and in the multi-GPU modes
// 2 CTAs of 256 threads (at most 128 registers, which every optimizer but RMSprop fits) -- the grid of a multi-GPU
// step (up to 2 CTAs per SM) must be resident, since with zero_grads every CTA waits at the exit barrier.
constexpr int tfy_k4_min_blocks(int opt, int mode, bool sched) {
    return !sched ? 0 : mode == TFY_MODE_LOCAL ? 3 : opt == TFY_OPT_RMSPROP ? 1 : 2;
}

// SCHED (launched with TFY_OPT_LR_SCHEDULE): hp heads a TfyHyperBlock, and advancing the step also writes the
// scheduled learning rate of the next one.
template <typename GT, typename PT, int OPT, int MODE, int U, bool SCHED = false>
__global__ void __launch_bounds__(256, tfy_k4_min_blocks(OPT, MODE, SCHED))
tfy_fused_step_kernel(TfyCommCtx c, uint64_t grad_off, uint64_t param_off, size_t shard_n,
                      float* __restrict__ master, float* __restrict__ s1, float* __restrict__ s2,
                      TfyOptHyper* __restrict__ hp, int zero_grads, size_t g_lo, size_t g_hi, int advance) {
    // Everything up to tfy_pdl_wait() only touches data this kernel itself wrote in the previous step (hyper
    // block, master, optimizer state): with programmatic dependent launch it overlaps the tail of the last
    // backward kernel.
    tfy_pdl_launch_dependents();
    using GP = TfyPack<GT>;
    constexpr int NG = 8 / GP::N;  // 16-byte packs per 8 gradient elements
    const size_t shard_start = (MODE == TFY_MODE_LOCAL) ? 0 : shard_n * (size_t)c.rank;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    const size_t tid = g_lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x;

    // The owned master / optimizer-state shard does not depend on the peers (nor, with programmatic dependent
    // launch, on the preceding backward kernel): its loads are issued BEFORE the dependency wait, the cross-GPU
    // barrier and the (2-3 us) in-switch reduction, so their latency hides behind all three.  (TFY_PDL_K4=1
    // assumes a different kernel separates two fused-step launches on the stream -- true for every train step.)
    TfyStepRegs<U, OPT == TFY_OPT_RMSPROP> r;
    float* s3 = nullptr;
    if constexpr (OPT == TFY_OPT_RMSPROP) tfy_rmsprop_states(hp, shard_n, s2, s3);
    tfy_step_load_state<OPT, U>(r, OPT, master, s1, s2, tid, nthreads, g_hi, s3);
    tfy_pdl_wait();                                     // the gradients of THIS rank are complete
    const TfyStepConsts k = tfy_step_consts(hp, c.world, OPT);
    const int step = hp->step;
    const uint32_t ep = (MODE != TFY_MODE_LOCAL) ? tfy_grid_epoch(c) : 0u;

    if (MODE != TFY_MODE_LOCAL) tfy_grid_entry(c, ep);  // all ranks finished backward

    for (size_t g8 = tid; g8 < g_hi; g8 += nthreads * U) {
        tfy_step_batch<GT, PT, OPT, MODE, U>(c, OPT, MODE, k, r, grad_off, param_off, shard_start, master, s1, s2, g8,
                                             nthreads, g_hi, s3);
        if (g8 + nthreads * U < g_hi)
            tfy_step_load_state<OPT, U>(r, OPT, master, s1, s2, g8 + nthreads * U, nthreads, g_hi, s3);
    }

    // updated params visible on every rank before the grid completes; with zero_grads every CTA waits, because it
    // goes on to clear gradients the peers were reading
    if (MODE != TFY_MODE_LOCAL) tfy_grid_exit(c, ep, zero_grads != 0);

    if (zero_grads) {
        // Clear the gradient replica for the next accumulation: after the exit barrier every CTA of EVERY rank
        // has finished reading, so this thread clears the groups `tid + k*nthreads` of every shard in the LOCAL
        // replica.
        const uint4 z = make_uint4(0, 0, 0, 0);
        char* gb = reinterpret_cast<char*>(c.peer_base[c.rank] + grad_off);
        const int nshards = (MODE == TFY_MODE_LOCAL) ? 1 : c.world;
        for (int rr = 0; rr < nshards; ++rr) {
            for (size_t g8 = tid; g8 < g_hi; g8 += nthreads) {
                char* p = gb + ((size_t)rr * shard_n + g8 * 8) * sizeof(GT);
#pragma unroll
                for (int q = 0; q < NG; ++q) tfy_st16(p + q * 16, z);
            }
        }
    }

    // advance the device-side step counter (and a scheduled learning rate) exactly once per launch
    if (MODE != TFY_MODE_LOCAL) {
        if (tfy_grid_finish(c, ep) && threadIdx.x == 0 && advance) {
            if constexpr (SCHED) tfy_advance_scheduled_step(hp, step);
            else hp->step = step + 1;
            if constexpr (OPT == TFY_OPT_NADAM) tfy_nadam_advance(hp, k);
        }
    } else {
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            const uint32_t prev = atomicAdd(&hp->done, 1u);
            if (prev == gridDim.x - 1) {
                hp->done = 0;
                if (advance) {
                    if constexpr (SCHED) tfy_advance_scheduled_step(hp, step);
                    else hp->step = step + 1;
                    if constexpr (OPT == TFY_OPT_NADAM) tfy_nadam_advance(hp, k);
                }
            }
        }
    }
}

// hp->lr = schedule(hp->step) of a TfyHyperBlock: the rate of the next step when the step counter is installed or
// restored, by the same device function the scheduled fused step evaluates
__global__ void tfy_lr_schedule_sync_kernel(TfyOptHyper* hp) {
    if (threadIdx.x == 0 && blockIdx.x == 0)
        hp->lr = tfy_lr_schedule_eval(reinterpret_cast<const TfyHyperBlock*>(hp)->sched, (int64_t)hp->step);
}

// ---------------------------------------------------------------------------
// host launchers (C ABI, called through ctypes; stream = raw cudaStream_t)
// ---------------------------------------------------------------------------
static inline int tfy_pick_grid(size_t work_items, int block, int max_grid) {
    size_t g = (work_items + block - 1) / block;
    if (g < 1) g = 1;
    if (g > (size_t)max_grid) g = max_grid;
    return (int)g;
}

// Largest grid of `kernel` whose CTAs are all resident at once.  A multi-GPU fused step needs that: with zero_grads
// every CTA waits at the exit barrier for the last one to arrive, so a CTA that has to wait for a free SM never
// starts.  The RMSprop instantiations take more than 128 registers and fit one 256-thread CTA per SM, not two.
template <typename K>
static int tfy_resident_grid(K kernel, int grid, int block) {
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0) != cudaSuccess)
        return grid;
    const int cap = per_sm * sms;
    return cap > 0 && grid > cap ? cap : grid;
}

extern "C" {

int tfy_lr_schedule_sync(TfyOptHyper* hp, cudaStream_t s) {
    tfy_lr_schedule_sync_kernel<<<1, 32, 0, s>>>(hp);
    return (int)cudaGetLastError();
}

int tfy_barrier(const TfyCommCtx* c, int grid, cudaStream_t s) {
    if (grid < 1) grid = 1;
    tfy_barrier_kernel<<<grid, 32, 0, s>>>(*c);
    return (int)cudaGetLastError();
}

// n = number of elements; must be a multiple of (16/sizeof(T)) [* world for algo 1,2]
int tfy_allreduce(const TfyCommCtx* c, int dtype, int algo, uint64_t off, size_t n, float scale, void* out,
                  int grid, int block, cudaStream_t s) {
    const size_t esz = dtype == TFY_BF16 ? 2 : 4;
    const size_t n_packs = n * esz / 16;
    if (n_packs * 16 != n * esz) return -2;
    if (algo != TFY_ALGO_ONESHOT && (n_packs % c->world) != 0) return -3;
    if (algo == TFY_ALGO_ONESHOT && out == nullptr) return -4;
    if (algo == TFY_ALGO_NVLS && c->mc_base == 0) return -5;
    if (block <= 0) block = 512;
    const size_t work = algo == TFY_ALGO_ONESHOT ? n_packs : n_packs / c->world;
    // small messages: one pack per thread (a single NVLink round trip); large ones: 2 CTAs per SM x 4 packs in flight
    if (grid <= 0) grid = tfy_pick_grid(work, block, TFY_NUM_SMS * 2);
    if (grid > TFY_MAX_BLOCKS) grid = TFY_MAX_BLOCKS;
#define TFY_AR(T, A) tfy_allreduce_kernel<T, A, 4><<<grid, block, 0, s>>>(*c, off, n_packs, scale, (uint4*)out)
    if (dtype == TFY_BF16) {
        if (algo == TFY_ALGO_ONESHOT) TFY_AR(__nv_bfloat16, TFY_ALGO_ONESHOT);
        else if (algo == TFY_ALGO_TWOSHOT) TFY_AR(__nv_bfloat16, TFY_ALGO_TWOSHOT);
        else TFY_AR(__nv_bfloat16, TFY_ALGO_NVLS);
    } else {
        if (algo == TFY_ALGO_ONESHOT) TFY_AR(float, TFY_ALGO_ONESHOT);
        else if (algo == TFY_ALGO_TWOSHOT) TFY_AR(float, TFY_ALGO_TWOSHOT);
        else TFY_AR(float, TFY_ALGO_NVLS);
    }
#undef TFY_AR
    return (int)cudaGetLastError();
}

int tfy_broadcast(const TfyCommCtx* c, uint64_t off, size_t nbytes, int root, int use_nvls, int grid, int block,
                  cudaStream_t s) {
    if (nbytes % 16) return -2;
    const size_t n_packs = nbytes / 16;
    if (block <= 0) block = 512;
    if (grid <= 0) grid = tfy_pick_grid(n_packs, block * 2, TFY_NUM_SMS);
    if (grid > TFY_MAX_BLOCKS) grid = TFY_MAX_BLOCKS;
    if (use_nvls && c->mc_base)
        tfy_broadcast_kernel<TFY_MODE_NVLS><<<grid, block, 0, s>>>(*c, off, n_packs, root);
    else
        tfy_broadcast_kernel<TFY_MODE_P2P><<<grid, block, 0, s>>>(*c, off, n_packs, root);
    return (int)cudaGetLastError();
}

int tfy_allgather(const TfyCommCtx* c, uint64_t off, size_t shard_bytes, int grid, int block, cudaStream_t s) {
    if (shard_bytes % 16) return -2;
    const size_t shard_packs = shard_bytes / 16;
    if (block <= 0) block = 512;
    if (grid <= 0) grid = tfy_pick_grid(shard_packs, block * 2, TFY_NUM_SMS);
    if (grid > TFY_MAX_BLOCKS) grid = TFY_MAX_BLOCKS;
    tfy_allgather_kernel<<<grid, block, 0, s>>>(*c, off, shard_packs);
    return (int)cudaGetLastError();
}

// The fused gradient step.  shard_n: elements owned by each rank (multiple of 8).
// mode: 0 local (world==1), 1 P2P, 2 NVLS.
static int tfy_fused_step_groups(const TfyCommCtx* c, int grad_dtype, int param_dtype, int opt, int mode,
                                 uint64_t grad_off, uint64_t param_off, size_t shard_n, float* master, float* s1,
                                 float* s2, TfyOptHyper* hp, int zero_grads, int grid, int block, size_t g_lo,
                                 size_t g_hi, size_t span_groups, int advance, cudaStream_t s) {
    if (mode == TFY_MODE_NVLS && c->mc_base == 0) return -5;
    const bool sched = (opt & TFY_OPT_LR_SCHEDULE) != 0;
    opt &= ~TFY_OPT_LR_SCHEDULE;
    if (block <= 0) block = (mode == TFY_MODE_LOCAL) ? 128 : 256;
    // single GPU: nothing to synchronise with, so oversubscribe the SMs for memory-level parallelism;
    // multi GPU: the cross-GPU barriers are grid-level (one signal per rank pair), 2 groups in flight per thread
    if (grid <= 0) grid = tfy_pick_grid(span_groups + 1, block * (mode == TFY_MODE_LOCAL ? 1 : 2),
                                        mode == TFY_MODE_LOCAL ? TFY_NUM_SMS * 6 : TFY_NUM_SMS * 2);
    if (grid > TFY_MAX_BLOCKS) grid = TFY_MAX_BLOCKS;
#define TFY_FS5(GT, PT, O, M, U, S)                                                                              \
    do {                                                                                                         \
        if (M != TFY_MODE_LOCAL) grid = tfy_resident_grid(tfy_fused_step_kernel<GT, PT, O, M, U, S>, grid, block); \
        tfy_launch_pdl_if(tfy_pdl_enabled() || tfy_pdl_k4_enabled(), (tfy_fused_step_kernel<GT, PT, O, M, U, S>), dim3(grid), dim3(block), 0, s, *c, grad_off, param_off, \
                       shard_n, master, s1, s2, hp, zero_grads, g_lo, g_hi, advance);                          \
    } while (0)
#define TFY_FS4(GT, PT, O, M, U)                          \
    do {                                                  \
        if (sched) TFY_FS5(GT, PT, O, M, U, true);        \
        else TFY_FS5(GT, PT, O, M, U, false);             \
    } while (0)
#define TFY_FS3(GT, PT, O)                                                  \
    do {                                                                    \
        if (mode == TFY_MODE_LOCAL) TFY_FS4(GT, PT, O, TFY_MODE_LOCAL, 1);  \
        else if (mode == TFY_MODE_P2P) TFY_FS4(GT, PT, O, TFY_MODE_P2P, 2); \
        else TFY_FS4(GT, PT, O, TFY_MODE_NVLS, 2);                          \
    } while (0)
#define TFY_FS2(GT, PT)                                            \
    do {                                                           \
        if (opt == TFY_OPT_SGD) TFY_FS3(GT, PT, TFY_OPT_SGD);      \
        else if (opt == TFY_OPT_ADADELTA) TFY_FS3(GT, PT, TFY_OPT_ADADELTA); \
        else if (opt == TFY_OPT_ADAM) TFY_FS3(GT, PT, TFY_OPT_ADAM); \
        else if (opt == TFY_OPT_FTRL) TFY_FS3(GT, PT, TFY_OPT_FTRL); \
        else if (opt == TFY_OPT_RMSPROP) TFY_FS3(GT, PT, TFY_OPT_RMSPROP); \
        else if (opt == TFY_OPT_ADAMAX) TFY_FS3(GT, PT, TFY_OPT_ADAMAX); \
        else if (opt == TFY_OPT_NADAM) TFY_FS3(GT, PT, TFY_OPT_NADAM); \
        else TFY_FS3(GT, PT, TFY_OPT_ADAGRAD);                     \
    } while (0)
    if (grad_dtype == TFY_BF16 && param_dtype == TFY_BF16) TFY_FS2(__nv_bfloat16, __nv_bfloat16);
    else if (grad_dtype == TFY_F32 && param_dtype == TFY_F32) TFY_FS2(float, float);
    else if (grad_dtype == TFY_BF16 && param_dtype == TFY_F32) TFY_FS2(__nv_bfloat16, float);
    else TFY_FS2(float, __nv_bfloat16);
#undef TFY_FS2
#undef TFY_FS3
#undef TFY_FS4
#undef TFY_FS5
    return (int)cudaGetLastError();
}

// element range [e0, e1) of the FLAT buffers (multiples of 8; e1 is clamped to the buffer): every rank handles the
// part of the range that falls into the shard it owns
int tfy_fused_step_range(const TfyCommCtx* c, int grad_dtype, int param_dtype, int opt, int mode, uint64_t grad_off,
                         uint64_t param_off, size_t shard_n, float* master, float* s1, float* s2, TfyOptHyper* hp,
                         int zero_grads, int grid, int block, size_t e0, size_t e1, int advance, cudaStream_t s) {
    if (shard_n % 8 || e0 % 8 || (e1 != (size_t)-1 && e1 % 8)) return -2;
    const size_t total = shard_n * (size_t)(mode == TFY_MODE_LOCAL ? 1 : c->world);
    if (e1 > total) e1 = total;
    if (e0 > e1) e0 = e1;
    const size_t shard_start = (mode == TFY_MODE_LOCAL) ? 0 : shard_n * (size_t)c->rank;
    const size_t lo_e = e0 > shard_start ? e0 - shard_start : 0;
    const size_t hi_e = e1 > shard_start ? e1 - shard_start : 0;
    const size_t g_lo = (lo_e < shard_n ? lo_e : shard_n) / 8;
    const size_t g_hi = (hi_e < shard_n ? hi_e : shard_n) / 8;
    // grid from the work of the busiest rank (the largest overlap of [e0, e1) with one shard): identical on every rank
    size_t span = e1 - e0;
    if (span > shard_n) span = shard_n;
    return tfy_fused_step_groups(c, grad_dtype, param_dtype, opt, mode, grad_off, param_off, shard_n, master, s1, s2,
                                 hp, zero_grads, grid, block, g_lo, g_hi, span / 8, advance, s);
}

// SHARD-RELATIVE groups of 8 elements [g0, g1) on every rank (the balanced split used when part of the step is
// overlapped with backward: each rank overlaps the same fraction of ITS shard)
int tfy_fused_step_shard_range(const TfyCommCtx* c, int grad_dtype, int param_dtype, int opt, int mode,
                               uint64_t grad_off, uint64_t param_off, size_t shard_n, float* master, float* s1,
                               float* s2, TfyOptHyper* hp, int zero_grads, int grid, int block, size_t g0, size_t g1,
                               int advance, cudaStream_t s) {
    if (shard_n % 8) return -2;
    if (g1 > shard_n / 8) g1 = shard_n / 8;
    if (g0 > g1) g0 = g1;
    return tfy_fused_step_groups(c, grad_dtype, param_dtype, opt, mode, grad_off, param_off, shard_n, master, s1, s2,
                                 hp, zero_grads, grid, block, g0, g1, g1 - g0, advance, s);
}

int tfy_fused_step(const TfyCommCtx* c, int grad_dtype, int param_dtype, int opt, int mode, uint64_t grad_off,
                   uint64_t param_off, size_t shard_n, float* master, float* s1, float* s2, TfyOptHyper* hp,
                   int zero_grads, int grid, int block, cudaStream_t s) {
    return tfy_fused_step_range(c, grad_dtype, param_dtype, opt, mode, grad_off, param_off, shard_n, master, s1, s2,
                                hp, zero_grads, grid, block, 0, (size_t)-1, 1, s);
}

}  // extern "C"
