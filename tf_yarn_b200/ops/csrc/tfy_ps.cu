// Parameter-server data plane over NVLink peer memory (sm_90a): K5 pull / K6 push.
//
// A ps rank owns shards in ITS HBM (inside the symmetric arena); chief/worker ranks map them and
// run these kernels against the peer addresses -- there is no server thread on the data path
// (reference path being replaced: TF gRPC RecvTensor pulls and Apply*/SparseApply*/ScatterAdd on the
// ps task, tf_yarn/tensorflow/cluster.py:41-67, tf_task_common.py:46-50).
//
//   pull   dense : peer fp32 master -> local replica (fp32 or bf16), 16-byte peer loads
//          sparse: gather the rows of a batch from a peer embedding table, fused with the bag
//                  reduction (sum / mean) that consumes them
//          GEMM  : weights stay remote and are streamed by TMA into the wgmma GEMM (tfy_gemm.cu)
//   push   dense : every worker applies its gradient to the peer master with red/atom -- asynchronous,
//                  lock free (TF's use_locking=False semantics), optimizer fused, chosen PER VARIABLE (wide-and-deep
//                  trains its linear tower with FTRL and its deep tower with Adagrad):
//                    SGD      w   += -lr*g                                       (red.v4.f32)
//                    Adagrad  acc += g^2 ; w += -lr*g/(sqrt(acc)+eps)            (atom.v4.f32 returns old acc)
//                    FTRL     n += g^2 ; z += g - (sqrt(n')-sqrt(n))/lr * w ;    (two atom.v4.f32)
//                             w  = |z|<=l1 ? 0 : -(z - sgn(z) l1) / ((beta+sqrt(n'))/lr + 2 l2)
//                    Adam     m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ;      (read-modify-write of m, v)
//                             w += -lr/(1-b1^t) m/(sqrt(v)/sqrt(1-b2^t)+eps)     (red.v4.f32; torch's formula, as
//                                                                                 K4 and the CPU plane)
//                  and refreshes the bf16 shadow copy that the GEMM pull reads
//          sparse: the same per touched embedding row.  The ids of one push are folded first: every distinct
//                  (table, row) receives the SUM of its gradients (x 1/L for a mean bag) and its optimizer runs ONCE,
//                  like TF's SparseApply* on IndexedSlices with repeated indices summed.  The fold is a stable radix
//                  sort of the (table, id) keys into caller-provided scratch, then the apply kernels, which reduce
//                  every run in a fixed order (a thread per short run, a warp per long one): a push is deterministic
//                  and needs no host synchronisation (capturable).  Rows outside the batch are not touched, Adam's
//                  m and v included (lazy Adam).  Out-of-range ids (< 0 or >= V) are skipped.
//   multi-hot / weighted (TF's embedding_column combiners), T tables x L ids per example, weight w (1 if none):
//          an occurrence is present iff 0 <= id < V and w != 0.  S = sum_present w row, out = S / den with
//          den = 1 (sum), sum_present w (mean), sqrt(sum_present w^2) (sqrtn), and 0 where den == 0.
//          tfy_ps_multi_bag_weighted writes out (a column slice per table, or all tables summed) and f = 1/den;
//          tfy_ps_multi_push_rows_weighted is the fold above with a compile-time weighted flag: zero weights get
//          the sentinel key, one more kernel writes every occurrence's factor w f into the sort's free buffer, and
//          the apply kernels add w f g in the sorted order.  The unweighted instantiations are unchanged; K5 and the
//          one-id kernels keep serving one-hot unweighted batches.
#include <cub/block/block_radix_sort.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "tfy_common.cuh"

struct TfyPsSeg {
    uint64_t remote_w;       // peer fp32 master
    uint64_t remote_s1;      // peer fp32 optimizer slot 1 (Adagrad / FTRL accumulator, Adam m), 0 if none
    uint64_t remote_s2;      // peer fp32 optimizer slot 2 (FTRL linear z, Adam v), 0 if none
    uint64_t remote_shadow;  // peer bf16 shadow of the master, 0 if none
    uint64_t local;          // local replica (pull destination) / local gradient (push source)
    uint64_t n;              // elements
    int32_t opt;             // TfyOpt of THIS variable
    float lr, eps, wd;
    float p1, p2, p3;        // FTRL: l1, l2, beta | Adam: beta1, beta2, -
    int32_t pad;
    // bf16 shadow of a 2-D weight [rows, cols]: rows are `shadow_ld` elements apart (cols rounded up to 8 so that
    // a TMA tensor map can describe it); cols == 0 means "flat, same indexing as the master"
    uint32_t cols, shadow_ld;
};

// optimizer hyper-parameters of one push (sparse rows: passed by value)
struct TfyPsHyper {
    int32_t opt;
    float lr, eps, wd, p1, p2, p3, grad_scale;
};

namespace {

__device__ __forceinline__ void red_add_f32x4(void* p, float4 v) {
    asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ float4 atom_add_f32x4(void* p, float4 v) {
    float4 o;
    asm volatile("atom.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4], {%5,%6,%7,%8};"
                 : "=f"(o.x), "=f"(o.y), "=f"(o.z), "=f"(o.w)
                 : "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
    return o;
}
// element index of the master -> element index of the (row-padded) shadow
__device__ __forceinline__ size_t shadow_index(size_t i, uint32_t cols, uint32_t ld) {
    return cols ? (i / cols) * (size_t)ld + (i % cols) : i;
}
__device__ __forceinline__ void st_shadow4(__nv_bfloat16* shadow, size_t i, float4 v, uint32_t cols, uint32_t ld);

__device__ __forceinline__ void st_shadow_bf16x4(void* p, float4 v) {
    uint2 u;
    u.x = tfy_pack_bf16x2(v.x, v.y);
    u.y = tfy_pack_bf16x2(v.z, v.w);
    asm volatile("st.global.relaxed.sys.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(u.x), "r"(u.y) : "memory");
}

__device__ __forceinline__ void st_shadow4(__nv_bfloat16* shadow, size_t i, float4 v, uint32_t cols, uint32_t ld) {
    if (cols == 0 || ((cols & 3u) == 0 && (ld & 3u) == 0)) {
        st_shadow_bf16x4(shadow + shadow_index(i, cols, ld), v);       // the 4-pack stays inside one row
    } else {
        const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) shadow[shadow_index(i + k, cols, ld)] = __float2bfloat16(f[k]);
    }
}

template <typename T>
__device__ __forceinline__ float4 ld_local4(const T* p);
template <>
__device__ __forceinline__ float4 ld_local4<float>(const float* p) {
    return *reinterpret_cast<const float4*>(p);
}
template <>
__device__ __forceinline__ float4 ld_local4<__nv_bfloat16>(const __nv_bfloat16* p) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    return make_float4(tfy_bf16lo(u.x), tfy_bf16hi(u.x), tfy_bf16lo(u.y), tfy_bf16hi(u.y));
}
template <typename T>
__device__ __forceinline__ void st_local4(T* p, float4 v);
template <>
__device__ __forceinline__ void st_local4<float>(float* p, float4 v) {
    *reinterpret_cast<float4*>(p) = v;
}
template <>
__device__ __forceinline__ void st_local4<__nv_bfloat16>(__nv_bfloat16* p, float4 v) {
    uint2 u;
    u.x = tfy_pack_bf16x2(v.x, v.y);
    u.y = tfy_pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(p) = u;
}

}  // namespace

// ------------------------------------------------------------------------------------- dense pull
template <typename LT>
__global__ void __launch_bounds__(256) tfy_ps_pull_kernel(const TfyPsSeg* __restrict__ segs) {
    const TfyPsSeg sg = segs[blockIdx.y];
    const float* src = reinterpret_cast<const float*>(sg.remote_w);
    LT* dst = reinterpret_cast<LT*>(sg.local);
    const size_t n4 = sg.n / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
        st_local4<LT>(dst + i * 4, tfy_ld_peer_f32x4(src + i * 4));
    if (blockIdx.x == 0)   // scalar tail (n % 4 elements)
        for (size_t i = n4 * 4 + threadIdx.x; i < sg.n; i += blockDim.x) dst[i] = (LT)src[i];
}

// ------------------------------------------------------------------------------------- dense push
namespace {

__device__ __forceinline__ float4 f4_mul(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ void st_peer_f32x4(void* p, float4 v) {
    asm volatile("st.global.relaxed.sys.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ float ftrl_w(float z, float n_new, float lr, float l1, float l2, float beta) {
    if (fabsf(z) <= l1) return 0.f;
    return -(z - copysignf(l1, z)) / ((beta + sqrtf(n_new)) / lr + 2.f * l2);
}

// One 4-element pack of an asynchronous update against the peer master: gv already scaled (and decayed).
// Returns the new weights when they are known (needed for the bf16 shadow), via `neww`; `want_new` tells whether
// the caller must refresh the shadow from them (true whenever a shadow exists).  Adam: lr already carries
// 1/(1-b1^t), vs = 1/sqrt(1-b2^t).
__device__ __forceinline__ void ps_apply4(int opt, float* w, float* s1, float* s2, float4 gv, float lr, float eps,
                                          float p1, float p2, float p3, float vs, bool want_new, float4& neww) {
    if (opt == TFY_OPT_FTRL) {
        const float4 g2 = make_float4(gv.x * gv.x, gv.y * gv.y, gv.z * gv.z, gv.w * gv.w);
        const float4 n_old = atom_add_f32x4(s1, g2);
        const float4 n_new = make_float4(n_old.x + g2.x, n_old.y + g2.y, n_old.z + g2.z, n_old.w + g2.w);
        const float4 wv = tfy_ld_peer_f32x4(w);
        const float inv_lr = 1.f / lr;
        const float4 dz = make_float4(gv.x - (sqrtf(n_new.x) - sqrtf(n_old.x)) * inv_lr * wv.x,
                                      gv.y - (sqrtf(n_new.y) - sqrtf(n_old.y)) * inv_lr * wv.y,
                                      gv.z - (sqrtf(n_new.z) - sqrtf(n_old.z)) * inv_lr * wv.z,
                                      gv.w - (sqrtf(n_new.w) - sqrtf(n_old.w)) * inv_lr * wv.w);
        const float4 z_old = atom_add_f32x4(s2, dz);
        neww = make_float4(ftrl_w(z_old.x + dz.x, n_new.x, lr, p1, p2, p3), ftrl_w(z_old.y + dz.y, n_new.y, lr, p1, p2, p3),
                           ftrl_w(z_old.z + dz.z, n_new.z, lr, p1, p2, p3), ftrl_w(z_old.w + dz.w, n_new.w, lr, p1, p2, p3));
        st_peer_f32x4(w, neww);        // w is a pure function of (z, n): last writer wins, as in TF without locking
        return;
    }
    float4 delta;
    if (opt == TFY_OPT_ADAGRAD) {
        const float4 g2 = make_float4(gv.x * gv.x, gv.y * gv.y, gv.z * gv.z, gv.w * gv.w);
        const float4 old = atom_add_f32x4(s1, g2);
        delta.x = -lr * gv.x / (sqrtf(old.x + g2.x) + eps);
        delta.y = -lr * gv.y / (sqrtf(old.y + g2.y) + eps);
        delta.z = -lr * gv.z / (sqrtf(old.z + g2.z) + eps);
        delta.w = -lr * gv.w / (sqrtf(old.w + g2.w) + eps);
    } else if (opt == TFY_OPT_ADAM) {
        float4 m = tfy_ld_peer_f32x4(s1), v = tfy_ld_peer_f32x4(s2);
        m = make_float4(p1 * m.x + (1.f - p1) * gv.x, p1 * m.y + (1.f - p1) * gv.y, p1 * m.z + (1.f - p1) * gv.z,
                        p1 * m.w + (1.f - p1) * gv.w);
        v = make_float4(p2 * v.x + (1.f - p2) * gv.x * gv.x, p2 * v.y + (1.f - p2) * gv.y * gv.y,
                        p2 * v.z + (1.f - p2) * gv.z * gv.z, p2 * v.w + (1.f - p2) * gv.w * gv.w);
        st_peer_f32x4(s1, m);
        st_peer_f32x4(s2, v);
        delta = make_float4(-lr * m.x / (sqrtf(v.x) * vs + eps), -lr * m.y / (sqrtf(v.y) * vs + eps),
                            -lr * m.z / (sqrtf(v.z) * vs + eps), -lr * m.w / (sqrtf(v.w) * vs + eps));
    } else {
        delta = f4_mul(gv, -lr);
    }
    if (want_new) {
        const float4 old = atom_add_f32x4(w, delta);
        neww = make_float4(old.x + delta.x, old.y + delta.y, old.z + delta.z, old.w + delta.w);
    } else {
        red_add_f32x4(w, delta);
    }
}

__device__ __forceinline__ float ps_apply1(int opt, float* w, float* s1, float* s2, float g, float lr, float eps, float p1,
                                           float p2, float p3, float vs) {
    if (opt == TFY_OPT_FTRL) {
        const float n_old = atomicAdd(s1, g * g), n_new = n_old + g * g;
        const float dz = g - (sqrtf(n_new) - sqrtf(n_old)) / lr * *w;
        const float z = atomicAdd(s2, dz) + dz;
        const float nw = ftrl_w(z, n_new, lr, p1, p2, p3);
        *w = nw;
        return nw;
    }
    float delta;
    if (opt == TFY_OPT_ADAGRAD) {
        const float old = atomicAdd(s1, g * g);
        delta = -lr * g / (sqrtf(old + g * g) + eps);
    } else if (opt == TFY_OPT_ADAM) {
        const float m = p1 * *s1 + (1.f - p1) * g, v = p2 * *s2 + (1.f - p2) * g * g;
        *s1 = m; *s2 = v;
        delta = -lr * m / (sqrtf(v) * vs + eps);
    } else {
        delta = -lr * g;
    }
    return atomicAdd(w, delta) + delta;
}

// Adam's bias correction: adam_scale = {1/(1-b1^t), 1/sqrt(1-b2^t)} in device memory (so that a captured CUDA graph
// sees it advance); nullptr = no correction.  Returns the learning rate to use and sets `vs`.
__device__ __forceinline__ float ps_adam_lr(int opt, float lr, const float* adam_scale, float& vs) {
    vs = 1.f;
    if (opt != TFY_OPT_ADAM || !adam_scale) return lr;
    vs = adam_scale[1];
    return lr * adam_scale[0];
}

}  // namespace

// The optimizer is a per-segment (= per-variable) runtime value (uniform per blockIdx.y).  grad_scale multiplies the
// local gradient first.
template <typename GT>
__global__ void __launch_bounds__(256)
tfy_ps_push_kernel(const TfyPsSeg* __restrict__ segs, float grad_scale, const float* __restrict__ adam_scale) {
    const TfyPsSeg sg = segs[blockIdx.y];
    float* w = reinterpret_cast<float*>(sg.remote_w);
    float* s1 = reinterpret_cast<float*>(sg.remote_s1);
    float* s2 = reinterpret_cast<float*>(sg.remote_s2);
    __nv_bfloat16* shadow = reinterpret_cast<__nv_bfloat16*>(sg.remote_shadow);
    const GT* g = reinterpret_cast<const GT*>(sg.local);
    const int opt = sg.opt;
    const float wd = sg.wd, eps = sg.eps, p1 = sg.p1, p2 = sg.p2, p3 = sg.p3;
    float vs;
    const float lr = ps_adam_lr(opt, sg.lr, adam_scale, vs);
    const size_t n4 = sg.n / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 gv = f4_mul(ld_local4<GT>(g + i * 4), grad_scale);
        if (wd != 0.f) {
            const float4 wv = tfy_ld_peer_f32x4(w + i * 4);
            gv.x += wd * wv.x; gv.y += wd * wv.y; gv.z += wd * wv.z; gv.w += wd * wv.w;
        }
        float4 neww;
        ps_apply4(opt, w + i * 4, s1 + i * 4, s2 + i * 4, gv, lr, eps, p1, p2, p3, vs, shadow != nullptr, neww);
        if (shadow) st_shadow4(shadow, i * 4, neww, sg.cols, sg.shadow_ld);
    }
    if (blockIdx.x == 0) {   // scalar tail (n % 4 elements)
        for (size_t i = n4 * 4 + threadIdx.x; i < sg.n; i += blockDim.x) {
            float gv = (float)g[i] * grad_scale;
            if (wd != 0.f) gv += wd * w[i];
            const float nw = ps_apply1(opt, w + i, s1 + i, s2 + i, gv, lr, eps, p1, p2, p3, vs);
            if (shadow) shadow[shadow_index(i, sg.cols, sg.shadow_ld)] = __float2bfloat16(nw);
        }
    }
}

// ------------------------------------------------------------------------------------ sparse pull
// out[b, :] = reduce_j table[ids[b, j], :]   (mode 0 sum, 1 mean); table is a PEER fp32 [V, D], D % 4 == 0.
template <typename OT>
__global__ void __launch_bounds__(256)
tfy_ps_embedding_bag_kernel(const float* __restrict__ table, const long long* __restrict__ ids, OT* __restrict__ out,
                            int B, int L, int D, long long V, int mean) {
    const int D4 = D / 4;
    const size_t total = (size_t)B * D4;
    const float scale = mean ? 1.f / (float)L : 1.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = i / D4, d = (i % D4) * 4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < L; ++j) {
            long long id = ids[(size_t)b * L + j];
            if (id < 0 || id >= V) continue;
            const float4 v = tfy_ld_peer_f32x4(table + (size_t)id * D + d);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
        st_local4<OT>(out + (size_t)b * D + d, acc);
    }
}

// any D (the wide tower's per-bucket weights are [V, 1] tables): one element per thread
template <typename OT>
__global__ void __launch_bounds__(256)
tfy_ps_embedding_bag_scalar_kernel(const float* __restrict__ table, const long long* __restrict__ ids,
                                   OT* __restrict__ out, int B, int L, int D, long long V, int mean) {
    const size_t total = (size_t)B * D;
    const float scale = mean ? 1.f / (float)L : 1.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = i / D, d = i % D;
        float acc = 0.f;
        for (int j = 0; j < L; ++j) {
            const long long id = ids[(size_t)b * L + j];
            if (id < 0 || id >= V) continue;
            float v;
            asm volatile("ld.global.relaxed.sys.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(table + (size_t)id * D + d)
                         : "memory");
            acc += v;
        }
        out[(size_t)b * D + d] = (OT)(acc * scale);
    }
}

// ------------------------------------------------------------------------------------ sparse push
// Both sparse pushes are one gradient scatter.  tfy_ps_push_rows is one table with L ids per example;
// tfy_ps_multi_push_rows is T tables with one id per example each.  Occurrence o in [0, T*B*L) is id ids[o] of table
// t = o / (B*L); its gradient is row b = (o % (B*L)) / L of dout, columns [t*col_stride, t*col_stride + D).
struct TfyPsRows {
    const uint64_t* tables;  // device arrays of T peer pointers (tfy_ps_multi_push_rows) ...
    const uint64_t* s1s;
    const uint64_t* s2s;
    float* w0;               // ... or, when they are nullptr, the single table of tfy_ps_push_rows
    float* s10;
    float* s20;
    const long long* ids;
    const void* dout;
    int B, L, T, D;
    long long V;
    int dout_ld, col_stride;
    float scale;             // grad_scale (x 1/L for a mean bag), applied to the folded sum
};

// Column -> table map of a shared push (tfy_ps_multi_push_rows_shared): the rows of column t live in table
// table_of[t] of n_tables distinct tables, and TfyPsRows' arrays hold those n_tables tables.  The key of an
// occurrence becomes table_of[t] * V + id, so two columns of one table fold into one run per row; its gradient still
// comes from its own column.  Preconditions (the caller's map guarantees them): 0 <= table_of[t] < n_tables, every
// table has at least one column and none has more than max_members.  The unmapped instantiations (M = false) take
// the map as a trailing argument and ignore it.
struct TfyPsMap {
    const int* table_of;
    int T, n_tables;
    int max_members;         // the most columns any one table has (1 unmapped): chooses the block sort on the host
};

namespace {
__device__ __forceinline__ float* rows_base(const uint64_t* arr, float* one, int t) {
    return arr ? reinterpret_cast<float*>(arr[t]) : one;
}
template <typename GT, int VEC>
__device__ __forceinline__ float4 ld_grad(const GT* p) {
    if constexpr (VEC == 4) return ld_local4<GT>(p);
    else return make_float4((float)p[0], 0.f, 0.f, 0.f);
}
}  // namespace

// Weighted pushes (W = true) take two more arrays, nullptr meaning "all ones": wts [T, B, L], the weight of every
// occurrence, and fs [T, B], the bag's per-example factor 1/den.  A zero-weight occurrence is absent: it gets the
// sentinel key like an out-of-range id, so it touches no row.  The unweighted instantiations ignore both.
// keys[o] = t * V + id, or T * V (sorts last, never applied) for an absent occurrence; occ[o] = o.  Mapped (M):
// table_of[t] * V + id, sentinel n_tables * V.
template <bool W, bool M>
__global__ void __launch_bounds__(256)
tfy_ps_row_keys_kernel(const long long* __restrict__ ids, int n, int per_table, long long V,
                       unsigned long long* __restrict__ keys, int* __restrict__ occ, const float* __restrict__ wts,
                       TfyPsMap m) {
    const unsigned long long sentinel = (unsigned long long)(M ? m.n_tables : n / per_table) * (unsigned long long)V;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n; o += gridDim.x * blockDim.x) {
        const long long id = ids[o];
        keys[o] = (id < 0 || id >= V || (W && wts && wts[o] == 0.f))
                      ? sentinel
                      : (unsigned long long)(M ? m.table_of[o / per_table] : o / per_table) * (unsigned long long)V + id;
        occ[o] = o;
    }
}

// The same keys for a push whose per-table segments (B*L occurrences each) fit one block: block t stably sorts
// segment t in shared memory.  The segments are in table order, so the concatenation is sorted by (table, id) too,
// except that a segment's out-of-range ids (the sentinel) sit at its end instead of the array's: the apply kernels
// skip sentinels wherever they are.  One launch instead of a key kernel plus a multi-pass device sort.
// Mapped (M): block t is table t.  It sorts the concatenation of its columns' segments (in column order, so equal ids
// stay in (column, b, j) order) and writes it after the segments of the columns of tables < t.
constexpr int kPsSortThreads = 256, kPsSortItems = 8, kPsBlockSortMax = kPsSortThreads * kPsSortItems;

template <bool W, bool M>
__global__ void __launch_bounds__(kPsSortThreads)
tfy_ps_segment_sort_kernel(const long long* __restrict__ ids, int per_table, long long V, int local_bits,
                           unsigned long long* __restrict__ keys, int* __restrict__ occ, const float* __restrict__ wts,
                           TfyPsMap m) {
    using Sort = cub::BlockRadixSort<unsigned int, kPsSortThreads, kPsSortItems, int>;
    __shared__ typename Sort::TempStorage tmp;
    const int t = blockIdx.x;
    size_t base = (size_t)t * per_table;
    int n_items = per_table;
    const int* cols = nullptr;
    if constexpr (M) {
        __shared__ int s_cols[kPsBlockSortMax];                      // the columns of table t, in column order
        __shared__ int s_n, s_before;
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            int n = 0, before = 0;
            for (int c0 = 0; c0 < m.T; c0 += 32) {
                const int c = c0 + lane;
                const int tc = c < m.T ? m.table_of[c] : -1;
                const unsigned mine = __ballot_sync(0xffffffffu, tc == t);
                const int k = n + __popc(mine & ((1u << lane) - 1u));
                if (tc == t && k < kPsBlockSortMax) s_cols[k] = c;
                n += __popc(mine);
                before += __popc(__ballot_sync(0xffffffffu, tc >= 0 && tc < t));
            }
            if (lane == 0) { s_n = n; s_before = before; }
        }
        __syncthreads();
        cols = s_cols;
        n_items = s_n * per_table;
        base = (size_t)s_before * per_table;
        // more columns than max_members promised: leave the table out rather than let the apply kernels read the
        // scratch's stale keys at the positions the block cannot hold
        if (n_items > kPsBlockSortMax) {
            const unsigned long long sentinel = (unsigned long long)gridDim.x * (unsigned long long)V;
            for (int r = threadIdx.x; r < n_items; r += kPsSortThreads) {
                keys[base + r] = sentinel;
                occ[base + r] = (int)base + r;
            }
            return;
        }
    }
    const unsigned long long sentinel = (unsigned long long)gridDim.x * (unsigned long long)V;
    unsigned int k[kPsSortItems];
    int v[kPsSortItems];
#pragma unroll
    for (int j = 0; j < kPsSortItems; ++j) {
        const int r = threadIdx.x * kPsSortItems + j;               // blocked arrangement: r keeps the original order
        // occurrence of item r: base + r, or (mapped) position r % per_table of the (r / per_table)-th column
        const int o = M ? cols[r < n_items ? r / per_table : 0] * per_table + r % per_table : 0;
        if (r < n_items) {
            const long long id = M ? ids[o] : ids[base + r];
            k[j] = (id < 0 || id >= V || (W && wts && (M ? wts[o] : wts[base + r]) == 0.f)) ? (unsigned int)V
                                                                                          : (unsigned int)id;
        } else {
            k[j] = 0xffffffffu;                                      // padding: after every real key
        }
        v[j] = M ? o : (int)base + r;
    }
    Sort(tmp).Sort(k, v, 0, local_bits);
#pragma unroll
    for (int j = 0; j < kPsSortItems; ++j) {
        const int r = threadIdx.x * kPsSortItems + j;
        if (r < n_items) {
            keys[base + r] = k[j] == (unsigned int)V ? sentinel : (unsigned long long)t * (unsigned long long)V + k[j];
            occ[base + r] = v[j];
        }
    }
}

// keys / occ: the occurrences stably sorted by key, so each run of equal keys is one (table, row) with its
// occurrences in their original order.  Two kernels apply the runs; each sums a run in a fixed order and runs the
// optimizer once per element, so the result does not depend on scheduling:
//   short runs (<= kPsShortRun occurrences, nearly every row of a hashed batch): one thread per (run, column group),
//     all in parallel, summing the run sequentially;
//   long runs (hot rows, up to the whole batch): a warp per run, its lanes (CL across the row's column groups x OL
//     along the run) summing strided partial sums that a butterfly reduction combines.
constexpr int kPsShortRun = 32;

namespace {
// peer row of `key` (= t * V + id) in table t, with its slots (nullptr when the optimizer has none)
struct RowRef {
    float* w;
    float* s1;
    float* s2;
    int t;
};
__device__ __forceinline__ RowRef row_of(const TfyPsRows& r, unsigned long long key) {
    RowRef x;
    x.t = (int)(key / (unsigned long long)r.V);
    const size_t row = (size_t)(key % (unsigned long long)r.V) * r.D;
    x.w = rows_base(r.tables, r.w0, x.t) + row;
    x.s1 = rows_base(r.s1s, r.s10, x.t);
    x.s2 = rows_base(r.s2s, r.s20, x.t);
    if (x.s1) x.s1 += row;
    if (x.s2) x.s2 += row;
    return x;
}
// gradient of occurrence o as the fold adds it: g, or cs[o] * g for a weighted push (cs = w_o * f[t, b], written by
// tfy_ps_occ_factors_kernel: one array read through a kernel parameter keeps the scalar apply paths spill-free)
template <bool W>
__device__ __forceinline__ void acc_occ(float4& acc, float4 gv, const float* cs, int o) {
    if constexpr (W) {
        const float c = cs[o];
        acc.x += c * gv.x; acc.y += c * gv.y; acc.z += c * gv.z; acc.w += c * gv.w;
    } else {
        acc.x += gv.x; acc.y += gv.y; acc.z += gv.z; acc.w += gv.w;
    }
}
template <int VEC>
__device__ __forceinline__ void apply_sum(const TfyPsHyper& h, const RowRef& x, size_t d, float4 acc, float scale,
                                          float lr, float vs) {
    if constexpr (VEC == 4) {
        float4 unused;
        ps_apply4(h.opt, x.w + d, x.s1 ? x.s1 + d : nullptr, x.s2 ? x.s2 + d : nullptr, f4_mul(acc, scale), lr, h.eps,
                  h.p1, h.p2, h.p3, vs, false, unused);
    } else {
        ps_apply1(h.opt, x.w + d, x.s1 ? x.s1 + d : nullptr, x.s2 ? x.s2 + d : nullptr, acc.x * scale, lr, h.eps, h.p1,
                  h.p2, h.p3, vs);
    }
}
}  // namespace

// Mapped (M): a key's table is table_of[t] of its occurrences' columns t, and each occurrence's gradient is read from
// its own column t.  occ and cs are then in sorted order, occ[q] being the element offset of the gradient row of the
// q-th sorted occurrence in dout (tfy_ps_occ_offsets_kernel): no division by B*L in the apply loops.
template <typename GT, int VEC, bool W, bool M>
__global__ void __launch_bounds__(256)
tfy_ps_apply_short_rows_kernel(TfyPsRows r, TfyPsHyper h, const float* __restrict__ adam_scale,
                               const unsigned long long* __restrict__ keys, const int* __restrict__ occ, int n,
                               const float* __restrict__ cs, TfyPsMap m) {
    const int DV = r.D / VEC, BL = r.B * r.L;
    const unsigned long long sentinel = (unsigned long long)(M ? m.n_tables : r.T) * (unsigned long long)r.V;
    float vs;
    const float lr = ps_adam_lr(h.opt, h.lr, adam_scale, vs);
    const GT* dout = reinterpret_cast<const GT*>(r.dout);
    const size_t total = (size_t)n * DV;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int p = (int)(i / DV), c = (int)(i % DV);
        const unsigned long long key = keys[p];
        if (key == sentinel || (p > 0 && keys[p - 1] == key)) continue;          // not the start of a run
        int e = p + 1;
        while (e < n && e - p <= kPsShortRun && keys[e] == key) ++e;
        if (e - p > kPsShortRun) continue;                                        // a long run: the warp kernel's
        const RowRef x = row_of(r, key);
        const GT* g = dout + (size_t)x.t * r.col_stride + c * VEC;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = p; q < e; ++q) {
            const int o = occ[q], b = (o % BL) / r.L;
            const GT* go = M ? dout + o + c * VEC : g + (size_t)b * r.dout_ld;
            acc_occ<W>(acc, ld_grad<GT, VEC>(go), cs, M ? q : o);
        }
        apply_sum<VEC>(h, x, (size_t)c * VEC, acc, r.scale, lr, vs);
    }
}

// The mapped instantiations carry a minimum-blocks hint of 1 (no constraint at 256 threads).  Without it ptxas held
// the scalar (VEC = 1) ones to 40 registers and spilled 16 bytes around the optimizer's division calls; with it they
// take 48 and do not spill.  The unmapped instantiations keep the plain bound and their code.
template <typename GT, int VEC, bool W, bool M>
__global__ void __launch_bounds__(256, M ? 1 : 0)
tfy_ps_apply_long_rows_kernel(TfyPsRows r, TfyPsHyper h, const float* __restrict__ adam_scale,
                              const unsigned long long* __restrict__ keys, const int* __restrict__ occ, int n,
                              int cl_log2, const float* __restrict__ cs, TfyPsMap m) {
    const int lane = threadIdx.x & 31;
    const int CL = 1 << cl_log2, OL = 32 >> cl_log2;
    const int cl = lane & (CL - 1), ol = lane >> cl_log2;
    const int DV = r.D / VEC, BL = r.B * r.L;
    const unsigned long long sentinel = (unsigned long long)(M ? m.n_tables : r.T) * (unsigned long long)r.V;
    float vs;
    const float lr = ps_adam_lr(h.opt, h.lr, adam_scale, vs);
    const GT* dout = reinterpret_cast<const GT*>(r.dout);
    const long long nwarp = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long base = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32; base < n;
         base += nwarp * 32) {
        const int p = (int)base + lane;
        const unsigned long long k = p < n ? keys[p] : sentinel;
        // the starts of runs longer than kPsShortRun (keys are sorted: the run reaches p + kPsShortRun)
        unsigned starts = __ballot_sync(0xffffffffu, k != sentinel && (p == 0 || keys[p - 1] != k) &&
                                                         p + kPsShortRun < n && keys[p + kPsShortRun] == k);
        while (starts) {
            const int src = __ffs(starts) - 1;
            starts &= starts - 1;
            const int p0 = (int)base + src;
            const unsigned long long key = __shfl_sync(0xffffffffu, k, src);
            int e = p0 + kPsShortRun + 1;      // the run ends at the first different key
            for (;;) {
                const int q = e + lane;
                const unsigned same = __ballot_sync(0xffffffffu, q < n && keys[q] == key);
                if (same != 0xffffffffu) {
                    e += __ffs(~same) - 1;
                    break;
                }
                e += 32;
            }
            const RowRef x = row_of(r, key);
            const GT* g = dout + (size_t)x.t * r.col_stride;
            for (int c0 = 0; c0 < DV; c0 += CL) {
                const int c = c0 + cl;
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                if (c < DV)
                    for (int q = p0 + ol; q < e; q += OL) {
                        const int o = occ[q], b = (o % BL) / r.L;
                        const GT* go = M ? dout + o : g + (size_t)b * r.dout_ld;
                        acc_occ<W>(acc, ld_grad<GT, VEC>(go + c * VEC), cs, M ? q : o);
                    }
                for (int off = 16; off >= CL; off >>= 1) {
                    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
                    if constexpr (VEC == 4) {
                        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
                        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
                        acc.w += __shfl_xor_sync(0xffffffffu, acc.w, off);
                    }
                }
                if (ol == 0 && c < DV) apply_sum<VEC>(h, x, (size_t)c * VEC, acc, r.scale, lr, vs);
            }
        }
    }
}

// cs[o] = w_o * f[t, b] of every occurrence o (nullptr arrays count as ones), in the original order
__global__ void __launch_bounds__(256)
tfy_ps_occ_factors_kernel(const float* __restrict__ wts, const float* __restrict__ fs, int n, int B, int L,
                          float* __restrict__ cs) {
    const int BL = B * L;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n; o += gridDim.x * blockDim.x)
        cs[o] = (wts ? wts[o] : 1.f) * (fs ? fs[(o / BL) * B + (o % BL) / L] : 1.f);
}

// Mapped pushes, in sorted order: for the q-th sorted occurrence o = occ[q] = (t, b, j), goff[q] = t * col_stride +
// b * dout_ld and (weighted) cs[q] = w_o * f[t, b]
template <bool W>
__global__ void __launch_bounds__(256)
tfy_ps_occ_offsets_kernel(const int* __restrict__ occ, const float* __restrict__ wts, const float* __restrict__ fs,
                          int n, int B, int L, int dout_ld, int col_stride, int* __restrict__ goff,
                          float* __restrict__ cs) {
    const int BL = B * L;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
        const int o = occ[q], t = o / BL, b = (o % BL) / L;
        goff[q] = t * col_stride + b * dout_ld;
        if (W) cs[q] = (wts ? wts[o] : 1.f) * (fs ? fs[t * B + b] : 1.f);
    }
}

namespace {

constexpr long long kPsRowsMaxOcc = 1LL << 30;

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// bytes of CUB's radix-sort temporary storage for n (key, occurrence) pairs over bits [0, end_bit)
size_t rows_sort_temp_bytes(int n, int end_bit) {
    size_t bytes = 0;
    cub::DoubleBuffer<unsigned long long> kb(nullptr, nullptr);
    cub::DoubleBuffer<int> vb(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, kb, vb, n, 0, end_bit) != cudaSuccess) return 0;
    return bytes;
}

size_t rows_scratch_fixed(int n) { return 2 * align256((size_t)n * 8) + 2 * align256((size_t)n * 4); }

// Fold + apply of one sparse push: key build, stable radix sort, apply of the short and of the long runs.
// W: the weighted kernels, with occurrence weights wts and per-example factors fs (either may be nullptr).
// M: the mapped kernels of a shared push, with the column -> table map m (m.T == r.T).
template <bool W, bool M>
int ps_push_rows_fold(const TfyPsRows& r, const TfyPsHyper& h, const float* adam_scale, int grad_is_bf16,
                      void* scratch, size_t scratch_bytes, cudaStream_t s, const float* wts, const float* fs,
                      const TfyPsMap& m) {
    const long long n_ll = (long long)r.T * r.B * r.L;
    if (n_ll == 0) return 0;
    if (n_ll < 0 || n_ll > kPsRowsMaxOcc || r.D < 1 || r.V < 1) return -2;
    const int n = (int)n_ll;
    const unsigned long long sentinel = (unsigned long long)m.n_tables * (unsigned long long)r.V;
    const int end_bit = 64 - __builtin_clzll(sentinel);            // enough bits for every key, the sentinel included
    const size_t temp_bytes = rows_sort_temp_bytes(n, end_bit);
    if (!scratch || temp_bytes == 0 || rows_scratch_fixed(n) + temp_bytes > scratch_bytes) return -5;
    char* p = static_cast<char*>(scratch);
    unsigned long long* k0 = reinterpret_cast<unsigned long long*>(p);
    unsigned long long* k1 = reinterpret_cast<unsigned long long*>(p + align256((size_t)n * 8));
    int* v0 = reinterpret_cast<int*>(p + 2 * align256((size_t)n * 8));
    int* v1 = reinterpret_cast<int*>(p + 2 * align256((size_t)n * 8) + align256((size_t)n * 4));
    void* temp = p + rows_scratch_fixed(n);

    cub::DoubleBuffer<unsigned long long> kb(k0, k1);
    cub::DoubleBuffer<int> vb(v0, v1);
    const int per_table = r.B * r.L;
    // the block sort holds one table's occurrences: max_members columns of B*L each at most
    if ((long long)m.max_members * per_table <= kPsBlockSortMax && r.V < 0x7fffffffLL) {
        const int local_bits = 64 - __builtin_clzll((unsigned long long)r.V);     // ids and the local sentinel V
        tfy_ps_segment_sort_kernel<W, M><<<m.n_tables, kPsSortThreads, 0, s>>>(r.ids, per_table, r.V, local_bits, k0,
                                                                               v0, W ? wts : nullptr, m);
    } else {
        size_t gk = ((size_t)n + 255) / 256;
        if (gk > TFY_NUM_SMS * 8) gk = TFY_NUM_SMS * 8;
        tfy_ps_row_keys_kernel<W, M><<<(unsigned)gk, 256, 0, s>>>(r.ids, n, per_table, r.V, k0, v0,
                                                                  W ? wts : nullptr, m);
        size_t tb = temp_bytes;
        cudaError_t err = cub::DeviceRadixSort::SortPairs(temp, tb, kb, vb, n, 0, end_bit, s);
        if (err != cudaSuccess) return (int)err;
    }

    // weighted: the per-occurrence factors go to the sort's alternate key buffer, free once the keys are sorted;
    // mapped: the sorted gradient offsets to its alternate value buffer, which the apply kernels then take as occ
    float* cs = nullptr;
    const int* occ = vb.Current();
    if (M) {
        if (W) cs = reinterpret_cast<float*>(kb.Current() == k0 ? k1 : k0);
        int* goff = vb.Current() == v0 ? v1 : v0;
        size_t gf = ((size_t)n + 255) / 256;
        if (gf > TFY_NUM_SMS * 8) gf = TFY_NUM_SMS * 8;
        tfy_ps_occ_offsets_kernel<W><<<(unsigned)gf, 256, 0, s>>>(occ, wts, fs, n, r.B, r.L, r.dout_ld, r.col_stride,
                                                                   goff, cs);
        occ = goff;
    } else if (W) {
        cs = reinterpret_cast<float*>(kb.Current() == k0 ? k1 : k0);
        size_t gf = ((size_t)n + 255) / 256;
        if (gf > TFY_NUM_SMS * 8) gf = TFY_NUM_SMS * 8;
        tfy_ps_occ_factors_kernel<<<(unsigned)gf, 256, 0, s>>>(wts, fs, n, r.B, r.L, cs);
    }
    // 16-byte gradient loads only when every row of every table slice starts on a 4-element boundary
    const size_t gsize = grad_is_bf16 ? 2 : 4;
    const bool vec = (r.D % 4 == 0) && (r.dout_ld % 4 == 0) && (r.col_stride % 4 == 0) &&
                     (reinterpret_cast<uintptr_t>(r.dout) % (4 * gsize) == 0);
    const int dv = vec ? r.D / 4 : r.D;
    int cl_log2 = 0;
    while (cl_log2 < 5 && (2 << cl_log2) <= dv) ++cl_log2;          // column lanes: largest power of 2 <= min(dv, 32)
    size_t gs = ((size_t)n * dv + 255) / 256;                           // one thread per (position, column group)
    if (gs > TFY_NUM_SMS * 8) gs = TFY_NUM_SMS * 8;
    size_t gl = ((size_t)n + 255) / 256;                                // one warp per 32 sorted positions
    if (gl > TFY_NUM_SMS * 8) gl = TFY_NUM_SMS * 8;
#define TFY_APPLY_ROWS(GT, VV)                                                                                         \
    do {                                                                                                               \
        tfy_ps_apply_short_rows_kernel<GT, VV, W, M><<<(unsigned)gs, 256, 0, s>>>(r, h, adam_scale, kb.Current(), occ, \
                                                                                   n, cs, m);                          \
        tfy_ps_apply_long_rows_kernel<GT, VV, W, M><<<(unsigned)gl, 256, 0, s>>>(r, h, adam_scale, kb.Current(), occ,  \
                                                                                  n, cl_log2, cs, m);                  \
    } while (0)
    if (grad_is_bf16) { if (vec) TFY_APPLY_ROWS(__nv_bfloat16, 4); else TFY_APPLY_ROWS(__nv_bfloat16, 1); }
    else { if (vec) TFY_APPLY_ROWS(float, 4); else TFY_APPLY_ROWS(float, 1); }
#undef TFY_APPLY_ROWS
    return (int)cudaGetLastError();
}

// The fold of one push, unmapped (every column its own table) unless map is given.
int ps_push_rows_launch(const TfyPsRows& r, const TfyPsHyper& h, const float* adam_scale, int grad_is_bf16,
                        void* scratch, size_t scratch_bytes, cudaStream_t s, bool weighted = false,
                        const float* wts = nullptr, const float* fs = nullptr, const TfyPsMap* map = nullptr) {
    const TfyPsMap m = map ? *map : TfyPsMap{nullptr, r.T, r.T, 1};
#define TFY_FOLD(WW, MM) ps_push_rows_fold<WW, MM>(r, h, adam_scale, grad_is_bf16, scratch, scratch_bytes, s, wts, fs, m)
    if (map) return weighted ? TFY_FOLD(true, true) : TFY_FOLD(false, true);
    return weighted ? TFY_FOLD(true, false) : TFY_FOLD(false, false);
#undef TFY_FOLD
}

}  // namespace
// ------------------------------------------------------------------------------- multi-table sparse ops
// A wide-and-deep step touches one row in each of T tables per example (26 hashed categorical columns, twice: the
// wide tower's [V, 1] tables and the deep tower's [V, 64] tables).  One launch per table made the step launch-bound
// (52 gathers + 52 pushes + 26 adds of ~3 us each, profiles/r2/ps_step_profile_r2q.txt); these kernels take the
// whole group: tables = device array of T peer pointers, ids = int64 [T, B].
//   multi_bag      : out[b, d] = sum_t table_t[ids[t, b], d]                      (the wide tower's logit)
//   multi_push_rows: row ids[t, b] of table t receives dout[b, t * col_stride + d] (col_stride 0: every table gets
//                    the same gradient -- wide tower; col_stride D: column slices of a wider matrix -- the fused
//                    first deep layer's dx), optimizer fused as in tfy_ps_push_rows.
template <typename OT>
__global__ void __launch_bounds__(256)
tfy_ps_multi_bag_kernel(const uint64_t* __restrict__ tables, const long long* __restrict__ ids, OT* __restrict__ out,
                        int B, int T, int D, long long V) {
    const size_t total = (size_t)B * D;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = i / D, d = i % D;
        float acc = 0.f;
        for (int t = 0; t < T; ++t) {
            const long long id = ids[(size_t)t * B + b];
            if (id < 0 || id >= V) continue;
            float v;
            asm volatile("ld.global.relaxed.sys.L1::no_allocate.f32 %0, [%1];"
                         : "=f"(v)
                         : "l"(reinterpret_cast<const float*>(tables[t]) + (size_t)id * D + d)
                         : "memory");
            acc += v;
        }
        out[i] = (OT)acc;
    }
}

// Weighted multi-hot bag (TF's embedding_column combiners, see the header): T tables x L ids per example.
//   out[b, t * col_stride + d] (col_stride > 0)  or  out[b, d] = sum_t (col_stride 0), of S_t[b, d] / den_t[b],
//   S = sum_present w table[i], den = 1 (sum), sum_present w (mean), sqrt(sum_present w^2) (sqrtn), 0 where den == 0.
// One thread per (b, column slice, VEC columns); each recomputes den from its L weights (L is small), so no second
// pass.  Sums run over t, then j.  fs[t, b] = 1/den (0 where den == 0) for the push; numeric [B, n_num] is copied
// to columns [T*D, T*D + n_num) as K5 does.  Other columns of out are not written (the caller's pad zeros stay).
namespace {
template <int VEC>
__device__ __forceinline__ float4 ld_row(const float* p) {
    if constexpr (VEC == 4) {
        return tfy_ld_peer_f32x4(p);
    } else {
        float v;
        asm volatile("ld.global.relaxed.sys.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
        return make_float4(v, 0.f, 0.f, 0.f);
    }
}
template <typename OT, int VEC>
__device__ __forceinline__ void st_out(OT* p, float4 v) {
    if constexpr (VEC == 4) st_local4<OT>(p, v);
    else *p = (OT)v.x;
}
}  // namespace

template <typename OT, int VEC>
__global__ void __launch_bounds__(256)
tfy_ps_multi_bag_weighted_kernel(const uint64_t* __restrict__ tables, const long long* __restrict__ ids,
                                 const float* __restrict__ wts, int combiner, int B, int L, int T, int D, long long V,
                                 OT* __restrict__ out, int out_ld, int col_stride, const float* __restrict__ numeric,
                                 int n_num, float* __restrict__ fs) {
    const int DV = D / VEC, TT = col_stride ? T : 1;
    const size_t total = (size_t)B * TT * DV;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int b = (int)(i / ((size_t)TT * DV)), r = (int)(i % ((size_t)TT * DV));
        const int tq = r / DV, c = r % DV;
        const int t0 = col_stride ? tq : 0, t1 = col_stride ? tq + 1 : T;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int t = t0; t < t1; ++t) {
            const size_t o0 = ((size_t)t * B + b) * L;
            const float* table = reinterpret_cast<const float*>(tables[t]) + (size_t)c * VEC;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            float den = 0.f;
            for (int j = 0; j < L; ++j) {
                const long long id = ids[o0 + j];
                const float w = wts ? wts[o0 + j] : 1.f;
                if (id < 0 || id >= V || w == 0.f) continue;
                const float4 v = ld_row<VEC>(table + (size_t)id * D);
                s.x += w * v.x; s.y += w * v.y; s.z += w * v.z; s.w += w * v.w;
                den += combiner == 2 ? w * w : w;
            }
            if (combiner == 0) den = 1.f;
            else if (combiner == 2) den = sqrtf(den);
            if (den != 0.f) {
                acc.x += s.x / den; acc.y += s.y / den; acc.z += s.z / den; acc.w += s.w / den;
            }
            if (fs && c == 0) fs[(size_t)t * B + b] = den != 0.f ? 1.f / den : 0.f;
        }
        st_out<OT, VEC>(out + (size_t)b * out_ld + (size_t)tq * col_stride + (size_t)c * VEC, acc);
    }
    const size_t nn = (size_t)B * n_num;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nn; i += stride)
        out[(i / n_num) * out_ld + (size_t)T * D + i % n_num] = (OT)numeric[i];
}

// fp32 -> bf16 shadow refresh of a whole segment (run by the chief after initialisation / restore)
__global__ void __launch_bounds__(256) tfy_ps_refresh_shadow_kernel(const TfyPsSeg* __restrict__ segs) {
    const TfyPsSeg sg = segs[blockIdx.y];
    if (!sg.remote_shadow) return;
    const float* w = reinterpret_cast<const float*>(sg.remote_w);
    __nv_bfloat16* sh = reinterpret_cast<__nv_bfloat16*>(sg.remote_shadow);
    const size_t n4 = sg.n / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
        st_shadow4(sh, i * 4, tfy_ld_peer_f32x4(w + i * 4), sg.cols, sg.shadow_ld);
    if (blockIdx.x == 0)
        for (size_t i = n4 * 4 + threadIdx.x; i < sg.n; i += blockDim.x)
            sh[shadow_index(i, sg.cols, sg.shadow_ld)] = __float2bfloat16(w[i]);
}

extern "C" {

int tfy_ps_pull(const TfyPsSeg* segs, int nseg, size_t max_n, int local_is_bf16, cudaStream_t s) {
    if (nseg <= 0) return 0;
    size_t gx = (max_n / 4 + 255) / 256;
    if (gx < 1) gx = 1;
    if (gx > TFY_NUM_SMS * 4) gx = TFY_NUM_SMS * 4;
    dim3 grid((unsigned)gx, nseg);
    if (local_is_bf16) tfy_ps_pull_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(segs);
    else tfy_ps_pull_kernel<float><<<grid, 256, 0, s>>>(segs);
    return (int)cudaGetLastError();
}

// adam_scale: device pointer to {1/(1-b1^t), 1/sqrt(1-b2^t)} (may be nullptr when no segment uses Adam)
int tfy_ps_push(const TfyPsSeg* segs, int nseg, size_t max_n, int grad_is_bf16, float grad_scale,
                const float* adam_scale, cudaStream_t s) {
    if (nseg <= 0) return 0;
    size_t gx = (max_n / 4 + 255) / 256;
    if (gx < 1) gx = 1;
    if (gx > TFY_NUM_SMS * 4) gx = TFY_NUM_SMS * 4;
    dim3 grid((unsigned)gx, nseg);
    if (grad_is_bf16) tfy_ps_push_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(segs, grad_scale, adam_scale);
    else tfy_ps_push_kernel<float><<<grid, 256, 0, s>>>(segs, grad_scale, adam_scale);
    return (int)cudaGetLastError();
}

int tfy_ps_refresh_shadow(const TfyPsSeg* segs, int nseg, size_t max_n, cudaStream_t s) {
    if (nseg <= 0) return 0;
    size_t gx = (max_n / 4 + 255) / 256;
    if (gx < 1) gx = 1;
    if (gx > TFY_NUM_SMS * 4) gx = TFY_NUM_SMS * 4;
    dim3 grid((unsigned)gx, nseg);
    tfy_ps_refresh_shadow_kernel<<<grid, 256, 0, s>>>(segs);
    return (int)cudaGetLastError();
}

int tfy_ps_embedding_bag(const void* table, const void* ids, void* out, int out_is_bf16, int B, int L, int D,
                         long long V, int mean, cudaStream_t s) {
    if (D % 4) {
        size_t g1 = ((size_t)B * D + 255) / 256;
        if (g1 < 1) g1 = 1;
        if (g1 > TFY_NUM_SMS * 8) g1 = TFY_NUM_SMS * 8;
        if (out_is_bf16)
            tfy_ps_embedding_bag_scalar_kernel<__nv_bfloat16><<<(unsigned)g1, 256, 0, s>>>(
                (const float*)table, (const long long*)ids, (__nv_bfloat16*)out, B, L, D, V, mean);
        else
            tfy_ps_embedding_bag_scalar_kernel<float><<<(unsigned)g1, 256, 0, s>>>(
                (const float*)table, (const long long*)ids, (float*)out, B, L, D, V, mean);
        return (int)cudaGetLastError();
    }
    size_t gx = ((size_t)B * (D / 4) + 255) / 256;
    if (gx < 1) gx = 1;
    if (gx > TFY_NUM_SMS * 8) gx = TFY_NUM_SMS * 8;
    if (out_is_bf16)
        tfy_ps_embedding_bag_kernel<__nv_bfloat16><<<(unsigned)gx, 256, 0, s>>>(
            (const float*)table, (const long long*)ids, (__nv_bfloat16*)out, B, L, D, V, mean);
    else
        tfy_ps_embedding_bag_kernel<float><<<(unsigned)gx, 256, 0, s>>>((const float*)table, (const long long*)ids,
                                                                        (float*)out, B, L, D, V, mean);
    return (int)cudaGetLastError();
}

// Scratch (device bytes) that a sparse push of n = B*L (tfy_ps_push_rows) or T*B (tfy_ps_multi_push_rows) ids needs:
// the keys and occurrence indices of the fold, double-buffered, and the radix sort's temporary storage.
size_t tfy_ps_push_rows_scratch_bytes(long long n) {
    if (n <= 0 || n > kPsRowsMaxOcc) return 0;
    return rows_scratch_fixed((int)n) + rows_sort_temp_bytes((int)n, 64);
}

int tfy_ps_push_rows(void* table, void* s1_table, void* s2_table, const void* ids, const void* dout, int grad_is_bf16,
                     int B, int L, int D, long long V, int mean, int opt, float lr, float eps, float p1, float p2, float p3,
                     float grad_scale, const float* adam_scale, int dout_ld, void* scratch, size_t scratch_bytes,
                     cudaStream_t s) {
    // dout_ld: row pitch (elements) of dout; 0 = D (contiguous [B, D]).  A larger pitch lets the caller push a
    // column slice of a wider gradient matrix (the fused first layer's dx) without copying it out.
    if (dout_ld <= 0) dout_ld = D;
    if (opt != TFY_OPT_SGD && opt != TFY_OPT_ADAGRAD && opt != TFY_OPT_ADAM && opt != TFY_OPT_FTRL) return -3;
    if (opt != TFY_OPT_SGD && !s1_table) return -4;
    if ((opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL) && !s2_table) return -4;
    TfyPsHyper h;
    h.opt = opt; h.lr = lr; h.eps = eps; h.wd = 0.f; h.p1 = p1; h.p2 = p2; h.p3 = p3; h.grad_scale = grad_scale;
    TfyPsRows r = {};
    r.w0 = (float*)table; r.s10 = (float*)s1_table; r.s20 = (float*)s2_table;
    r.ids = (const long long*)ids; r.dout = dout;
    r.B = B; r.L = L; r.T = 1; r.D = D; r.V = V; r.dout_ld = dout_ld; r.col_stride = 0;
    r.scale = (mean ? 1.f / (float)L : 1.f) * grad_scale;
    return ps_push_rows_launch(r, h, adam_scale, grad_is_bf16, scratch, scratch_bytes, s);
}

int tfy_ps_multi_bag(const uint64_t* tables, const void* ids, void* out, int out_is_bf16, int B, int T, int D,
                     long long V, cudaStream_t s) {
    if (B < 1 || T < 1 || D < 1) return -2;
    size_t gx = ((size_t)B * D + 255) / 256;
    if (gx > TFY_NUM_SMS * 8) gx = TFY_NUM_SMS * 8;
    if (out_is_bf16)
        tfy_ps_multi_bag_kernel<__nv_bfloat16><<<(unsigned)gx, 256, 0, s>>>(tables, (const long long*)ids,
                                                                           (__nv_bfloat16*)out, B, T, D, V);
    else
        tfy_ps_multi_bag_kernel<float><<<(unsigned)gx, 256, 0, s>>>(tables, (const long long*)ids, (float*)out, B, T, D, V);
    return (int)cudaGetLastError();
}

// s1s / s2s: device arrays of T slot-table pointers (nullptr when the optimizer has no such slot)
int tfy_ps_multi_push_rows(const uint64_t* tables, const uint64_t* s1s, const uint64_t* s2s, const void* ids,
                           const void* dout, int grad_is_bf16, int B, int T, int D, long long V, int opt, float lr,
                           float eps, float p1, float p2, float p3, float grad_scale, const float* adam_scale,
                           int dout_ld, int col_stride, void* scratch, size_t scratch_bytes, cudaStream_t s) {
    if (opt != TFY_OPT_SGD && opt != TFY_OPT_ADAGRAD && opt != TFY_OPT_ADAM && opt != TFY_OPT_FTRL) return -3;
    if (opt != TFY_OPT_SGD && !s1s) return -4;
    if ((opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL) && !s2s) return -4;
    if (dout_ld <= 0) dout_ld = D;
    TfyPsHyper h;
    h.opt = opt; h.lr = lr; h.eps = eps; h.wd = 0.f; h.p1 = p1; h.p2 = p2; h.p3 = p3; h.grad_scale = grad_scale;
    TfyPsRows r = {};
    r.tables = tables; r.s1s = s1s; r.s2s = s2s;
    r.ids = (const long long*)ids; r.dout = dout;
    r.B = B; r.L = 1; r.T = T; r.D = D; r.V = V; r.dout_ld = dout_ld; r.col_stride = col_stride;
    r.scale = grad_scale;
    return ps_push_rows_launch(r, h, adam_scale, grad_is_bf16, scratch, scratch_bytes, s);
}

// ids int64 [T, B, L]; weights fp32 [T, B, L] or nullptr (all 1); combiner 0 sum, 1 mean, 2 sqrtn.  out (fp32 or
// bf16, row pitch out_ld): table t in columns [t * col_stride, t * col_stride + D), or, col_stride 0, all tables
// summed into [0, D).  numeric fp32 [B, n_num] (n_num <= 64, col_stride == D) goes to columns [T*D, T*D + n_num).
// f fp32 [T, B] receives 1/den (0 where den == 0), or nullptr.
int tfy_ps_multi_bag_weighted(const uint64_t* tables, const void* ids, const float* weights, int combiner, int B,
                              int L, int T, int D, long long V, void* out, int out_is_bf16, int out_ld, int col_stride,
                              const float* numeric, int n_num, float* f, cudaStream_t s) {
    if (B < 1 || L < 1 || T < 1 || D < 1 || V < 1 || combiner < 0 || combiner > 2) return -2;
    if (col_stride != 0 && col_stride < D) return -2;
    if (n_num < 0 || n_num > 64 || (n_num > 0 && (col_stride != D || !numeric))) return -2;
    if (out_ld < (col_stride ? (T - 1) * col_stride + D : D) + n_num) return -2;
    const size_t osize = out_is_bf16 ? 2 : 4;
    const bool vec = (D % 4 == 0) && (out_ld % 4 == 0) && (col_stride % 4 == 0) &&
                     (reinterpret_cast<uintptr_t>(out) % (4 * osize) == 0);
    const size_t total = (size_t)B * (col_stride ? T : 1) * (vec ? D / 4 : D);
    size_t gx = (total > (size_t)B * n_num ? total : (size_t)B * n_num) + 255;
    gx /= 256;
    if (gx > TFY_NUM_SMS * 8) gx = TFY_NUM_SMS * 8;
    const long long* idp = (const long long*)ids;
#define TFY_BAG_W(OT, VV)                                                                                              \
    tfy_ps_multi_bag_weighted_kernel<OT, VV><<<(unsigned)gx, 256, 0, s>>>(tables, idp, weights, combiner, B, L, T, D, \
                                                                          V, (OT*)out, out_ld, col_stride, numeric,   \
                                                                          n_num, f)
    if (out_is_bf16) { if (vec) TFY_BAG_W(__nv_bfloat16, 4); else TFY_BAG_W(__nv_bfloat16, 1); }
    else { if (vec) TFY_BAG_W(float, 4); else TFY_BAG_W(float, 1); }
#undef TFY_BAG_W
    return (int)cudaGetLastError();
}

// The sparse push of a weighted bag: the arguments of tfy_ps_multi_push_rows, plus L ids per example, the
// occurrence weights (or nullptr) and the bag's f = 1/den (or nullptr = 1, only for combiner 0 = sum).  Occurrence
// (t, b, j) adds weights[t, b, j] * f[t, b] * dout[b, t * col_stride + d] to its row's folded gradient.
int tfy_ps_multi_push_rows_weighted(const uint64_t* tables, const uint64_t* s1s, const uint64_t* s2s, const void* ids,
                                    const void* dout, int grad_is_bf16, int B, int T, int D, long long V, int opt,
                                    float lr, float eps, float p1, float p2, float p3, float grad_scale,
                                    const float* adam_scale, int dout_ld, int col_stride, int L, const float* weights,
                                    const float* f, int combiner, void* scratch, size_t scratch_bytes,
                                    cudaStream_t s) {
    if (L < 1 || B < 0 || T < 0 || combiner < 0 || combiner > 2) return -2;
    if (opt != TFY_OPT_SGD && opt != TFY_OPT_ADAGRAD && opt != TFY_OPT_ADAM && opt != TFY_OPT_FTRL) return -3;
    if (opt != TFY_OPT_SGD && !s1s) return -4;
    if ((opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL) && !s2s) return -4;
    if (!f && combiner != 0) return -4;
    if (dout_ld <= 0) dout_ld = D;
    TfyPsHyper h;
    h.opt = opt; h.lr = lr; h.eps = eps; h.wd = 0.f; h.p1 = p1; h.p2 = p2; h.p3 = p3; h.grad_scale = grad_scale;
    TfyPsRows r = {};
    r.tables = tables; r.s1s = s1s; r.s2s = s2s;
    r.ids = (const long long*)ids; r.dout = dout;
    r.B = B; r.L = L; r.T = T; r.D = D; r.V = V; r.dout_ld = dout_ld; r.col_stride = col_stride;
    r.scale = grad_scale;
    return ps_push_rows_launch(r, h, adam_scale, grad_is_bf16, scratch, scratch_bytes, s, true, weights, f);
}

// The sparse push of columns that share tables (shared embedding columns): the arguments of
// tfy_ps_multi_push_rows_weighted, except that tables / s1s / s2s hold n_tables DISTINCT tables and the device
// int32 table_of[T] names the table of every column (0 <= table_of[t] < n_tables, every table named at least once),
// and max_members is the largest number of columns of any one table: the fold takes the block sort when max_members
// * B * L <= 2048.  A table with more columns than max_members is then left out of the push.
// Every distinct (table, row) receives the sum, in (t, b, j) order, of weights[t, b, j] * f[t, b] *
// dout[b, t * col_stride + d] over the occurrences of all its columns, and its optimizer runs once.  weights and f
// both nullptr: the unweighted kernels (a one-hot K5 push, combiner 0).
int tfy_ps_multi_push_rows_shared(const uint64_t* tables, const uint64_t* s1s, const uint64_t* s2s, const void* ids,
                                  const void* dout, int grad_is_bf16, int B, int T, int D, long long V, int opt,
                                  float lr, float eps, float p1, float p2, float p3, float grad_scale,
                                  const float* adam_scale, int dout_ld, int col_stride, int L, const float* weights,
                                  const float* f, int combiner, int n_tables, const int* table_of, int max_members,
                                  void* scratch,
                                  size_t scratch_bytes, cudaStream_t s) {
    if (L < 1 || B < 0 || T < 0 || combiner < 0 || combiner > 2) return -2;
    if (n_tables < 1 || n_tables > T || !table_of) return -2;
    if (max_members < 1 || max_members > T - n_tables + 1) return -2;
    if (opt != TFY_OPT_SGD && opt != TFY_OPT_ADAGRAD && opt != TFY_OPT_ADAM && opt != TFY_OPT_FTRL) return -3;
    if (opt != TFY_OPT_SGD && !s1s) return -4;
    if ((opt == TFY_OPT_ADAM || opt == TFY_OPT_FTRL) && !s2s) return -4;
    if (!f && combiner != 0) return -4;
    if (dout_ld <= 0) dout_ld = D;
    if ((long long)(T - 1) * col_stride + (long long)(B > 0 ? B - 1 : 0) * dout_ld + D > 0x7fffffffLL) return -2;
    TfyPsHyper h;
    h.opt = opt; h.lr = lr; h.eps = eps; h.wd = 0.f; h.p1 = p1; h.p2 = p2; h.p3 = p3; h.grad_scale = grad_scale;
    TfyPsRows r = {};
    r.tables = tables; r.s1s = s1s; r.s2s = s2s;
    r.ids = (const long long*)ids; r.dout = dout;
    r.B = B; r.L = L; r.T = T; r.D = D; r.V = V; r.dout_ld = dout_ld; r.col_stride = col_stride;
    r.scale = grad_scale;
    const TfyPsMap map = {table_of, T, n_tables, max_members};
    return ps_push_rows_launch(r, h, adam_scale, grad_is_bf16, scratch, scratch_bytes, s, weights || f, weights, f,
                               &map);
}

}  // extern "C"
