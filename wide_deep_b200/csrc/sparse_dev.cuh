// Device helpers shared by sparse.cu (replicated tables) and shard.cu (row-sharded tables): cache-hinted loads, binary searches,
// the hot-row chunk layout and the per-row optimizer update (reference python/lib/utils/model_util.py:62-105; SURVEY A.9).
#pragma once
#include "common.cuh"

namespace wd {

__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// Rows touched at most kChunk times are summed by one lane group directly.  Hotter rows (small tables, skewed ids) are split into
// chunks of kChunk occurrences that are summed in parallel and then combined in chunk order (deterministic).
constexpr int kChunk = 16;

__device__ __forceinline__ int chunk_owner(const int32_t* __restrict__ choff, int nu, int c) {
    int lo = 0, hi = nu;                         // last u with choff[u] <= c
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (choff[mid] <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}
__device__ __forceinline__ int lower_bound_u32(const uint32_t* __restrict__ a, int n, uint32_t key) {
    int lo = 0, hi = n;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ int upper_bound_u32(const uint32_t* __restrict__ a, int n, uint32_t key) {
    int lo = 0, hi = n;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (a[mid] <= key) lo = mid + 1; else hi = mid; }
    return lo;
}

struct OptParams { int kind; float lr, l1, l2, init_acc, beta1, beta2, epsilon, rho, momentum; };
inline OptParams make_opt(const WdOptimizer& o) { return OptParams{o.kind, o.lr, o.l1, o.l2, o.init_acc, o.beta1, o.beta2, o.epsilon, o.rho, o.momentum}; }
// initial value of optimizer slot 1 (Adagrad accumulator / FTRL n / Adam m / RMSProp rms); slot 2 always starts at 0
inline float slot1_init(const WdOptimizer& o) {
    if (o.kind == WD_OPT_ADAGRAD || o.kind == WD_OPT_FTRL) return o.init_acc;
    return o.kind == WD_OPT_RMSPROP ? 1.f : 0.f;
}
inline int opt_nslots(const WdOptimizer& o) { return o.kind == WD_OPT_SGD ? 0 : (o.kind == WD_OPT_ADAGRAD ? 1 : 2); }

// One update of a TOUCHED row element from its summed gradient g (duplicates already summed: "sum duplicates, apply once").
// Adam is the exception: TensorFlow's sparse Adam decays m and v over the whole variable and moves every row each step
// (AdamOptimizer._apply_sparse_shared), so here the touched rows only receive the scatter-add of (1 - beta) * g terms; the decay
// before it and the step after it are dense passes over the table (adam_decay_kernel / adam_step_kernel in sparse.cu).
__device__ __forceinline__ void opt_update(const OptParams& o, float g, float& w, float& s1, float& s2) {
    if (o.kind == WD_OPT_ADAGRAD) {                 // tf.train.AdagradOptimizer: acc += g^2; w -= lr*g/sqrt(acc)
        s1 += g * g;
        w -= o.lr * g / sqrtf(s1);
    } else if (o.kind == WD_OPT_FTRL) {             // tf.train.FtrlOptimizer, lr_power = -0.5 (SURVEY A.9)
        float n1 = s1 + g * g;
        float z1 = s2 + g - (sqrtf(n1) - sqrtf(s1)) / o.lr * w;
        float wn = 0.f;
        if (fabsf(z1) > o.l1) wn = (copysignf(o.l1, z1) - z1) / (sqrtf(n1) / o.lr + 2.f * o.l2);
        w = wn; s1 = n1; s2 = z1;
    } else if (o.kind == WD_OPT_RMSPROP) {          // SparseApplyRMSProp: ms += (g^2 - ms)(1 - rho); mom = mom * momentum + lr * g * rsqrt(ms + eps)
        s1 += (g * g - s1) * (1.f - o.rho);
        s2 = s2 * o.momentum + (g * o.lr) / sqrtf(s1 + o.epsilon);
        w -= s2;
    } else if (o.kind == WD_OPT_ADAM) {             // scatter-add stage of sparse Adam
        s1 += g * (1.f - o.beta1);
        s2 += g * g * (1.f - o.beta2);
    } else {
        w -= o.lr * g;
    }
}

// ---- list machinery implemented in sparse.cu, used by shard.cu for the rows a rank owns
// sort (row, occurrence) pairs of e_row[0 .. *d_n) by row, unique rows, segment starts, hot-row chunk layout -> list `which`
int list_group(WdModel* m, int which, const int32_t* d_n, const uint32_t* e_row);
int list_sort_by_key(WdModel* m, int which, const int32_t* d_n, const uint32_t* e_key);
// ugrad[u] = fixed-order sum of the chunk partials of multi-chunk rows (after the two gradient-sum passes)
int list_chunk_combine(WdModel* m, int which, int width);
// optimizer over the unique rows of list `which`: embedding tables given in row order / one wide record array.  d_stage (optional,
// [ntab]): 0 = record in place, else the table is staged and the record of unique row u is at stage + u * d_stage[t]
int list_apply_emb(WdModel* m, int which, int width, int ntab, const int64_t* d_row_base, float* const* d_data, const int32_t* d_dim,
                   const int32_t* d_stride, const WdOptimizer& o, const int32_t* d_stage = nullptr, float* stage = nullptr);
int list_apply_wide(WdModel* m, int which, float4* wide, const WdOptimizer& o);

}  // namespace wd
