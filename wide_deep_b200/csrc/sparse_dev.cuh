// Device code shared by sparse.cu (replicated tables) and shard.cu (row-sharded tables): cache-hinted loads, binary searches, the
// hot-row chunk layout, the per-row optimizer update (reference python/lib/utils/model_util.py:62-105; SURVEY A.9) and where it
// finds a row's record (RowRecords), and the per-row gradient sums over an occurrence source (emb_grad_sum_kernel /
// wide_grad_sum_kernel).
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
// rows of a list's chunk partials (RowList::cpart): a row of len > kChunk entries has ceil(len / kChunk) <= 2 len / kChunk chunks
inline int64_t chunk_cap(int64_t max_nnz) { return 2 * (max_nnz / kChunk) + 64; }

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
// last i with base[i] <= key (base ascending, base[0] <= key): the table of a row from the tables' row bases (tables are few)
__device__ __forceinline__ int table_of(const int64_t* __restrict__ base, int n, int64_t key) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (base[mid] <= key) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Adam also carries its device beta powers bpow = {beta1^t, beta2^t} (step size lr_t: with_lr_t) and `touched`, the bitmap of the
// record set being updated (bit r: row r of the set was updated this step; adam_untouched_* moves the others and clears it).
struct OptParams {
    int kind; float lr, l1, l2, init_acc, beta1, beta2, epsilon, rho, momentum;
    const float* bpow; uint32_t* touched; float lr_t;
};
inline OptParams make_opt(const WdOptimizer& o, const float* bpow = nullptr, uint32_t* touched = nullptr) {
    return OptParams{o.kind, o.lr, o.l1, o.l2, o.init_acc, o.beta1, o.beta2, o.epsilon, o.rho, o.momentum, bpow, touched, 0.f};
}
// Adam: lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t) of this step, read once per thread
__device__ __forceinline__ OptParams with_lr_t(OptParams o) {
    if (o.kind == WD_OPT_ADAM) o.lr_t = o.lr * sqrtf(1.f - o.bpow[1]) / (1.f - o.bpow[0]);
    return o;
}
__device__ __forceinline__ void mark_touched(const OptParams& o, int64_t row) {
    if (o.touched) atomicOr(o.touched + (row >> 5), 1u << (row & 31));
}
// initial value of optimizer slot 1 (Adagrad accumulator / FTRL n / Adam m / RMSProp rms); slot 2 always starts at 0
inline float slot1_init(const WdOptimizer& o) {
    if (o.kind == WD_OPT_ADAGRAD || o.kind == WD_OPT_FTRL) return o.init_acc;
    return o.kind == WD_OPT_RMSPROP ? 1.f : 0.f;
}
// optimizer slots of an embedding record (a deferred table's record has a stamp behind them: the count is not stride / dim - 1)
__host__ __device__ __forceinline__ int kind_nslots(int kind) { return kind == WD_OPT_SGD ? 0 : (kind == WD_OPT_ADAGRAD ? 1 : 2); }
inline int opt_nslots(const WdOptimizer& o) { return kind_nslots(o.kind); }

// Sparse Adam (tf.train.AdamOptimizer on IndexedSlices, AdamOptimizer._apply_sparse_shared) decays m and v over the WHOLE variable,
// scatter-adds the summed gradients of the touched rows, then moves EVERY row by lr_t * m / (sqrt(v) + eps).  A touched row does all
// three in opt_update, a row nobody touched the decay and the step in adam_untouched4: one read and one write of each record.  The
// decay is rounded on its own (__fmul_rn: never contracted into the scatter-add's multiply-add), so either way the row gets exactly
// the values of three separate passes.
__device__ __forceinline__ void adam_decay(const OptParams& o, float& m, float& v) {
    m = __fmul_rn(m, o.beta1);
    v = __fmul_rn(v, o.beta2);
}
__device__ __forceinline__ void adam_step(const OptParams& o, float& w, float m, float v) { w -= o.lr_t * m / (sqrtf(v) + o.epsilon); }

// One update of a TOUCHED row element from its summed gradient g (duplicates already summed: "sum duplicates, apply once").
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
    } else if (o.kind == WD_OPT_ADAM) {             // sparse Adam: decay, scatter-add, step (o.lr_t: with_lr_t)
        adam_decay(o, s1, s2);
        s1 += g * (1.f - o.beta1);
        s2 += g * g * (1.f - o.beta2);
        adam_step(o, w, s1, s2);
    } else {
        w -= o.lr * g;
    }
}

// One update of four consecutive elements of an embedding record [w | s1 | s2]: w points at them, slot k at w + k * gap.
__device__ __forceinline__ void update_record4(const OptParams& o, float* w, int gap, int nslots, float4 g) {
    float4 x = *reinterpret_cast<float4*>(w);
    float4 s1 = nslots >= 1 ? *reinterpret_cast<float4*>(w + gap) : make_float4(0, 0, 0, 0);
    float4 s2 = nslots >= 2 ? *reinterpret_cast<float4*>(w + 2 * gap) : make_float4(0, 0, 0, 0);
    opt_update(o, g.x, x.x, s1.x, s2.x);
    opt_update(o, g.y, x.y, s1.y, s2.y);
    opt_update(o, g.z, x.z, s1.z, s2.z);
    opt_update(o, g.w, x.w, s1.w, s2.w);
    *reinterpret_cast<float4*>(w) = x;
    if (nslots >= 1) *reinterpret_cast<float4*>(w + gap) = s1;
    if (nslots >= 2) *reinterpret_cast<float4*>(w + 2 * gap) = s2;
}
// Adam on four consecutive elements of an embedding record [w | m | v] that no gradient touched this step.
__device__ __forceinline__ void adam_untouched4(const OptParams& o, float* w, int gap) {
    float4 x = *reinterpret_cast<float4*>(w);
    float4 m = *reinterpret_cast<float4*>(w + gap);
    float4 v = *reinterpret_cast<float4*>(w + 2 * gap);
    adam_decay(o, m.x, v.x); adam_step(o, x.x, m.x, v.x);
    adam_decay(o, m.y, v.y); adam_step(o, x.y, m.y, v.y);
    adam_decay(o, m.z, v.z); adam_step(o, x.z, m.z, v.z);
    adam_decay(o, m.w, v.w); adam_step(o, x.w, m.w, v.w);
    *reinterpret_cast<float4*>(w) = x;
    *reinterpret_cast<float4*>(w + gap) = m;
    *reinterpret_cast<float4*>(w + 2 * gap) = v;
}
// One update of a wide record {w, s1, s2, -}.
__device__ __forceinline__ void update_wide(const OptParams& o, float4* rec, float g) {
    float4 r = *rec;
    opt_update(o, g, r.x, r.y, r.z);
    *rec = r;
}

// record of unique row u of the list (global row urow[u], read only for a record in place) in table t.  (Both cases are offsets
// from the table pointer data[t], a pointer loaded from global memory: the compiler then keeps the record's loads and stores global
// ones, where a choice between two pointers would make them generic.)
__device__ __forceinline__ float* record(const RowRecords& r, int t, const uint32_t* urow, int64_t u) {
    float* data = r.data[t];
    const int sst = r.stage ? r.stage[t] : 0;
    return data + (sst ? (r.stage_base - data) + (r.uslot ? (int64_t)r.uslot[u] : u) * sst : ((int64_t)urow[u] - r.row_base[t]) * r.stride[t]);
}

// The optimizer the single-GPU step fuses into its gradient sums: unique row u of the list is global row urow[u]; embedding records
// as `rec` says, wide records at wide[row].
struct RowApply {
    const uint32_t* urow;
    RowRecords rec;
    float4* wide;
    OptParams o;
};

// ---- per unique row: g = ordered sum of its occurrences' gradients.
// Rows touched at most kChunk times are summed by one lane group directly.  Hotter rows (small tables, skewed ids) are split into
// chunks of kChunk occurrences that are summed in parallel and then combined in chunk order (chunk_combine_kernel in sparse.cu),
// so the result stays deterministic and no single group walks thousands of occurrences.  One launch covers both kinds of work
// item: items [0, nu) are the unique rows (summed directly into ugrad unless they are hot), items [nu, nu + nchunks) are the
// chunks of the hot rows (summed into cpart).

// Where an occurrence's gradient comes from is the source's business (Src: LocalEmb / LocalWide in sparse.cu for the batch's own
// lists, PeerEmb / PeerWide in shard.cu for the rows a rank owns).  key(j) is occurrence j of the sorted list; the rows of an item
// all belong to one table, layout(key of its first occurrence) gives (t, dim, x0); row(key, x0, q) is float4 q of the
// occurrence's gradient row and its bag scale inv (embedding), row(key) its dlogit (wide).  Keys are loaded four at a time, then
// their rows, so that four gradient rows are in flight.
// Embedding rows: 8 lanes per work item, each lane covers float4 chunks lig, lig + 8, ... of the row.  APPLY (single-GPU step,
// row-local optimizer): a directly summed row is updated right after its sum — the summed gradient never reaches memory; the hot
// rows are updated by chunk_combine_kernel<1>.
template <class Src, bool APPLY>
__global__ void __launch_bounds__(256) emb_grad_sum_kernel(const int32_t* __restrict__ d_nuniq, const int32_t* __restrict__ d_nchunks,
                                                           const int32_t* __restrict__ ustart, const int32_t* __restrict__ choff, Src src,
                                                           float* __restrict__ ugrad, float* __restrict__ cpart, int width, RowApply ra) {
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int nu = *d_nuniq;
    const int64_t nitems = (int64_t)nu + *d_nchunks;
    const int64_t g0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4 + grp;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    for (int64_t it = g0; it < nitems; it += gstep) {
        int s, e;
        float* out;
        const bool direct = it < nu;
        if (direct) {
            s = ustart[it]; e = ustart[it + 1];
            if (e - s > kChunk) continue;                     // hot row: summed chunk by chunk
            out = ugrad + it * width;
        } else {
            const int c = (int)(it - nu);
            const int u = chunk_owner(choff, nu, c);
            s = ustart[u] + (c - choff[u]) * kChunk;
            e = min(ustart[u + 1], s + kChunk);
            out = cpart + (int64_t)c * width;
        }
        int t, dim, x0;
        src.layout(src.key(s), t, dim, x0);
        for (int q = lig; q * 4 < width; q += 8) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q * 4 < dim) {
                int j = s;
                for (; j + 4 <= e; j += 4) {                  // 4 gradient rows in flight
                    uint32_t k[4]; float4 v[4]; float inv[4];
#pragma unroll
                    for (int r = 0; r < 4; ++r) k[r] = src.key(j + r);
#pragma unroll
                    for (int r = 0; r < 4; ++r) v[r] = src.row(k[r], x0, q, inv[r]);
#pragma unroll
                    for (int r = 0; r < 4; ++r) { acc.x += v[r].x * inv[r]; acc.y += v[r].y * inv[r]; acc.z += v[r].z * inv[r]; acc.w += v[r].w * inv[r]; }
                }
                for (; j < e; ++j) {
                    float inv;
                    const float4 v = src.row(src.key(j), x0, q, inv);
                    acc.x += v.x * inv; acc.y += v.y * inv; acc.z += v.z * inv; acc.w += v.w * inv;
                }
            }
            if (APPLY && direct) {
                if (q * 4 < dim)
                    update_record4(ra.o, record(ra.rec, t, ra.urow, it) + q * 4, dim, kind_nslots(ra.o.kind), acc);
            } else {
                *reinterpret_cast<float4*>(out + q * 4) = acc;
            }
        }
    }
}

// Wide rows: one thread per work item, items as in emb_grad_sum_kernel; APPLY: record {w, s1, s2, -} updated in place.
template <class Src, bool APPLY>
__global__ void wide_grad_sum_kernel(const int32_t* __restrict__ d_nuniq, const int32_t* __restrict__ d_nchunks,
                                     const int32_t* __restrict__ ustart, const int32_t* __restrict__ choff, Src src,
                                     float* __restrict__ ugrad, float* __restrict__ cpart, RowApply ra) {
    const int nu = *d_nuniq;
    const int64_t nitems = (int64_t)nu + *d_nchunks;
    for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < nitems; it += (int64_t)gridDim.x * blockDim.x) {
        int s, e;
        const bool direct = it < nu;
        if (direct) {
            s = ustart[it]; e = ustart[it + 1];
            if (e - s > kChunk) continue;
        } else {
            const int c = (int)(it - nu);
            const int u = chunk_owner(choff, nu, c);
            s = ustart[u] + (c - choff[u]) * kChunk;
            e = min(ustart[u + 1], s + kChunk);
        }
        float acc = 0.f;
        for (int j = s; j < e; ++j) acc += src.row(src.key(j));
        if (!direct) cpart[it - nu] = acc;
        else if (APPLY) update_wide(ra.o, ra.wide + ra.urow[it], acc);
        else ugrad[it] = acc;
    }
}

// ---- list machinery implemented in sparse.cu, used by shard.cu for the rows a rank owns
// sort (row, occurrence) pairs of e_row[0 .. *d_n) by row, unique rows, segment starts, hot-row chunk layout -> list l
int list_group(WdModel* m, RowList& l, const int32_t* d_n, const uint32_t* e_row);
int list_sort_by_key(WdModel* m, RowList& l, const int32_t* d_n, const uint32_t* e_key);
// ugrad[u] = fixed-order sum of the chunk partials of multi-chunk rows (after the two gradient-sum passes)
int list_chunk_combine(WdModel* m, const RowList& l);
// optimizer over the unique rows of list l: embedding records as `rec` says (tables in row order) / one wide record array
int list_apply_emb(WdModel* m, const RowList& l, const RowRecords& rec, const OptParams& o);
int list_apply_wide(WdModel* m, const RowList& l, float4* wide, const OptParams& o);
// the optimizer of table space `space` (0 embedding rows: dnn_optimizer, 1 wide rows: linear_optimizer); Adam: with its beta powers
// and the bitmap `touched` of the record set it updates
OptParams space_opt(const WdModel* m, int space, uint32_t* touched);
// Adam, the untouched pass of one record set (after every touched-row update of the step, on the stream that ran the last of
// them): decay + step of every row whose bit in o.touched is clear, all bits cleared.  Embedding records of `set` in place, table t
// holding set.rows[t] rows from its row base, bits 0 .. nbits; wide records wide[0 .. nbits).  Nothing unless o is Adam.
int adam_untouched_emb(WdModel* m, const RecordSet& set, int64_t nbits, const OptParams& o);
int adam_untouched_wide(WdModel* m, float4* wide, int64_t nbits, const OptParams& o);

}  // namespace wd
