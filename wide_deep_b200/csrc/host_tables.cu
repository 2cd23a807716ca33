// Placement of the embedding tables and the device descriptors every kernel finds their records through.
//
// Record sets (build_record_sets: RecordSet / RowRecords in common.cuh, record() in sparse_dev.cuh).  One builder uploads all of
// them once every table and staging buffer exists and the shard layout is final:
//   set                   order                 row space                 read by
//   by table              plan order            global rows (shard rows   LocalEmb (dim, x0), the fused direct-row update
//     WdModel::tabs                             for a sharded table)      (RowApply ra), the id stage (DevPlan::table_row_base)
//   replicated, by row    global row order:     global rows               the fused hot-row update (ha), emb_apply_kernel, the
//     WdModel::rtabs      large, then small                               small-table block (gs_off), stage-in / write-back /
//                                                                         remap / flush of host tables and the cache, Adam's
//                                                                         untouched pass (rows)
//   shard                 slot order            this rank's shard rows    serve, combine, PeerEmb, the owner apply, stage-in /
//     ShardSpace::set                                                     write-back / flush of host shards and their cache,
//                                                                         the shard's untouched pass
//   HostCache             per record set: WdModel::hcache in front of the replicated set (list 0), ShardSpace::cache in front
//                         of the shard set (list 2); its uslot is the set's RowRecords::uslot
//   gather view           per width,            global rows; a host       emb_pool_fwd_rows_kernel, emb_pool_fwd_kernel<G>
//     WdModel::d_dim_desc table order           table at its staging row
// A host table is staged in the by-table and replicated sets (stage[t] = stage_stride, records in d_stage) and read by the gather
// from the staging buffer; a host shard is staged in the shard set (records in the owner's ShardSpace::d_stage).
//
// Embedding tables in page-locked host memory (WdPlanDesc::table_placement).  The reference keeps its tables in host RAM: it
// trains on the CPU or spreads them over parameter servers (reference python/lib/build_estimator.py:211-214, joint.py:141-143).
//
// A host table's [w | slots] records live in mapped, page-locked host memory.  Every step already sorts its embedding ids into the
// unique-row list urow[0] / ustart[0] (sparse_group_which), and every touched row takes exactly one optimizer update, so one step
// moves exactly one record per unique host row each way over PCIe:
//   stage-in    host_rows_kernel<true>: record of unique row u (host tables only) -> HBM staging buffer row u
//   remap       host_remap_kernel: the gather reads ids in which a host-table entry carries u instead of its global row; the
//               gather kernels see the host tables as (data = staging buffer, row base 0, stride = staging stride)
//   apply       the fused updates address the staged record of u (RowRecords::stage in sparse_dev.cuh)
//   write-back  host_rows_kernel<false>: staging buffer row u -> host record, after the list's apply, on its stream
// With the opt-in HBM cache (wd_host_cache_enable, below) row u is staged in a cache slot that outlives the step, and only the
// rows that miss are moved.
// Every kernel downstream of the stage-in runs on bit-identical values in the same order, so the result equals the HBM-resident
// model's bit for bit.  Updates that do not go through the fused kernels (data-parallel lists: wd_step_backward + wd_step_apply)
// address the host records directly through their mapped pointers.
// Row-sharded tables (shard_world > 1) keep a rank's shard here instead: its owner groups the rows it received (list 2) before
// serving them and stages them into its own buffer through stage_in_rows / write_back_rows (the owner-side step is in shard.cu),
// behind its own HBM cache when wd_shard_cache_enable made one.  Only the sharded tables may go to the host then; the replicated
// ones, the single-GPU staging buffer and the single-GPU cache stay out of it.
//
// Adam (WD_PLACE_DEFER_ADAM).  Sparse Adam moves every row every step; for a row no gradient touched that step is a fixed
// function of the record and the step's lr_t (m *= b1, v *= b2, w -= lr_t m / (sqrt(v) + eps)).  A deferred table skips the
// untouched pass (its RecordSet::rows are 0) and carries a stamp in its record, [w | m | v | stamp float4]: the last Adam step the
// record reflects.  The stamp travels inside the stride through every transfer above.  Invariant: wherever a deferred record lives
// (host, staging row, cache slot), it is the exact state as of its stamp.  stage_in_rows then catches every staged row up
// (adam_catch_up_kernel): steps s+1 .. g (g = WdModel::d_adam_step) in order, with lr_t[j] from the table deferred_adam_setup
// builds with with_lr_t's own expression, so the values are bit-identical to the untouched passes of the table in HBM.  A train
// call stamps g + 1 (the list's update follows, on the staged record, then the write-back); a forward-only call stamps g.  Reads
// of the whole table (wd_tensor_io) settle every host record first; writes stamp every record with g.  wd_tensor_io_rows does the
// same for its rows only.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "sparse_dev.cuh"

namespace wd {

// ---------------------------------------------------------------------------------------------------------- HBM cache
// wd_host_cache_enable (one GPU) and wd_shard_cache_enable (an owner's host shards) turn the front of a staging buffer into an
// 8-way set-associative, write-back cache of host records (HostCache, common.cuh):
//   stage = [C cache slots | overflow rows], one overflow row per unique row a call can stage; slot s * 8 + w is way w of set s
//   set of a row  Fibonacci hash of the row in the set's row space (global rows / shard rows; the hot rows of skewed id streams
//                 are the low ids of every table: a plain modulo would put them into neighbouring sets)
//   stage-in      keys (set of every unique host row) -> stable radix sort by set -> assign (one thread per run of one set: hits
//                 keep their slot, misses take the other ways by (last use, way index), empty ways first, and rows beyond the
//                 ways overflow to staging row C + u) -> transfer (dirty victim home, then the new record in) -> remap
//   write-back    after the list's apply, overflow rows only; cached records stay dirty until they are evicted or flushed
// Train calls mark every slot they use dirty; forward-only calls mark nothing dirty.  Without a cache (C = 0) every row is an
// overflow row at staging row u, uslot is null and the key / sort / assign launches are skipped.
constexpr int kWays = 8;
constexpr uint8_t kLoad = 1, kVictimDirty = 2;      // d_uflag bits

__device__ __forceinline__ uint32_t cache_set_of(uint32_t row, int set_bits) {
    return set_bits ? (row * 0x9E3779B1u) >> (32 - set_bits) : 0u;
}

// key = set of unique row u (host rows) or nsets (HBM rows: sorted last, never assigned), value = u; bumps the call's stamp
__global__ void __launch_bounds__(256) cache_keys_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow, RowRecords rr,
                                                         int set_bits, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                         uint32_t* __restrict__ now) {
    if (blockIdx.x == 0 && threadIdx.x == 0) ++*now;
    const int nu = *d_nuniq;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += gridDim.x * blockDim.x) {
        const uint32_t row = urow[u];
        keys[u] = rr.stage[table_of(rr.row_base, rr.ntab, row)] != 0 ? cache_set_of(row, set_bits) : (1u << set_bits);
        vals[u] = (uint32_t)u;
    }
}

struct CacheMeta { uint32_t* tag; uint32_t* stamp; uint8_t* dirty; const uint32_t* now; unsigned long long* stats; };

// One thread per run of equal sets in the sorted (set, u) pairs; a run lists its rows in ascending row order (stable sort of the
// ascending unique rows).  Writes uslot / uvict / uflag of the run's rows and the set's metadata; counters: hits, loads, overflow
// rows, dirty evictions.
__global__ void __launch_bounds__(256) cache_assign_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ keys,
                                                           const uint32_t* __restrict__ vals, const uint32_t* __restrict__ urow, int set_bits,
                                                           int64_t C, int train, CacheMeta cm, int32_t* __restrict__ uslot,
                                                           uint32_t* __restrict__ uvict, uint8_t* __restrict__ uflag) {
    const int n = *d_nuniq;
    const uint32_t nsets = 1u << set_bits, now = *cm.now;
    unsigned nhit = 0, nload = 0, nover = 0, nevict = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t s = keys[i];
        if (s >= nsets || (i > 0 && keys[i - 1] == s)) continue;
        int e = i + 1;
        while (e < n && keys[e] == s) ++e;
        const int64_t base = (int64_t)s * kWays;
        uint32_t tag[kWays], st[kWays];
        uint8_t dty[kWays];
#pragma unroll
        for (int w = 0; w < kWays; ++w) { tag[w] = cm.tag[base + w]; st[w] = cm.stamp[base + w]; dty[w] = cm.dirty[base + w]; }
        unsigned used = 0;
        for (int j = i; j < e; ++j) {                                   // hits keep their slot
            const uint32_t u = vals[j], row = urow[u];
#pragma unroll
            for (int w = 0; w < kWays; ++w)
                if (tag[w] == row) { used |= 1u << w; uslot[u] = (int32_t)(base + w); uflag[u] = 0; uvict[u] = kInvalidRow; ++nhit; }
        }
        // the other ways by (last use, way index); an empty way has stamp 0, every used one a stamp >= 1
        int order[kWays], nfree = 0;
        for (int w = 0; w < kWays; ++w) {
            if ((used >> w) & 1) continue;
            const uint32_t k = tag[w] == kInvalidRow ? 0u : st[w];
            int p = nfree++;
            for (; p > 0 && (tag[order[p - 1]] == kInvalidRow ? 0u : st[order[p - 1]]) > k; --p) order[p] = order[p - 1];
            order[p] = w;
        }
        int next = 0;
        for (int j = i; j < e; ++j) {                                   // misses, in row order
            const uint32_t u = vals[j], row = urow[u];
            bool hit = false;
#pragma unroll
            for (int w = 0; w < kWays; ++w) hit |= tag[w] == row;      // (a way loaded below holds a row of this run: never equal)
            if (hit) continue;
            if (next < nfree) {
                const int w = order[next++];
                const bool vd = tag[w] != kInvalidRow && dty[w];
                uslot[u] = (int32_t)(base + w);
                uvict[u] = tag[w];
                uflag[u] = kLoad | (vd ? kVictimDirty : 0);
                nevict += vd;
                ++nload;
                tag[w] = row;
                dty[w] = 0;
                used |= 1u << w;
            } else {                                                    // the set is full: staged without a slot
                uslot[u] = (int32_t)(C + u);
                uvict[u] = kInvalidRow;
                uflag[u] = kLoad;
                ++nover;
            }
        }
#pragma unroll
        for (int w = 0; w < kWays; ++w) {
            if ((used >> w) & 1) { st[w] = now; if (train) dty[w] = 1; }
            cm.tag[base + w] = tag[w]; cm.stamp[base + w] = st[w]; cm.dirty[base + w] = dty[w];
        }
    }
    nhit = __reduce_add_sync(0xffffffffu, nhit); nload = __reduce_add_sync(0xffffffffu, nload);
    nover = __reduce_add_sync(0xffffffffu, nover); nevict = __reduce_add_sync(0xffffffffu, nevict);
    if ((threadIdx.x & 31) == 0) {
        if (nhit) atomicAdd(&cm.stats[0], (unsigned long long)nhit);
        if (nload) atomicAdd(&cm.stats[1], (unsigned long long)nload);
        if (nover) atomicAdd(&cm.stats[2], (unsigned long long)nover);
        if (nevict) atomicAdd(&cm.stats[3], (unsigned long long)nevict);
    }
}

// Transfer between the host records of the step's unique host rows (the staged tables of rr) and their staging rows in
// rr.stage_base (rr.uslot[u], or u without a cache).  IN: the record of every row to load -> its staging row; a dirty victim's
// record goes home first (uvict[u], the row the slot held).  !IN: overflow staging rows (>= C) -> host records.  One thread per
// float4 of a staged record, consecutive threads on consecutive float4 of a record (the PCIe transfers are whole records); each
// thread keeps kInFlight float4 in flight.  The thread that writes float4 q of a slot has read the victim's float4 q before, so the
// eviction needs no barrier; a victim is never a row of the current call (that row would have been a hit).
constexpr int kInFlight = 4;
struct StageMap { const uint32_t* uvict; const uint8_t* uflag; int64_t C; };
template <bool IN>
__global__ void __launch_bounds__(256) host_rows_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow, RowRecords rr,
                                                        int S, StageMap sm) {
    float* const stage = rr.stage_base;
    const int q4 = S >> 2;
    const int64_t total = (int64_t)*d_nuniq * q4;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += T * kInFlight) {
        float4 v[kInFlight], vv[kInFlight];
        float *dst[kInFlight], *vdst[kInFlight];
#pragma unroll
        for (int k = 0; k < kInFlight; ++k) {
            dst[k] = vdst[k] = nullptr;
            const int64_t i = i0 + k * T;
            if (i >= total) continue;
            const int64_t u = i / q4;
            const int q = (int)(i - u * q4);
            const int64_t row = urow[u];
            const int lo = table_of(rr.row_base, rr.ntab, row);
            if (rr.stage[lo] == 0) continue;                                 // HBM table
            int64_t srow = u;
            if (rr.uslot) {
                srow = rr.uslot[u];
                if (IN) {
                    const uint8_t f = sm.uflag[u];
                    if (!(f & kLoad)) continue;                              // hit: the slot holds the record
                    if (f & kVictimDirty) {
                        const int64_t vr = sm.uvict[u];
                        const int vlo = table_of(rr.row_base, rr.ntab, vr);
                        const int vstride = rr.stride[vlo];
                        if (q * 4 < vstride) {
                            vv[k] = *reinterpret_cast<const float4*>(stage + srow * S + q * 4);
                            vdst[k] = rr.data[vlo] + (vr - rr.row_base[vlo]) * vstride + q * 4;
                        }
                    }
                } else if (srow < sm.C) continue;                            // cached: stays in its slot
            }
            const int stride = rr.stride[lo];
            if (q * 4 >= stride) continue;                                   // beyond this table's record
            float* rec = rr.data[lo] + (row - rr.row_base[lo]) * stride + q * 4;
            float* st = stage + srow * S + q * 4;
            if (IN) { v[k] = *reinterpret_cast<const float4*>(rec); dst[k] = st; }
            else { v[k] = *reinterpret_cast<const float4*>(st); dst[k] = rec; }
        }
#pragma unroll
        for (int k = 0; k < kInFlight; ++k) {
            if (IN && vdst[k]) *reinterpret_cast<float4*>(vdst[k]) = vv[k];
            if (dst[k]) *reinterpret_cast<float4*>(dst[k]) = v[k];
        }
    }
}

// gather ids: e_emb, with the entries of host tables replaced by the staging row of their unique row u (uslot[u], or u without a
// cache; urow[0..nu) is sorted ascending)
__global__ void __launch_bounds__(256) host_remap_kernel(const int32_t* __restrict__ d_nnz, const uint32_t* __restrict__ e_emb,
                                                         const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow, RowRecords rr,
                                                         uint32_t* __restrict__ g_emb) {
    const int n = *d_nnz, nu = *d_nuniq;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t r = e_emb[i];
        uint32_t g = r;
        if (r != kInvalidRow && rr.stage[table_of(rr.row_base, rr.ntab, r)] != 0) {
            const int u = lower_bound_u32(urow, nu, r);
            g = rr.uslot ? (uint32_t)rr.uslot[u] : (uint32_t)u;
        }
        g_emb[i] = g;
    }
}

// dirty slots of rr.stage_base that hold a row in [row_lo, row_hi) -> host records: one warp per slot reads the slot's tag and dirty
// byte once, and its lanes copy the record's float4s
__global__ void __launch_bounds__(256) cache_flush_kernel(int64_t C, int S, const uint32_t* __restrict__ tag, const uint8_t* __restrict__ dirty,
                                                          RowRecords rr, int64_t row_lo, int64_t row_hi) {
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, wstep = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t slot = w0; slot < C; slot += wstep) {
        const int64_t row = tag[slot];
        if (!dirty[slot] || row == kInvalidRow || row < row_lo || row >= row_hi) continue;
        const int t = table_of(rr.row_base, rr.ntab, row);
        const int stride = rr.stride[t];
        float* dst = rr.data[t] + (row - rr.row_base[t]) * stride;
        const float* src = rr.stage_base + slot * S;
        for (int q = lane; q * 4 < stride; q += 32)
            *reinterpret_cast<float4*>(dst + q * 4) = *reinterpret_cast<const float4*>(src + q * 4);
    }
}
// slots whose tag is in [row_lo, row_hi) (every slot, empty ones included, when the range covers all 32-bit tags)
__global__ void cache_clear_kernel(int64_t C, uint32_t* __restrict__ tag, uint32_t* __restrict__ stamp, uint8_t* __restrict__ dirty, int invalidate,
                                   int64_t row_lo, int64_t row_hi) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < C; i += (int64_t)gridDim.x * blockDim.x) {
        if ((int64_t)tag[i] < row_lo || (int64_t)tag[i] >= row_hi) continue;
        dirty[i] = 0;
        if (invalidate) { tag[i] = kInvalidRow; stamp[i] = 0; }
    }
}

// ---------------------------------------------------------------------------------------------------- deferred Adam
// Steps past lr_t_last have lr_t == lr exactly (both 1 - beta^j round to 1).  The table must end there: betas so close to 1 that it
// would be longer than this are refused.
constexpr int64_t kMaxLrT = 1 << 22;
struct AdamReplay { const float* lr_t; int64_t last; const uint32_t* now; unsigned long long* stats; };

// Steps s+1 .. g of Adam's untouched update on four consecutive elements of a record [w | m | v] (gap floats apart); returns the
// steps run.  Past `last` every step is the same map, so once a step leaves all twelve values' bits unchanged the rest are skipped.
__device__ __forceinline__ uint32_t adam_replay4(OptParams o, const AdamReplay& ar, float* w, int gap, uint32_t s, uint32_t g) {
    float4 x = *reinterpret_cast<float4*>(w), mm = *reinterpret_cast<float4*>(w + gap), vv = *reinterpret_cast<float4*>(w + 2 * gap);
    uint32_t j = s + 1;
    for (; j <= g; ++j) {
        o.lr_t = (int64_t)j <= ar.last ? ar.lr_t[j] : o.lr;
        const float4 x0 = x, m0 = mm, v0 = vv;
        adam_decay(o, mm.x, vv.x); adam_step(o, x.x, mm.x, vv.x);
        adam_decay(o, mm.y, vv.y); adam_step(o, x.y, mm.y, vv.y);
        adam_decay(o, mm.z, vv.z); adam_step(o, x.z, mm.z, vv.z);
        adam_decay(o, mm.w, vv.w); adam_step(o, x.w, mm.w, vv.w);
        if ((int64_t)j > ar.last) {
            const bool same = __float_as_uint(x.x) == __float_as_uint(x0.x) && __float_as_uint(x.y) == __float_as_uint(x0.y) &&
                              __float_as_uint(x.z) == __float_as_uint(x0.z) && __float_as_uint(x.w) == __float_as_uint(x0.w) &&
                              __float_as_uint(mm.x) == __float_as_uint(m0.x) && __float_as_uint(mm.y) == __float_as_uint(m0.y) &&
                              __float_as_uint(mm.z) == __float_as_uint(m0.z) && __float_as_uint(mm.w) == __float_as_uint(m0.w) &&
                              __float_as_uint(vv.x) == __float_as_uint(v0.x) && __float_as_uint(vv.y) == __float_as_uint(v0.y) &&
                              __float_as_uint(vv.z) == __float_as_uint(v0.z) && __float_as_uint(vv.w) == __float_as_uint(v0.w);
            if (same) { ++j; break; }
        }
    }
    if (j > s + 1) {
        *reinterpret_cast<float4*>(w) = x;
        *reinterpret_cast<float4*>(w + gap) = mm;
        *reinterpret_cast<float4*>(w + 2 * gap) = vv;
    }
    return j - (s + 1);
}

// One deferred record caught up by the 8 lanes of a lane group (mask gm; lane lig takes float4 chunks lig, lig + 8, ...), then
// stamped: train ? g + 1 : max(stamp, g).  Counters of lane 0 of the group accumulate in cnt.
struct CatchUpCount { unsigned long long rows = 0, replayed = 0, skipped = 0, gap = 0; };
__device__ __forceinline__ void catch_up_record(const OptParams& o, const AdamReplay& ar, float* rec, int dim, uint32_t g, bool train,
                                                unsigned gm, int lig, CatchUpCount& cnt) {
    uint32_t* stamp = reinterpret_cast<uint32_t*>(rec + 3 * dim);
    const uint32_t s = *stamp;
    uint32_t run = 0;
    if (s < g)
        for (int q = lig; q * 4 < dim; q += 8) run = max(run, adam_replay4(o, ar, rec + q * 4, dim, s, g));
    run = __reduce_max_sync(gm, run);                   // (every lane has read the stamp before lane 0 writes it)
    if (lig == 0) {
        *stamp = train ? g + 1 : max(s, g);
        if (s < g) {
            cnt.rows++; cnt.replayed += run; cnt.skipped += (g - s) - run;
            cnt.gap = max(cnt.gap, (unsigned long long)(g - s));
        }
    }
}
__device__ __forceinline__ void catch_up_flush(const AdamReplay& ar, const CatchUpCount& c) {
    unsigned long long r = c.rows, p = c.replayed, k = c.skipped, gp = c.gap;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        r += __shfl_xor_sync(0xffffffffu, r, d); p += __shfl_xor_sync(0xffffffffu, p, d);
        k += __shfl_xor_sync(0xffffffffu, k, d); gp = max(gp, __shfl_xor_sync(0xffffffffu, gp, d));
    }
    if ((threadIdx.x & 31) == 0 && r) {
        atomicAdd(&ar.stats[0], r); atomicAdd(&ar.stats[1], p); atomicAdd(&ar.stats[2], k); atomicMax(&ar.stats[3], gp);
    }
}

// The staged records of list L's unique host rows (rr.uslot[u], or u), one lane group of 8 per row.  The trip count of a warp's
// loop is made warp-uniform so that the counters are reduced by the whole warp.
__global__ void __launch_bounds__(256) adam_catch_up_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow,
                                                            RowRecords rr, OptParams o, AdamReplay ar, int train) {
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const unsigned gm = 0xFFu << (grp * 8);
    const int nu = *d_nuniq;
    const uint32_t g = *ar.now;
    const int64_t w0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    CatchUpCount cnt;
    for (int64_t u0 = w0; u0 < nu; u0 += gstep) {
        const int64_t u = u0 + grp;
        if (u >= nu) continue;
        const int64_t row = urow[u];
        const int t = table_of(rr.row_base, rr.ntab, row);
        if (rr.stage[t] == 0) continue;                                  // HBM table
        catch_up_record(o, ar, record(rr, t, urow, u), rr.dim[t], g, train != 0, gm, lig, cnt);
    }
    catch_up_flush(ar, cnt);
}

// Host records row0 .. row0 + rows - 1 of one deferred table in place (records of `stride` floats at data): caught up to g, or only
// stamped g.
__global__ void __launch_bounds__(256) adam_settle_kernel(float* data, int64_t row0, int64_t rows, int dim, int stride, OptParams o,
                                                          AdamReplay ar, int stamp_only) {
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const unsigned gm = 0xFFu << (grp * 8);
    const uint32_t g = *ar.now;
    const int64_t w0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    CatchUpCount cnt;
    for (int64_t r0 = w0; r0 < rows; r0 += gstep) {
        const int64_t r = r0 + grp;
        if (r >= rows) continue;
        float* rec = data + (row0 + r) * stride;
        if (stamp_only) { if (lig == 0) *reinterpret_cast<uint32_t*>(rec + 3 * dim) = g; }
        else catch_up_record(o, ar, rec, dim, g, false, gm, lig, cnt);
    }
    catch_up_flush(ar, cnt);
}

// lr_t[j] = with_lr_t of step j (beta powers bp[2j], bp[2j + 1]), j = 1 .. n
__global__ void adam_lr_t_kernel(OptParams o, const float* __restrict__ bp, int64_t n, float* __restrict__ lr_t) {
    for (int64_t j = 1 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j <= n; j += (int64_t)gridDim.x * blockDim.x) {
        OptParams p = o;
        p.bpow = bp + 2 * j;
        lr_t[j] = with_lr_t(p).lr_t;
    }
}

static AdamReplay adam_replay(const WdModel* m) { return AdamReplay{m->d_lr_t, m->lr_t_last, m->d_adam_step, m->d_defer_stats}; }

// The lr_t table of the deferred tables and their counters.  The beta powers are multiplied up on the host in fp32 exactly as
// adam_tick_kernel and wd_set_opt_step do (beta^1 before the first step), up to the first step at which both 1 - beta^j round to
// 1; lr_t itself is computed on the device by with_lr_t's expression.
int deferred_adam_setup(WdModel* m) {
    const WdOptimizer& o = m->dnn_opt;
    std::vector<float> bp = {0.f, 0.f, o.beta1, o.beta2};
    float b1 = o.beta1, b2 = o.beta2;
    int64_t j = 1;
    while (!(1.f - b1 == 1.f && 1.f - b2 == 1.f)) {
        if (j >= kMaxLrT) {
            set_error("WD_PLACE_DEFER_ADAM: Adam betas (%g, %g) need more than %lld steps before lr_t reaches lr", (double)o.beta1,
                      (double)o.beta2, (long long)kMaxLrT);
            return WD_EUNSUPPORTED;
        }
        b1 *= o.beta1; b2 *= o.beta2;
        bp.push_back(b1); bp.push_back(b2);
        ++j;
    }
    m->lr_t_last = j;
    int rc;
    float* d_bp = nullptr;
    if ((rc = dev_alloc(m, &m->d_lr_t, j + 1))) return rc;
    if ((rc = dev_alloc(m, &m->d_defer_stats, 4))) return rc;
    if ((rc = upload(m, &d_bp, bp))) return rc;
    adam_lr_t_kernel<<<grid_for(j, 256), 256, 0, m->stream>>>(make_opt(o), d_bp, j, m->d_lr_t);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return dev_free(m, d_bp);
}

static int adam_catch_up(WdModel* m, int L, const RowRecords& rr, bool train) {
    const RowList& l = m->lists[L];
    adam_catch_up_kernel<<<grid_for(m->max_nnz * 8, 256), 256, 0, m->stream>>>(l.nuniq, l.urow, rr, make_opt(m->dnn_opt), adam_replay(m),
                                                                               train ? 1 : 0);
    m->launches++;
    mark(m, "adam_catch_up");
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int deferred_adam_settle(WdModel* m, const EmbTable& tb, int64_t row0, int64_t rows, bool stamp_only) {
    if (rows <= 0) return WD_OK;
    adam_settle_kernel<<<grid_for(rows * 8, 256), 256, 0, m->stream>>>(tb.data, row0, rows, tb.dim, tb.stride, make_opt(m->dnn_opt),
                                                                      adam_replay(m), stamp_only ? 1 : 0);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int stage_in_rows(WdModel* m, HostCache& c, int L, const RowRecords& rr, int S, bool train, const CacheMarks& marks) {
    const RowList& l = m->lists[L];
    const int64_t C = c.slots;
    if (C > 0) {
        const int g = grid_for(m->max_nnz, 256);
        cache_keys_kernel<<<g, 256, 0, m->stream>>>(l.nuniq, l.urow, rr, c.set_bits, c.d_ck[0], c.d_cv[0], c.d_now);
        m->launches++;
        int rc = radix_sort_pairs(m, &c.d_ck[0], &c.d_cv[0], &c.d_ck[1], &c.d_cv[1], c.set_bits + 1, l.nuniq);
        if (rc) return rc;
        mark(m, marks.sort);
        const CacheMeta cm{c.d_tag, c.d_stamp, c.d_dirty, c.d_now, c.d_stats};
        cache_assign_kernel<<<g, 256, 0, m->stream>>>(l.nuniq, c.d_ck[0], c.d_cv[0], l.urow, c.set_bits, C, train ? 1 : 0, cm,
                                                     c.d_uslot, c.d_uvict, c.d_uflag);
        m->launches++;
        mark(m, marks.assign);
    }
    const StageMap sm{c.d_uvict, c.d_uflag, C};
    host_rows_kernel<true><<<grid_for(m->max_nnz * (S / 4) / kInFlight, 256), 256, 0, m->stream>>>(l.nuniq, l.urow, rr, S, sm);
    m->launches++;
    if (marks.in) mark(m, marks.in);
    WD_CUDA(cudaGetLastError());
    // with Adam every staged table is a deferred one (place_tables): its rows (loads and cache hits alike) catch up here
    return m->n_defer_tab > 0 ? adam_catch_up(m, L, rr, train) : WD_OK;
}

int write_back_rows(WdModel* m, const HostCache& c, int L, const RowRecords& rr, int S, const CacheMarks& marks) {
    const RowList& l = m->lists[L];
    const StageMap sm{c.d_uvict, c.d_uflag, c.slots};
    host_rows_kernel<false><<<grid_for(m->max_nnz * (S / 4) / kInFlight, 256), 256, 0, m->stream>>>(l.nuniq, l.urow, rr, S, sm);
    m->launches++;
    mark(m, marks.out);
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

static const CacheMarks kHostMarks{"cache_sort", "cache_assign", nullptr, "write_back"};

int host_tables_stage_in(WdModel* m, bool train) {
    const RowRecords& rr = m->rtabs.rec;
    int rc = stage_in_rows(m, m->hcache, 0, rr, m->stage_stride, train, kHostMarks);
    if (rc) return rc;
    host_remap_kernel<<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(m->d_nnz, m->d_e_emb, m->lists[0].nuniq, m->lists[0].urow, rr, m->d_g_emb);
    m->launches++;
    mark(m, "stage_in");
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int host_tables_write_back(WdModel* m) { return write_back_rows(m, m->hcache, 0, m->rtabs.rec, m->stage_stride, kHostMarks); }

// Everything that reads or writes host records outside the step, for the slots holding a row of [row_lo, row_hi) in the set's row
// space: flush = dirty slots home (they stay cached, now clean), invalidate = empty the slots (after the host records were
// rewritten).  Enqueued on the model stream.  One pass over the slots' metadata either way, whatever the range.
static int cache_sync(WdModel* m, HostCache& c, const RowRecords& rr, int S, bool flush, bool invalidate, int64_t row_lo, int64_t row_hi) {
    const int64_t C = c.slots;
    if (C == 0) return WD_OK;
    if (flush) {
        cache_flush_kernel<<<grid_for(C * 32, 256), 256, 0, m->stream>>>(C, S, c.d_tag, c.d_dirty, rr, row_lo, row_hi);
        m->launches++;
    }
    cache_clear_kernel<<<grid_for(C, 256), 256, 0, m->stream>>>(C, c.d_tag, c.d_stamp, c.d_dirty, invalidate ? 1 : 0, row_lo, row_hi);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
constexpr int64_t kEveryTag = int64_t(1) << 32;       // hi of a range that holds every tag, kInvalidRow (empty slots) included
// the model's cache, whichever it has (the single-GPU one or the owner's cache of its host shards)
int host_cache_sync(WdModel* m, bool flush, bool invalidate) {
    ShardSpace& se = m->shard.sp[0];
    int rc = cache_sync(m, m->hcache, m->rtabs.rec, m->stage_stride, flush, invalidate, 0, kEveryTag);
    return rc ? rc : cache_sync(m, se.cache, se.set.rec, se.stage_stride, flush, invalidate, 0, kEveryTag);
}
// The cached records of host table tb's rows row0 .. row0 + rows - 1 (local rows; a shard's rows for a sharded table): dirty ones
// go home, and with invalidate the slots holding them are emptied.  The single-GPU cache tags global rows, an owner's cache its
// shard rows: tb.row_base counts in that space either way.
int host_cache_sync_rows(WdModel* m, const EmbTable& tb, int64_t row0, int64_t rows, bool invalidate) {
    ShardSpace& se = m->shard.sp[0];
    const int64_t row_lo = tb.row_base + row0;
    if (tb.sharded) return cache_sync(m, se.cache, se.set.rec, se.stage_stride, true, invalidate, row_lo, row_lo + rows);
    return cache_sync(m, m->hcache, m->rtabs.rec, m->stage_stride, true, invalidate, row_lo, row_lo + rows);
}

// Allocates every embedding table — in HBM (WD_PLACE_HBM, and WD_PLACE_AUTO tables while they fit, largest first, with
// `hbm_reserve` bytes held back for the buffers allocated after wd_model_create) or in mapped page-locked host memory — and the
// staging buffer of the host tables.  The descriptors that point at them come later (build_record_sets).  A row-sharded model
// (shard_world > 1) may place only its sharded tables on the host: this rank's shard lives there and its owner-side step
// (shard.cu) stages it through the owner staging buffer allocated here.
int place_tables(WdModel* m, int64_t hbm_reserve) {
    const int nt = (int)m->tables.size();
    auto host_ok = [&](const EmbTable& tb) {
        if (m->dnn_opt.kind == WD_OPT_ADAM && !tb.defer) return false;
        return m->shard.world > 1 ? tb.sharded : m->dense_exchange_max_rows <= 0;
    };
    for (int t = 0; t < nt; ++t)
        if (m->tables[t].place == WD_PLACE_HOST && !host_ok(m->tables[t])) {
            set_error("table %d: host placement is not supported for a replicated table of a row-sharded model, with "
                      "dense_exchange_max_rows > 0 on one GPU or with the Adam dnn optimizer (its sparse update decays the whole table "
                      "every step, unless the table has WD_PLACE_DEFER_ADAM)", t);
            return WD_EUNSUPPORTED;
        }
    auto bytes_of = [&](int t) { return m->tables[t].arows * (int64_t)m->tables[t].stride * 4; };
    int rc;
    std::vector<int> autos;
    for (int t = 0; t < nt; ++t) {
        EmbTable& tb = m->tables[t];
        tb.host = tb.place == WD_PLACE_HOST;
        if (tb.place == WD_PLACE_AUTO && host_ok(tb)) autos.push_back(t);
        else if (!tb.host && (rc = dev_alloc(m, &tb.data, tb.arows * tb.stride, true))) return rc;
    }
    if (!autos.empty()) {
        std::stable_sort(autos.begin(), autos.end(), [&](int a, int b) { return bytes_of(a) > bytes_of(b); });
        void* hold = nullptr;
        if (hbm_reserve > 0 && cudaMalloc(&hold, (size_t)hbm_reserve) != cudaSuccess) { hold = nullptr; cudaGetLastError(); }
        for (int t : autos) {
            EmbTable& tb = m->tables[t];
            if (dev_alloc(m, &tb.data, tb.arows * tb.stride, true) != WD_OK) { cudaGetLastError(); tb.host = true; }
        }
        if (hold) cudaFree(hold);
        set_error("");
    }
    for (int t = 0; t < nt; ++t) {
        EmbTable& tb = m->tables[t];
        if (!tb.host) continue;
        void* p = nullptr;
        if (cudaHostAlloc(&p, (size_t)bytes_of(t), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError();
            set_error("table %d: cudaHostAlloc of %lld bytes failed", t, (long long)bytes_of(t));
            return WD_ENOMEM;
        }
        m->host_allocs.push_back(p);
        m->host_bytes += bytes_of(t);
        void* dp = nullptr;
        WD_CUDA(cudaHostGetDevicePointer(&dp, p, 0));
        tb.data = (float*)dp;                // every element is written by init_sparse_tables before first use
        if (!tb.sharded) m->n_host_tab++;    // (a host shard is staged by its owner, in the shard's own buffer)
        if (tb.defer) m->n_defer_tab++;
        int& stage_stride = tb.sharded ? m->shard.sp[0].stage_stride : m->stage_stride;
        stage_stride = std::max(stage_stride, tb.stride);
    }

    if (m->n_host_tab > 0) {
        if ((rc = dev_alloc(m, &m->d_stage, m->max_nnz * (int64_t)m->stage_stride, true))) return rc;
        if ((rc = dev_alloc(m, &m->d_g_emb, m->max_nnz, true))) return rc;
    } else {
        m->d_g_emb = m->d_e_emb;             // nothing on the host: the gather reads the step's own ids
    }
    // host shards: the owner's staging rows of the step's unique owned rows (+1: see the serve in shard.cu)
    ShardSpace& se = m->shard.sp[0];
    if (se.stage_stride > 0 && (rc = dev_alloc(m, &se.d_stage, (m->max_nnz + 1) * (int64_t)se.stage_stride, false))) return rc;
    return m->n_defer_tab > 0 ? deferred_adam_setup(m) : WD_OK;
}

// dst = per-table values f(table) of the tables `ids`, in that order
template <typename T, typename F>
static int upload_per_table(WdModel* m, T** dst, const std::vector<int>& ids, F f) {
    std::vector<std::remove_const_t<T>> h;
    for (int t : ids) h.push_back(f(m->tables[t]));
    return upload(m, dst, h);
}
// the records of the tables `ids`, in that order; a host table is staged (stage stride S, records in stage_base) when S > 0
static int upload_records(WdModel* m, RowRecords& r, const std::vector<int>& ids, int S, float* stage_base, const int32_t* uslot) {
    int rc;
    r.ntab = (int)ids.size();
    r.stage_base = stage_base;
    r.uslot = uslot;
    if ((rc = upload_per_table(m, &r.row_base, ids, [](const EmbTable& tb) { return tb.row_base; }))) return rc;
    if ((rc = upload_per_table(m, &r.data, ids, [](const EmbTable& tb) { return tb.data; }))) return rc;
    if ((rc = upload_per_table(m, &r.dim, ids, [](const EmbTable& tb) { return (int32_t)tb.dim; }))) return rc;
    if ((rc = upload_per_table(m, &r.stride, ids, [](const EmbTable& tb) { return (int32_t)tb.stride; }))) return rc;
    if (S > 0 && (rc = upload_per_table(m, &r.stage, ids, [&](const EmbTable& tb) { return tb.host ? S : 0; }))) return rc;
    return WD_OK;
}

// Uploads the record sets and the gather view (table at the top of this file) from the tables as they stand.  build_model runs it
// once every table and staging buffer exists and the shard layout is final (shard_build moves the sharded tables' row bases into
// the shard's row space); wd_host_cache_enable and wd_shard_cache_enable run it again after replacing a staging buffer: every array
// exists by then and is overwritten in place.
int build_record_sets(WdModel* m) {
    int rc;
    std::vector<int> all(m->tables.size()), slots;
    for (size_t t = 0; t < m->tables.size(); ++t) {
        all[t] = (int)t;
        if (m->tables[t].sharded) slots.push_back((int)t);          // slot order = table order (shard_build)
    }
    auto x0_of = [](const EmbTable& tb) { return (int32_t)tb.x0_off; };
    auto rows_of = [](const EmbTable& tb) { return deferred(tb) ? (int64_t)0 : tb.arows; };   // (read by the untouched pass only)
    if (!m->tables.empty()) {
        // by table
        if ((rc = upload_records(m, m->tabs.rec, all, m->stage_stride, m->d_stage, m->hcache.d_uslot))) return rc;
        if ((rc = upload_per_table(m, &m->tabs.x0, all, x0_of))) return rc;
        m->dplan.table_row_base = m->tabs.rec.row_base;
        // replicated, by row
        if ((rc = upload_records(m, m->rtabs.rec, m->rtab_order, m->stage_stride, m->d_stage, m->hcache.d_uslot))) return rc;
        if ((rc = upload_per_table(m, &m->rtabs.rows, m->rtab_order, rows_of))) return rc;
        if ((rc = upload_per_table(m, &m->rtabs.gs_off, m->rtab_order, [](const EmbTable& tb) { return tb.gs_off; }))) return rc;
    }
    // shard: the embedding space's records; the wide space has only its columns' row bases
    ShardSpace& se = m->shard.sp[0];
    if (se.on) {
        if ((rc = upload_records(m, se.set.rec, slots, se.stage_stride, se.d_stage, se.cache.d_uslot))) return rc;
        if ((rc = upload_per_table(m, &se.set.x0, slots, x0_of))) return rc;
        if ((rc = upload_per_table(m, &se.set.rows, slots, rows_of))) return rc;
    }
    ShardSpace& sw = m->shard.sp[1];
    if (sw.on) {
        sw.set.rec.ntab = sw.n_slots;
        if ((rc = upload(m, &sw.set.rec.row_base, sw.h_slot_base))) return rc;
    }
    // gather view: per width, the replicated tables in table order; a host table read from the staging buffer (row base 0)
    for (int i = 0; i < m->n_dims; ++i) {
        std::vector<TabDesc> descs;
        for (const EmbTable& tb : m->tables) {
            if (tb.dim != m->dims[i] || tb.sharded) continue;
            descs.push_back(tb.host ? TabDesc{m->d_stage, 0, m->stage_stride, tb.x0_off, tb.col, tb.dim}
                                    : TabDesc{tb.data, tb.row_base, tb.stride, tb.x0_off, tb.col, tb.dim});
        }
        if ((rc = upload(m, &m->d_dim_desc[i], descs))) return rc;
    }
    return WD_OK;
}

// Turns the front of the staging buffer *stage (stride S, `rows` rows: one per unique row a call can stage) into cache `c` of at
// most `bytes` of slots: *stage becomes [C slots | rows overflow rows] and the record sets are uploaded again.  Capacity 0 (nothing
// allocated) when the budget is below one set.  `who` names the entry point in the error messages.
static int cache_enable(WdModel* m, HostCache& c, int64_t bytes, int S, int64_t rows, float** stage, const char* who) {
    const int64_t slot_bytes = (int64_t)S * 4;
    const int64_t sets = bytes / (kWays * slot_bytes);
    if (sets < 1) return WD_OK;
    int bits = 0;
    while (((int64_t)2 << bits) <= sets) ++bits;
    const int64_t C = (int64_t)kWays << bits;
    if (C + rows >= ((int64_t)1 << 31)) {
        set_error("%s: %lld slots + %lld overflow rows do not fit 31-bit staging rows", who, (long long)C, (long long)rows);
        return WD_EINVAL;
    }
    // HBM the cache adds: its slots, per-slot tag / stamp / dirty, and per unique row uslot / uvict / uflag + the (set, u) sort pairs
    const int64_t meta = C * 9 + 4 + 4 * 8 + rows * 9 + 4 * (m->max_nnz + 8) * 4;
    size_t free_b = 0, total_b = 0;
    WD_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const int64_t reserve = hbm_reserve_bytes(m);
    if ((int64_t)free_b - (C * slot_bytes + meta) < reserve) {
        set_error("%s: a cache of %lld bytes would leave %lld bytes of HBM free, less than the %lld the model keeps for its later allocations",
                  who, (long long)(C * slot_bytes), (long long)((int64_t)free_b - C * slot_bytes - meta), (long long)reserve);
        return WD_ENOMEM;
    }
    // the staging buffer grows to [C slots | rows overflow rows]: the old one is freed and every descriptor re-pointed
    WD_CUDA(cudaStreamSynchronize(m->stream));
    int rc;
    if ((rc = dev_free(m, *stage))) return rc;
    *stage = nullptr;
    if ((rc = dev_alloc(m, stage, (C + rows) * S, false))) return rc;
    if ((rc = dev_alloc(m, &c.d_tag, C, false))) return rc;
    WD_CUDA(cudaMemsetAsync(c.d_tag, 0xFF, C * 4, m->stream));         // kInvalidRow
    if ((rc = dev_alloc(m, &c.d_stamp, C))) return rc;
    if ((rc = dev_alloc(m, &c.d_dirty, C))) return rc;
    if ((rc = dev_alloc(m, &c.d_now, 1))) return rc;
    if ((rc = dev_alloc(m, &c.d_stats, 4))) return rc;
    if ((rc = dev_alloc(m, &c.d_uslot, rows))) return rc;
    if ((rc = dev_alloc(m, &c.d_uvict, rows))) return rc;
    if ((rc = dev_alloc(m, &c.d_uflag, rows))) return rc;
    for (int k = 0; k < 2; ++k) {
        if ((rc = dev_alloc(m, &c.d_ck[k], m->max_nnz + 8))) return rc;
        if ((rc = dev_alloc(m, &c.d_cv[k], m->max_nnz + 8))) return rc;
    }
    c.slots = C;
    c.set_bits = bits;
    if ((rc = build_record_sets(m))) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

// the checks both entry points share: arguments, and no step or forward issued and no cache yet
static int cache_enable_check(WdModel* m, int64_t bytes, const char* who) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    if (bytes < 0) { set_error("%s: negative budget %lld", who, (long long)bytes); return WD_EINVAL; }
    if (m->stepped) { set_error("%s after the first step or forward: the step graphs are already captured", who); return WD_ESTATE; }
    if (m->hcache.slots > 0 || m->shard.sp[0].cache.slots > 0) { set_error("%s: the cache is already enabled", who); return WD_ESTATE; }
    return WD_OK;
}

// ------------------------------------------------------------------------------------------------------------ C-ABI
extern "C" int wd_host_cache_enable(WdModel* m, int64_t bytes) {
    int rc = cache_enable_check(m, bytes, "wd_host_cache_enable");
    if (rc) return rc;
    WD_CUDA(cudaSetDevice(m->device));
    if (m->shard.world > 1 && m->host_bytes > 0) {
        set_error("wd_host_cache_enable: the host-placed shards of a row-sharded model are cached by their owner: use wd_shard_cache_enable");
        return WD_EUNSUPPORTED;
    }
    if (m->n_host_tab == 0) return WD_OK;                                // nothing on the host: capacity 0
    return cache_enable(m, m->hcache, bytes, m->stage_stride, m->max_nnz, &m->d_stage, "wd_host_cache_enable");
}

// The owner's cache of this rank's host shards: the rows of list 2 (every unique owned row of a call, max_nnz + 1 staging rows:
// see the serve in shard.cu) in the shard set's row space.
extern "C" int wd_shard_cache_enable(WdModel* m, int64_t bytes) {
    int rc = cache_enable_check(m, bytes, "wd_shard_cache_enable");
    if (rc) return rc;
    if (m->shard.world <= 1) {
        set_error("wd_shard_cache_enable: the model is not row-sharded (shard_world <= 1); its host tables are cached by wd_host_cache_enable");
        return WD_EUNSUPPORTED;
    }
    WD_CUDA(cudaSetDevice(m->device));
    ShardSpace& se = m->shard.sp[0];
    if (se.stage_stride == 0) return WD_OK;                              // no host shard on this rank: capacity 0
    return cache_enable(m, se.cache, bytes, se.stage_stride, m->max_nnz + 1, &se.d_stage, "wd_shard_cache_enable");
}

extern "C" int wd_deferred_adam_stats(WdModel* m, int64_t* out, int32_t n, int32_t reset) {
    if (!m || n < 0 || (n > 0 && !out)) { set_error("null argument"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    unsigned long long h[4] = {0, 0, 0, 0};
    if (m->d_defer_stats) WD_CUDA(cudaMemcpy(h, m->d_defer_stats, sizeof(h), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n && i < 4; ++i) out[i] = (int64_t)h[i];
    if (reset && m->d_defer_stats) {
        WD_CUDA(cudaMemsetAsync(m->d_defer_stats, 0, sizeof(h), m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
    }
    return WD_OK;
}

extern "C" int wd_host_cache_stats(WdModel* m, int64_t* out, int32_t n, int32_t reset) {
    if (!m || n < 0 || (n > 0 && !out)) { set_error("null argument"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    const HostCache& c = m->hcache.slots > 0 ? m->hcache : m->shard.sp[0].cache;
    unsigned long long h[4] = {0, 0, 0, 0};
    if (c.d_stats) WD_CUDA(cudaMemcpy(h, c.d_stats, sizeof(h), cudaMemcpyDeviceToHost));
    const int64_t v[5] = {c.slots, (int64_t)h[0], (int64_t)h[1], (int64_t)h[2], (int64_t)h[3]};
    for (int i = 0; i < n && i < 5; ++i) out[i] = v[i];
    if (reset && c.d_stats) {
        WD_CUDA(cudaMemsetAsync(c.d_stats, 0, sizeof(h), m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
    }
    return WD_OK;
}

}  // namespace wd
