// Row-sharded tables: embedding tables and wide columns too large to replicate are split by row over the G ranks of one box
// (row id -> owner rank id mod G, local row id / G) and reached through PEER MEMORY over NVLink instead of a collective library.
//
// The reference partitions its large variables over parameter-server tasks with tf.min_max_variable_partitioner (reference
// python/lib/joint.py:141-143) and lets every worker pull rows / push sparse updates asynchronously (python/train.py:197-217).
// Here the same partitioning is synchronous and exact — G ranks on G batch shards compute what one rank computes on the
// concatenated batch — and every transfer is fused into the kernel that produces or consumes the data:
//
//   route + send   (requester) ids of sharded columns are grouped by owner (one stable radix pass) and written as
//                  {local row, bag} pairs straight into the owner's inbox (P2P stores)
//   serve          (owner)     gathers the rows of each received bag from its shard, pools them (partial sum) and writes the
//                  pooled vector straight into the requester's receive buffer (P2P stores): gather + all-to-all in one kernel
//   combine        (requester) sums the <= G partials of a bag in rank order, applies the mean, writes the deep-input slice /
//                  adds the wide partial logits
//   backward       (owner)     sorts the received rows, then PULLS each occurrence's gradient (the requester's dX0 slice or
//                  dlogit, P2P loads) while summing per row in a fixed order — the gradient-sum kernels of the local lists
//                  (sparse_dev.cuh) over a peer occurrence source —, and applies Adagrad / FTRL to its shard: the all-to-all of
//                  gradients is fused into the segmented reduction, the optimizer runs once per touched row
//   dense          gradients of the MLP / wide bias / small replicated tables: two-shot all-reduce over peer memory (each rank
//                  reduces one slice in rank order, then every rank gathers the slices) — deterministic, identical on all ranks
//
// A rank's shard of an embedding table may live in mapped, page-locked host memory (WdPlanDesc::table_placement).  The owner then
// moves exactly one record per unique owned host row each way per train step (inward only for a forward):
//   1. group        after barrier A, on the main stream: flatten + group the received rows (list 2) — the grouping the backward
//                   needs anyway, moved in front of the serve
//   2. stage-in     host_rows_kernel<true> (host_tables.cu): record of unique row u of a host slot -> owner staging buffer row u
//   3. serve        a host slot's records are read from staging row u (lower_bound of the local row in urow[2])
//   4. apply        emb_apply_kernel updates the staged record of u (RowRecords with a per-slot stage stride; 0 = HBM slot,
//                   updated in place)
//   5. write-back   host_rows_kernel<false>, right after the apply on the same stream, which joins the main stream before the step
//                   ends (before the next stage-in); forward-only calls skip it
// Every kernel reads the same values and sums them in the same order as with the shard in HBM: the results are bit-identical.
//
// One function, shard_step, issues a rank's step; it is cut into segments at the barriers that close them.  Ranks of a
// multi-process job run it whole and synchronise with flag barriers in peer memory (st.release.sys / ld.acquire.sys).  When all
// ranks live in ONE process (tests on a single GPU), barriers issue nothing and the caller runs the step segment by segment on
// every rank, with wd_shard_local_sync standing in for the barriers between segments (wd_shard_phase).
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "sparse_dev.cuh"

namespace wd {

constexpr uint32_t kTagBagBits = 27;
constexpr uint32_t kTagBagMask = (1u << kTagBagBits) - 1;
enum { BAR_A = 0, BAR_B = 1, BAR_CW = 2, BAR_CE = 3, BAR_G = 4, BAR_R = 5, BAR_END = 6 };

// ------------------------------------------------------------------------------------------------- flag barrier
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long gtimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// One warp: lane r signals rank r ("rank `me` reached barrier k for the e-th time") and waits for rank r's signal.  The epoch
// lives in device memory so the kernel can be replayed from a CUDA graph.  A rank that never arrives trips a 20 s timeout that
// raises an error flag instead of hanging the device.
// `trace` (optional): [kBarriers][2] globaltimer stamps {barrier entered, barrier left} of the last step (wd_debug_shard_trace).
__global__ void shard_barrier_kernel(uint32_t* const* __restrict__ peer_flags, uint32_t* __restrict__ my_flags, uint32_t* __restrict__ epoch,
                                     int k, int G, int me, int32_t* __restrict__ err, unsigned long long* __restrict__ trace) {
    __shared__ uint32_t e_sh;
    if (threadIdx.x == 0) { e_sh = epoch[k] + 1u; epoch[k] = e_sh; if (trace) trace[2 * k] = gtimer_ns(); }
    __syncthreads();
    const uint32_t e = e_sh;
    const int r = threadIdx.x;
    if (r < G) {
        __threadfence_system();                                   // everything this device wrote before (peer stores included)
        st_release_sys(peer_flags[r] + k * kMaxRanks + me, e);
        const unsigned long long t0 = gtimer_ns();
        while ((int32_t)(ld_acquire_sys(my_flags + k * kMaxRanks + r) - e) < 0) {
            __nanosleep(100);
            if (gtimer_ns() - t0 > 20000000000ull) { atomicOr(err, 4); break; }
        }
    }
    __threadfence_system();
    __syncwarp();
    if (threadIdx.x == 0 && trace) trace[2 * k + 1] = gtimer_ns();
}

__global__ void shard_stamp_kernel(unsigned long long* __restrict__ t) { *t = gtimer_ns(); }

// --------------------------------------------------------------------------------------------- requester: route + send
// starts[o] = first position of owner o in the owner-sorted key list (keys >= G are "not a sharded column"), o = 0 .. G
__global__ void shard_starts_kernel(const int32_t* __restrict__ d_n, const uint32_t* __restrict__ keys, int G, int32_t* __restrict__ ostart) {
    const int o = threadIdx.x;
    if (o <= G) ostart[o] = lower_bound_u32(keys, *d_n, (uint32_t)o);
}

template <bool EMB>
__device__ __forceinline__ int shard_bag(int bc, int C, int n_slots, const int32_t* __restrict__ col_slot) {
    const int b = bc / C;
    return EMB ? b * n_slots + col_slot[bc - b * C] : b;
}

template <bool EMB>
__global__ void __launch_bounds__(256) shard_send_kernel(const int32_t* __restrict__ ostart, const uint32_t* __restrict__ sk, const uint32_t* __restrict__ sv,
                                                         const uint32_t* __restrict__ lrow, const int32_t* __restrict__ e_bc,
                                                         const int32_t* __restrict__ offs, int C, int n_slots, const int32_t* __restrict__ col_slot,
                                                         const ShardPeer* __restrict__ peers, int G, int me, int64_t pair_cap,
                                                         int32_t* __restrict__ bagmask, float* __restrict__ bagscale, int32_t* __restrict__ err) {
    const int total = ostart[G];
    if (blockIdx.x == 0 && threadIdx.x < G) {
        const int o = threadIdx.x;
        int c = ostart[o + 1] - ostart[o];
        if ((int64_t)c > pair_cap) { c = (int)pair_cap; atomicOr(err, 2); }
        peers[o].inbox_cnt[me] = c;
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
        const int o = (int)sk[p];
        const int e = (int)sv[p];
        const int i = p - ostart[o];
        if ((int64_t)i >= pair_cap) continue;
        const int bc = e_bc[e];
        const int bag = shard_bag<EMB>(bc, C, n_slots, col_slot);
        peers[o].inbox[(int64_t)me * pair_cap + i] = make_uint2(lrow[e], (uint32_t)bag);
        const bool head = i == 0 || shard_bag<EMB>(e_bc[sv[p - 1]], C, n_slots, col_slot) != bag;
        if (head) {
            atomicOr(&bagmask[bag], 1 << o);
            if (EMB) bagscale[bag] = 1.f / (float)(offs[bc + 1] - offs[bc]);      // combiner = mean (same value from every owner's head)
        }
    }
}

// ------------------------------------------------------------------------------------------------------- owner: serve
// flat index f over the received entries of all sources -> (source rank r, position i)
__device__ __forceinline__ bool shard_locate(int64_t f, const int32_t* __restrict__ cnt, int G, int& r, int& i) {
    for (r = 0; r < G; ++r) {
        const int c = __ldcg(cnt + r);
        if (f < c) { i = (int)f; return true; }
        f -= c;
    }
    return false;
}

// embedding space: 8 lanes per received entry; the lanes of a bag's first entry pool the whole run and store the partial sum.
// slot_stage (null: every shard in HBM): a host slot's records are read from the owner staging buffer, at uslot[u] (the owner's
// cache) or row u without a cache, u = position of the local row in the step's unique owned rows urow[0 .. *d_nuniq) (list 2,
// sorted ascending).  (Entries beyond the max_nnz the grouping keeps — flagged as truncated — find u <= max_nnz: the staging
// buffer has one spare overflow row and uslot one spare entry.)
__global__ void __launch_bounds__(256) shard_serve_emb_kernel(const uint2* __restrict__ inbox, const int32_t* __restrict__ cnt, int G, int me,
                                                              int64_t pair_cap, int n_slots, const int64_t* __restrict__ slot_base,
                                                              float* const* __restrict__ slot_data, const int32_t* __restrict__ slot_dim,
                                                              const int32_t* __restrict__ slot_stride, const ShardPeer* __restrict__ peers,
                                                              int64_t nbags_cap, int width, const int32_t* __restrict__ slot_stage,
                                                              const float* __restrict__ stage, const uint32_t* __restrict__ urow,
                                                              const int32_t* __restrict__ d_nuniq, const int32_t* __restrict__ uslot) {
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    int64_t total = 0;
    for (int r = 0; r < G; ++r) total += __ldcg(cnt + r);
    const int64_t g0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4 + grp;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    for (int64_t f = g0; f < total; f += gstep) {
        int r, i;
        if (!shard_locate(f, cnt, G, r, i)) break;
        const uint2* box = inbox + (int64_t)r * pair_cap;
        const uint2 en = __ldcg(box + i);
        if (i > 0 && __ldcg(box + i - 1).y == en.y) continue;     // not the head of its bag
        const int lo = table_of(slot_base, n_slots, en.x);
        const int sst = slot_stage ? slot_stage[lo] : 0;
        const int dim = slot_dim[lo], stride = sst ? sst : slot_stride[lo];
        const float* data = sst ? stage : slot_data[lo];
        const int64_t base = slot_base[lo];
        const int nu = sst ? *d_nuniq : 0;
        auto rec = [&](uint32_t lrow) -> int64_t {
            if (!sst) return (int64_t)lrow - base;
            const int u = lower_bound_u32(urow, nu, lrow);
            return uslot ? (int64_t)__ldg(uslot + u) : (int64_t)u;
        };
        const int n = __ldcg(cnt + r);
        float* dst = peers[r].recv + ((int64_t)me * nbags_cap + en.y) * width;
        for (int q = lig; q * 4 < dim; q += 8) {
            float4 acc = ldg_nc_f4(data + rec(en.x) * stride + q * 4);
            for (int j = i + 1; j < n; ++j) {
                const uint2 e2 = __ldcg(box + j);
                if (e2.y != en.y) break;
                const float4 v = ldg_nc_f4(data + rec(e2.x) * stride + q * 4);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            *reinterpret_cast<float4*>(dst + q * 4) = acc;
        }
    }
}

// wide space: thread per received entry; partial logit of the example = sum of the weights of its run
__global__ void __launch_bounds__(256) shard_serve_wide_kernel(const uint2* __restrict__ inbox, const int32_t* __restrict__ cnt, int G, int me,
                                                               int64_t pair_cap, const float4* __restrict__ wide, const ShardPeer* __restrict__ peers,
                                                               int64_t nbags_cap) {
    int64_t total = 0;
    for (int r = 0; r < G; ++r) total += __ldcg(cnt + r);
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += (int64_t)gridDim.x * blockDim.x) {
        int r, i;
        if (!shard_locate(f, cnt, G, r, i)) break;
        const uint2* box = inbox + (int64_t)r * pair_cap;
        const uint2 en = __ldcg(box + i);
        if (i > 0 && __ldcg(box + i - 1).y == en.y) continue;
        const int n = __ldcg(cnt + r);
        float acc = __ldg(&wide[en.x].x);
        for (int j = i + 1; j < n; ++j) {
            const uint2 e2 = __ldcg(box + j);
            if (e2.y != en.y) break;
            acc += __ldg(&wide[e2.x].x);
        }
        peers[r].recv[(int64_t)me * nbags_cap + en.y] = acc;
    }
}

// received entries of all sources, flattened in (source rank, position) order = global (example, column, id) order of the
// concatenated batch, so the per-row gradient sums run in the order a single rank would use
__global__ void __launch_bounds__(256) shard_flatten_kernel(const uint2* __restrict__ inbox, const int32_t* __restrict__ cnt, int G, int64_t pair_cap,
                                                            uint32_t* __restrict__ rrow, uint32_t* __restrict__ rtag, int32_t* __restrict__ d_nrecv,
                                                            int64_t cap, int32_t* __restrict__ err) {
    int64_t total = 0;
    for (int r = 0; r < G; ++r) total += __ldcg(cnt + r);
    if (total > cap) {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(err, 2);
        total = cap;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *d_nrecv = (int)total;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += (int64_t)gridDim.x * blockDim.x) {
        int r, i;
        if (!shard_locate(f, cnt, G, r, i)) break;
        const uint2 en = __ldcg(inbox + (int64_t)r * pair_cap + i);
        rrow[f] = en.x;
        rtag[f] = ((uint32_t)r << kTagBagBits) | (en.y & kTagBagMask);
    }
}

// --------------------------------------------------------------------------------------------------- requester: combine
__global__ void __launch_bounds__(256) shard_combine_emb_kernel(int B, int n_slots, const int32_t* __restrict__ slot_dim, const int32_t* __restrict__ slot_x0,
                                                                const int32_t* __restrict__ bagmask, const float* __restrict__ bagscale,
                                                                const float* __restrict__ recv, int G, int64_t nbags_cap, int width,
                                                                float* __restrict__ X0, int ld) {
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int64_t nb = (int64_t)B * n_slots;
    const int64_t g0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4 + grp;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    for (int64_t bag = g0; bag < nb; bag += gstep) {
        const int b = (int)(bag / n_slots), slot = (int)(bag - (int64_t)b * n_slots);
        const int mask = bagmask[bag];
        const float scale = mask ? bagscale[bag] : 0.f;
        const int dim = slot_dim[slot];
        for (int q = lig; q * 4 < dim; q += 8) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int o = 0; o < G; ++o)
                if (mask >> o & 1) {
                    const float4 v = __ldcg(reinterpret_cast<const float4*>(recv + ((int64_t)o * nbags_cap + bag) * width + q * 4));
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                }
            acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
            *reinterpret_cast<float4*>(X0 + (int64_t)b * ld + slot_x0[slot] + q * 4) = acc;
        }
    }
}
__global__ void __launch_bounds__(256) shard_combine_wide_kernel(int B, const int32_t* __restrict__ bagmask, const float* __restrict__ recv, int G,
                                                                 int64_t nbags_cap, float* __restrict__ wide_logit) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
        const int mask = bagmask[b];
        float acc = 0.f;
        for (int o = 0; o < G; ++o)
            if (mask >> o & 1) acc += __ldcg(recv + (int64_t)o * nbags_cap + b);
        wide_logit[b] += acc;
    }
}

// -------------------------------------------------------------------------------------- owner: gradient sums (P2P pull)
// Occurrence sources of the owner's per-row gradient sums (emb_grad_sum_kernel / wide_grad_sum_kernel, sparse_dev.cuh): occurrence
// j of the sorted received rows is the received entry svals[j], whose tag (source rank << kTagBagBits | bag) says where its
// gradient is — read from the requester's memory.
// embedding space: (requester's dX0 slice of the bag) / (ids in the bag); a bag is example * n_slots + slot
// (the tags, lists and peer table are read-only during the sums: loaded through the read-only path; the peers' gradients with
// ld.global.cg, they live in another device's memory)
__device__ __forceinline__ const ShardPeer& peer_of(const ShardPeer* peers, uint32_t tg) { return peers[tg >> kTagBagBits]; }
__device__ __forceinline__ const float* ldg_ptr(const float* const* p) {
    return reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(p)));
}
struct PeerEmb {
    const uint32_t* svals;
    const uint32_t* rtag;
    const ShardPeer* peers;
    int n_slots;
    const int32_t* slot_dim;
    const int32_t* slot_x0;
    int ld;
    __device__ __forceinline__ uint32_t key(int j) const { return __ldg(rtag + __ldg(svals + j)); }
    __device__ __forceinline__ void layout(uint32_t tg, int& t, int& dim, int& x0) const {
        t = (int)((tg & kTagBagMask) % (uint32_t)n_slots);
        dim = __ldg(slot_dim + t); x0 = __ldg(slot_x0 + t);
    }
    __device__ __forceinline__ float4 row(uint32_t tg, int x0, int q, float& inv) const {
        const ShardPeer& pr = peer_of(peers, tg);
        const uint32_t bag = tg & kTagBagMask;
        const float4 v = __ldcg(reinterpret_cast<const float4*>(ldg_ptr(&pr.gradbase) + (int64_t)(bag / (uint32_t)n_slots) * ld + x0 + q * 4));
        inv = __ldcg(ldg_ptr(&pr.bagscale) + bag);
        return v;
    }
};
// wide space: the example's dlogit on its own rank
struct PeerWide {
    const uint32_t* svals;
    const uint32_t* rtag;
    const ShardPeer* peers;
    __device__ __forceinline__ uint32_t key(int j) const { return __ldg(rtag + __ldg(svals + j)); }
    __device__ __forceinline__ float row(uint32_t tg) const { return __ldcg(ldg_ptr(&peer_of(peers, tg).gradbase) + (tg & kTagBagMask)); }
};

// ----------------------------------------------------------------------------------------- dense gradients: all-reduce
// two-shot over peer memory: rank `me` sums slice `me` of every rank's arena in rank order, then every rank copies all slices
__global__ void __launch_bounds__(256) shard_ar_reduce_kernel(float* const* __restrict__ peer_G, float* __restrict__ gred, int64_t n4, int64_t slice4,
                                                              int G, int me) {
    const int64_t lo = (int64_t)me * slice4, hi = min(n4, lo + slice4);
    for (int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (int64_t)gridDim.x * blockDim.x) {
        // every rank's value in flight before the first add (a peer load is ~2 us: one round trip instead of G), summed in rank order
        float4 v[kMaxRanks];
#pragma unroll
        for (int r = 0; r < kMaxRanks; ++r)
            v[r] = r < G ? __ldcg(reinterpret_cast<const float4*>(peer_G[r]) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 acc = v[0];
#pragma unroll
        for (int r = 1; r < kMaxRanks; ++r)
            if (r < G) { acc.x += v[r].x; acc.y += v[r].y; acc.z += v[r].z; acc.w += v[r].w; }
        reinterpret_cast<float4*>(gred)[i] = acc;
    }
}
__global__ void __launch_bounds__(256) shard_ar_gather_kernel(float* const* __restrict__ peer_gred, float* __restrict__ Gout, int64_t n4, int64_t slice4) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const int owner = (int)(i / slice4);
        reinterpret_cast<float4*>(Gout)[i] = __ldcg(reinterpret_cast<const float4*>(peer_gred[owner]) + i);
    }
}

// ------------------------------------------------------------------------------------------- eval metrics: reduction
// every rank's metric accumulator (in its exchange segment) summed in rank order: the same doubles, bit for bit, on every rank
struct PeerMetrics { const double* acc[kMaxRanks]; };
__global__ void __launch_bounds__(256) shard_metrics_reduce_kernel(PeerMetrics peers, int G, double* __restrict__ out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kMetricsDoubles; i += gridDim.x * blockDim.x) {
        double s = __ldcg(peers.acc[0] + i);
        for (int r = 1; r < G; ++r) s += __ldcg(peers.acc[r] + i);
        out[i] = s;
    }
}

// ================================================================================================== host side
static int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// Lays out the sharded spaces and the exchange segment and allocates their scratch and lists 2 - 5.  Called by build_model (world
// > 1) before the embedding tables are placed, so that their auto placement finds this HBM taken: by then the dense arena size is
// known; d_dX0 / d_dlogit / d_G live INSIDE the segment so that peers can read them.  The sharded tables' row bases move into the
// shard's row space here; the shard set that describes them is uploaded after (build_record_sets).  The owner staging buffer of
// host-placed shards is place_tables' (which shards go to the host is known there).
int shard_build(WdModel* m, const WdPlanDesc* d) {
    ShardState& S = m->shard;
    S.world = d->shard_world; S.rank = d->shard_rank;
    const int G = S.world, C = m->n_columns;
    if (G > kMaxRanks) { set_error("shard_world %d > %d", G, kMaxRanks); return WD_EUNSUPPORTED; }
    int rc;
    const int64_t route_cap = m->max_nnz;                                  // ids one rank can route per step and space
    // ---- embedding space
    {
        ShardSpace& sp = S.sp[0];
        std::vector<int32_t> col_slot(C, -1);
        std::vector<int64_t> base;
        int64_t rows = 0;
        for (EmbTable& tb : m->tables) {
            if (!tb.sharded) continue;
            col_slot[tb.col] = sp.n_slots++;
            base.push_back(rows);
            tb.row_base = rows;
            rows += (tb.rows + G - 1) / G;            // the SAME layout on every rank (a requester computes the owner's local row): ceil(rows / G) per table
            sp.width = std::max(sp.width, tb.dim);
        }
        sp.on = sp.n_slots > 0;
        sp.local_rows = rows;
        sp.bags_per_row = sp.n_slots;
        sp.h_col_slot = col_slot; sp.h_slot_base = base;
        if (sp.on && (rc = upload(m, &sp.d_col_slot, col_slot))) return rc;
    }
    // ---- wide space
    {
        ShardSpace& sp = S.sp[1];
        std::vector<int32_t> col_slot(C, -1);
        std::vector<int64_t> base;
        int64_t rows = 0;
        if (m->use_wide && d->col_wide_sharded)
            for (int c = 0; c < C; ++c)
                if (d->col_wide_sharded[c]) {
                    col_slot[c] = sp.n_slots++;
                    base.push_back(rows);
                    rows += (d->col_buckets[c] + G - 1) / G;     // rank-independent layout: ceil(buckets / G) rows per column
                }
        sp.h_col_slot = col_slot; sp.h_slot_base = base;
        sp.on = sp.n_slots > 0;
        sp.local_rows = rows;
        sp.width = 1;
        sp.bags_per_row = 1;
        if (sp.on) {
            if ((rc = upload(m, &sp.d_col_slot, col_slot))) return rc;
            if ((rc = dev_alloc(m, &sp.d_wide, rows))) return rc;
        }
    }
    for (int s = 0; s < 2; ++s)
        if (S.sp[s].on && (s == 0 ? m->dnn_opt : m->lin_opt).kind == WD_OPT_ADAM &&
            (rc = dev_alloc(m, &S.sp[s].d_adam_touched, (S.sp[s].local_rows + 31) / 32))) return rc;
    for (int s = 0; s < 2; ++s)
        if (S.sp[s].local_rows >= (1ll << 30)) { set_error("more than 2^30 sharded rows per rank in one table space"); return WD_EUNSUPPORTED; }
    // ---- per-space scratch (requester + owner) and the sort lists 2 + s (owned rows) / 4 + s (routing)
    for (int s = 0; s < 2; ++s) {
        ShardSpace& sp = S.sp[s];
        if (!sp.on) continue;
        sp.nbags_cap = (int64_t)m->max_batch * sp.bags_per_row;
        if (sp.nbags_cap > (int64_t)kTagBagMask) { set_error("too many sharded bags per step for the tag encoding"); return WD_EUNSUPPORTED; }
        sp.pair_cap = route_cap;
        if ((rc = dev_alloc(m, &sp.d_own, m->max_nnz + 8))) return rc;
        if ((rc = dev_alloc(m, &sp.d_lrow, m->max_nnz + 8))) return rc;
        if ((rc = dev_alloc(m, &sp.d_ostart, kMaxRanks + 2))) return rc;
        if ((rc = dev_alloc(m, &sp.d_bagmask, sp.nbags_cap + 8))) return rc;
        if ((rc = dev_alloc(m, &sp.d_rtag, m->max_nnz + 8))) return rc;
        if ((rc = dev_alloc(m, &sp.d_rrow, m->max_nnz + 8))) return rc;
        if ((rc = dev_alloc(m, &sp.d_nrecv, 4))) return rc;
        if ((rc = dev_alloc(m, &sp.d_peers, kMaxRanks))) return rc;
        if ((rc = list_alloc(m, 2 + s, sp.local_rows, sp.width, false))) return rc;     // owned rows, in the shard's row space
        if ((rc = list_alloc(m, 4 + s, G, 1, true))) return rc;                         // routing: keys are owner ranks
    }
    // ---- exchange segment layout (identical on every rank)
    int64_t off = 0;
    auto take = [&](int64_t bytes) { int64_t o = off; off = align_up(off + bytes, 256); return o; };
    S.off_flags = take((int64_t)kBarriers * kMaxRanks * 4);
    for (int s = 0; s < 2; ++s) {
        ShardSpace& sp = S.sp[s];
        if (!sp.on) continue;
        sp.off_inbox = take((int64_t)G * sp.pair_cap * (int64_t)sizeof(uint2));   // reused every step: see the hazard note at shard_step
        sp.off_cnt = take(kMaxRanks * 4);
        sp.off_recv = take((int64_t)G * sp.nbags_cap * sp.width * 4);
        sp.off_bagscale = take(sp.nbags_cap * 4);
    }
    const int64_t x0n = m->use_deep ? (int64_t)m->max_batch_pad * std::max(m->d0_phys, 1) : 4;
    S.sp[0].off_grad = take(x0n * 4);                                      // dX0
    S.sp[1].off_grad = take((int64_t)m->max_batch * 4 + 64);               // dlogit
    S.ar_count = align_up(m->dense_count + m->gs_count, 4);
    S.off_G = take(std::max<int64_t>(S.ar_count, 4) * 4);
    S.off_gred = take(std::max<int64_t>(S.ar_count, 4) * 4);
    S.off_metrics = take(kMetricsDoubles * 8);
    S.seg_bytes = off;
    if ((rc = dev_alloc(m, &S.seg, S.seg_bytes))) return rc;
    m->d_dX0 = reinterpret_cast<float*>(S.seg + S.sp[0].off_grad);
    m->d_dlogit = reinterpret_cast<float*>(S.seg + S.sp[1].off_grad);
    m->d_G = reinterpret_cast<float*>(S.seg + S.off_G);
    S.gred = reinterpret_cast<float*>(S.seg + S.off_gred);
    m->d_metrics = reinterpret_cast<double*>(S.seg + S.off_metrics);      // peers read it in wd_shard_eval_finish
    if ((rc = dev_alloc(m, &S.d_msum, kMetricsDoubles))) return rc;
    if ((rc = dev_alloc(m, &S.d_peer_flags, kMaxRanks))) return rc;
    if ((rc = dev_alloc(m, &S.d_epoch, kBarriers))) return rc;
    if (getenv("WD_SHARD_TRACE") && (rc = dev_alloc(m, &S.d_trace, 2 * kBarriers))) return rc;
    if ((rc = dev_alloc(m, &S.d_peer_G, kMaxRanks))) return rc;
    if ((rc = dev_alloc(m, &S.d_peer_gred, kMaxRanks))) return rc;
    for (cudaEvent_t* ev : {&S.ev_a, &S.ev_ids2, &S.ev_routed1, &S.ev_a2, &S.ev_aux_done}) WD_CUDA(new_event(m, ev, cudaEventDisableTiming));
    WD_CUDA(new_stream(m, &S.aux));
    return WD_OK;
}

// peer segment bases known: fill the per-peer pointer tables
static int shard_finish_connect(WdModel* m) {
    ShardState& S = m->shard;
    const int G = S.world;
    std::vector<uint32_t*> pf(kMaxRanks, nullptr);
    std::vector<float*> pg(kMaxRanks, nullptr), pr(kMaxRanks, nullptr);
    for (int r = 0; r < G; ++r) {
        uint8_t* b = S.peer_seg[r];
        pf[r] = reinterpret_cast<uint32_t*>(b + S.off_flags);
        pg[r] = reinterpret_cast<float*>(b + S.off_G);
        pr[r] = reinterpret_cast<float*>(b + S.off_gred);
        for (int s = 0; s < 2; ++s) {
            ShardSpace& sp = S.sp[s];
            if (!sp.on) continue;
            ShardPeer& p = sp.peers[r];
            p.inbox = reinterpret_cast<uint2*>(b + sp.off_inbox);
            p.inbox_cnt = reinterpret_cast<int32_t*>(b + sp.off_cnt);
            p.recv = reinterpret_cast<float*>(b + sp.off_recv);
            p.bagscale = reinterpret_cast<const float*>(b + sp.off_bagscale);
            p.gradbase = reinterpret_cast<const float*>(b + sp.off_grad);
        }
    }
    WD_CUDA(cudaMemcpyAsync(S.d_peer_flags, pf.data(), kMaxRanks * sizeof(void*), cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaMemcpyAsync(S.d_peer_G, pg.data(), kMaxRanks * sizeof(void*), cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaMemcpyAsync(S.d_peer_gred, pr.data(), kMaxRanks * sizeof(void*), cudaMemcpyHostToDevice, m->stream));
    for (int s = 0; s < 2; ++s)
        if (S.sp[s].on) WD_CUDA(cudaMemcpyAsync(S.sp[s].d_peers, S.sp[s].peers, sizeof(ShardPeer) * kMaxRanks, cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    S.connected = true;
    return WD_OK;
}

static int barrier(WdModel* m, int k) {
    ShardState& S = m->shard;
    if (!S.ipc) return WD_OK;                                  // ranks of one process: the caller orders the segments with events
    shard_barrier_kernel<<<1, 32, 0, m->stream>>>(S.d_peer_flags, reinterpret_cast<uint32_t*>(S.seg + S.off_flags), S.d_epoch, k, S.world, S.rank,
                                                  m->d_flags, S.d_trace);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---- requester: group the step's sharded ids by owner and store them into the owners' inboxes
static int shard_route_send(WdModel* m, int s) {
    ShardState& S = m->shard;
    ShardSpace& sp = S.sp[s];
    if (!sp.on) return WD_OK;
    const int G = S.world;
    RowList& l = m->lists[4 + s];
    int rc;
    WD_CUDA(cudaMemsetAsync(sp.d_bagmask, 0, (size_t)(m->dbatch.B * (int64_t)sp.bags_per_row) * 4, m->stream));
    // keys = owner (or "not sharded" = 1 << bits, sorts last), values = entry index; one stable radix pass
    if ((rc = list_sort_by_key(m, l, m->d_nnz, sp.d_own))) return rc;
    shard_starts_kernel<<<1, 32, 0, m->stream>>>(m->d_nnz, l.keys, G, sp.d_ostart);
    float* bagscale = const_cast<float*>(sp.peers[S.rank].bagscale);
    const int g = grid_for(m->max_nnz, 256);
    if (s == 0)
        shard_send_kernel<true><<<g, 256, 0, m->stream>>>(sp.d_ostart, l.keys, l.vals, sp.d_lrow, m->d_e_bc, m->d_col_offs, m->n_columns,
            sp.n_slots, sp.d_col_slot, sp.d_peers, G, S.rank, sp.pair_cap, sp.d_bagmask, bagscale, m->d_flags);
    else
        shard_send_kernel<false><<<g, 256, 0, m->stream>>>(sp.d_ostart, l.keys, l.vals, sp.d_lrow, m->d_e_bc, m->d_col_offs, m->n_columns,
            sp.n_slots, sp.d_col_slot, sp.d_peers, G, S.rank, sp.pair_cap, sp.d_bagmask, bagscale, m->d_flags);
    m->launches += 2;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

static int shard_owner_group(WdModel* m, int s);

// a space whose owner stages host-placed shards groups its received rows before serving them (the serve reads the staged records)
static bool staged(const WdModel* m, int s) { return m->shard.sp[s].stage_stride > 0; }
static const CacheMarks kShardMarks{"shard_cache_sort", "shard_cache_assign", "shard_stage_in", "shard_write_back"};

// ---- owner: pooled partial sums of the received bags -> requesters' receive buffers
static int shard_serve(WdModel* m, int s, bool train) {
    ShardState& S = m->shard;
    ShardSpace& sp = S.sp[s];
    if (!sp.on) return WD_OK;
    const ShardPeer& me = sp.peers[S.rank];
    int rc;
    if (staged(m, s)) {                          // unique owned rows (list 2), then the records of the host rows among them -> HBM
        if ((rc = shard_owner_group(m, s))) return rc;
        if ((rc = stage_in_rows(m, sp.cache, 2, sp.set.rec, sp.stage_stride, train, kShardMarks))) return rc;
    }
    if (s == 0)
        shard_serve_emb_kernel<<<grid_for(m->max_nnz * 8, 256, kNumSms * 8), 256, 0, m->stream>>>(me.inbox, me.inbox_cnt, S.world, S.rank, sp.pair_cap,
            sp.n_slots, sp.set.rec.row_base, sp.set.rec.data, sp.set.rec.dim, sp.set.rec.stride, sp.d_peers, sp.nbags_cap, sp.width,
            sp.set.rec.stage, sp.d_stage, m->lists[2].urow, m->lists[2].nuniq, sp.cache.d_uslot);
    else
        shard_serve_wide_kernel<<<grid_for(m->max_nnz, 256, kNumSms * 8), 256, 0, m->stream>>>(me.inbox, me.inbox_cnt, S.world, S.rank, sp.pair_cap,
            sp.d_wide, sp.d_peers, sp.nbags_cap);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---- owner: sort the received rows (depends only on ids: runs beside the towers)
static int shard_owner_group(WdModel* m, int s) {
    ShardState& S = m->shard;
    ShardSpace& sp = S.sp[s];
    if (!sp.on) return WD_OK;
    const ShardPeer& me = sp.peers[S.rank];
    shard_flatten_kernel<<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(me.inbox, me.inbox_cnt, S.world, sp.pair_cap, sp.d_rrow, sp.d_rtag,
                                                                            sp.d_nrecv, m->max_nnz, m->d_flags);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return list_group(m, m->lists[2 + s], sp.d_nrecv, sp.d_rrow);
}

static int shard_combine(WdModel* m, int s) {
    ShardState& S = m->shard;
    ShardSpace& sp = S.sp[s];
    if (!sp.on) return WD_OK;
    const int B = m->dbatch.B;
    const ShardPeer& me = sp.peers[S.rank];
    if (s == 0)
        shard_combine_emb_kernel<<<grid_for((int64_t)B * sp.n_slots * 8, 256, kNumSms * 8), 256, 0, m->stream>>>(B, sp.n_slots, sp.set.rec.dim, sp.set.x0,
            sp.d_bagmask, me.bagscale, me.recv, S.world, sp.nbags_cap, sp.width, m->d_X0, m->d0_phys);
    else
        shard_combine_wide_kernel<<<grid_for(B, 256), 256, 0, m->stream>>>(B, sp.d_bagmask, me.recv, S.world, sp.nbags_cap, m->d_wide_logit);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---- owner: per-row gradient sums (pulled from the requesters) + optimizer on the shard
static int shard_owner_reduce_apply(WdModel* m, int s) {
    ShardState& S = m->shard;
    ShardSpace& sp = S.sp[s];
    if (!sp.on) return WD_OK;
    const int L = 2 + s;
    const RowList& l = m->lists[L];
    const int64_t ncap = m->max_nnz + chunk_cap(m->max_nnz);     // unique rows + hot-row chunks
    int rc;
    if (s == 0) {
        const PeerEmb src{l.vals, sp.d_rtag, sp.d_peers, sp.n_slots, sp.set.rec.dim, sp.set.x0, m->d0_phys};
        emb_grad_sum_kernel<PeerEmb, false><<<grid_for(ncap * 8, 256), 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad,
                                                                                            l.cpart, l.width, RowApply{});
        m->launches++;
        if ((rc = list_chunk_combine(m, l))) return rc;
        const OptParams o = space_opt(m, 0, sp.d_adam_touched);
        if ((rc = list_apply_emb(m, l, sp.set.rec, o))) return rc;
        // Adam: the shard's rows no rank touched, after its touched ones (host-placed shards with Adam are deferred: their rows
        // are 0 here, their staged records were caught up by the serve's stage-in)
        if ((rc = adam_untouched_emb(m, sp.set, sp.local_rows, o))) return rc;
        // staged records home (overflow rows only with a cache), on this stream: it joins the main stream before the step ends, so
        // the next stage-in comes after
        if (staged(m, s) && (rc = write_back_rows(m, sp.cache, L, sp.set.rec, sp.stage_stride, kShardMarks))) return rc;
    } else {
        const PeerWide src{l.vals, sp.d_rtag, sp.d_peers};
        wide_grad_sum_kernel<PeerWide, false><<<grid_for(ncap, 256), 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad, l.cpart,
                                                                                          RowApply{});
        m->launches++;
        if ((rc = list_chunk_combine(m, l))) return rc;
        const OptParams o = space_opt(m, 1, sp.d_adam_touched);
        if ((rc = list_apply_wide(m, l, sp.d_wide, o))) return rc;
        if ((rc = adam_untouched_wide(m, sp.d_wide, sp.local_rows, o))) return rc;
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

static int shard_ar_reduce(WdModel* m) {
    ShardState& S = m->shard;
    if (S.ar_count == 0) return WD_OK;
    const int64_t n4 = S.ar_count / 4, slice4 = (n4 + S.world - 1) / S.world;
    shard_ar_reduce_kernel<<<grid_for(slice4, 256), 256, 0, m->stream>>>(S.d_peer_G, S.gred, n4, slice4, S.world, S.rank);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
static int shard_ar_gather(WdModel* m) {
    ShardState& S = m->shard;
    if (S.ar_count == 0) return WD_OK;
    const int64_t n4 = S.ar_count / 4, slice4 = (n4 + S.world - 1) / S.world;
    shard_ar_gather_kernel<<<grid_for(n4, 256), 256, 0, m->stream>>>(S.d_peer_gred, m->d_G, n4, slice4);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ---------------------------------------------------------------------------------------------------------- the step
int sparse_forward(WdModel* m);
int mlp_forward(WdModel* m, bool train);
int loss_forward(WdModel* m, bool need_grad);
int ids_prepare(WdModel* m);
int group_async(WdModel* m);        // api.cu: replicated lists' grouping on the side streams
int backward_core(WdModel* m);      // api.cu: towers' backward + replicated lists + dense gradient arena
int apply_core(WdModel* m);         // api.cu: dense optimizer + small-table block + joins

// The critical chain in front of the towers is   ids -> route + send (embedding space) -> [A] -> serve (embedding space) -> [B].
// Everything else that must exist before the towers — the wide space's routing, its serve, and this rank's local gathers
// (replicated tables, wide bias) — is independent of that chain, so it runs beside it on an auxiliary stream: routing right after
// the ids, serving + local gathers once barrier A has passed, joined before barrier B.  (The two side streams cannot take it: they
// already hold the grouping of the replicated lists, ~100 us of sort launches enqueued before barrier A.)
static bool aux_split(WdModel* m) { return m->shard.sp[0].on && m->shard.sp[1].on; }

// after barrier A: serve both spaces and run the local part of the forward (needed only by this rank's towers, while every peer's
// barrier B waits for the serves)
// (The embedding space's stage-in sorts its cache keys on the main stream while the aux stream and the side streams may be sorting
// too: every stream has its own scan / sort scratch, on_stream.)
static int shard_serve_both(WdModel* m, bool train) {
    ShardState& S = m->shard;
    int rc;
    if (aux_split(m)) {
        WD_CUDA(cudaEventRecord(S.ev_a2, m->stream));
        WD_CUDA(cudaStreamWaitEvent(S.aux, S.ev_a2, 0));
        if ((rc = on_aux(m, [&] { int r = shard_serve(m, 1, train); return r ? r : sparse_forward(m); }))) return rc;
        WD_CUDA(cudaEventRecord(S.ev_aux_done, S.aux));
        if ((rc = shard_serve(m, 0, train))) return rc;
        WD_CUDA(cudaStreamWaitEvent(m->stream, S.ev_aux_done, 0));
        return WD_OK;
    }
    for (int s = 0; s < 2; ++s) if ((rc = shard_serve(m, s, train))) return rc;
    return sparse_forward(m);
}

// The whole step of one rank.  Main stream: ids, routing, serve, combine, towers, dense all-reduce and optimizers, with flag
// barriers A (ids delivered), B (pooled sums delivered), G (gradient arenas final), R (slices reduced) and END.  Side stream of
// each table space: the owner-side grouping of the received rows (needs only ids: runs beside the towers) and, once every rank's
// dlogit / dX0 exists (barriers Cw / Ce, on the side streams), the owners' pulled gradient sums and optimizer — hidden behind the
// remaining weight gradients, the dense all-reduce and the dense optimizer.
// The step is cut into segments at the barriers that close them: segment `seg` alone, or all of them for seg = kAllSegments.
//   0  ids, routing (+ the replicated lists' grouping)                                      closed by A
//   1  serve both spaces, local gathers (+ owner-side grouping)                              B
//   2  combine, towers forward (+ backward, replicated lists, dense gradient arena)          Cw / Ce / G; a forward: END
//   3  owners' gradient sums and updates, first half of the all-reduce                      R
//   4  second half of the all-reduce, dense optimizers, side streams joined                 END
// A forward is segments 0-2.  Ranks of one process have no flag barriers: their driver runs segment k on every rank, then
// wd_shard_local_sync, which stands in for every barrier that closes the segment.
// Buffer hazards: within a step every producer / consumer pair is separated by one of the barriers; the END barrier keeps a fast
// rank from starting the next step's sends while a slow owner still pulls this step's gradients and bag scales.
int shard_step(WdModel* m, bool train, int seg) {
    ShardState& S = m->shard;
    auto runs = [&](int k) { return seg == kAllSegments || seg == k; };
    int rc;
    if (runs(0)) {
        m->stepped = true;
        if (S.d_trace) { shard_stamp_kernel<<<1, 1, 0, m->stream>>>(S.d_trace + 2 * (kBarriers - 1)); m->launches++; }   // step start
        if ((rc = ids_prepare(m))) return rc;
        const bool split = aux_split(m);
        if (split) {
            WD_CUDA(cudaEventRecord(S.ev_ids2, m->stream));
            WD_CUDA(cudaStreamWaitEvent(S.aux, S.ev_ids2, 0));
            if ((rc = on_aux(m, [&] { return shard_route_send(m, 1); }))) return rc;
            WD_CUDA(cudaEventRecord(S.ev_routed1, S.aux));
        }
        if (train && (rc = group_async(m))) return rc;
        if ((rc = shard_route_send(m, 0))) return rc;
        if (!split && (rc = shard_route_send(m, 1))) return rc;
        if (split) WD_CUDA(cudaStreamWaitEvent(m->stream, S.ev_routed1, 0));
        if ((rc = barrier(m, BAR_A))) return rc;
    }
    if (runs(1)) {
        if ((rc = shard_serve_both(m, train))) return rc;
        if (train) {
            WD_CUDA(cudaEventRecord(S.ev_a, m->stream));
            for (int s = 0; s < 2; ++s) {
                if (!S.sp[s].on || staged(m, s)) continue;         // (a staged space was grouped before its serve)
                if (m->side_pending[s]) {
                    WD_CUDA(cudaStreamWaitEvent(m->sstream[s], S.ev_a, 0));
                    if ((rc = on_side(m, s, [&] { return shard_owner_group(m, s); }))) return rc;
                } else if ((rc = shard_owner_group(m, s))) return rc;
            }
        }
        if ((rc = barrier(m, BAR_B))) return rc;
    }
    if (runs(2)) {
        for (int s = 0; s < 2; ++s) if ((rc = shard_combine(m, s))) return rc;
        if ((rc = mlp_forward(m, train))) return rc;
        if ((rc = loss_forward(m, train))) return rc;
        if (!train) return barrier(m, BAR_END);
        if (m->side_pending[0] || m->side_pending[1]) WD_CUDA(cudaEventRecord(m->ev_head, m->stream));   // dlogit exists (as forward_core does)
        if (m->summary_armed && (rc = summary_launch(m))) return rc;     // layer summaries of this rank's rows
        if ((rc = backward_core(m))) return rc;
    }
    if (!train) return WD_OK;
    if (runs(3)) {
        for (int s = 1; s >= 0; --s) {
            if (!S.sp[s].on) continue;
            auto owner = [&]() -> int { int r = barrier(m, s == 1 ? BAR_CW : BAR_CE); return r ? r : shard_owner_reduce_apply(m, s); };
            if (m->side_active[s]) { if ((rc = on_side(m, s, owner))) return rc; }
            else if ((rc = owner())) return rc;
        }
        if ((rc = barrier(m, BAR_G))) return rc;                // every rank's gradient arena (dense + small-table block) is final
        if ((rc = shard_ar_reduce(m))) return rc;
        if ((rc = barrier(m, BAR_R))) return rc;
    }
    if (runs(4)) {
        if ((rc = shard_ar_gather(m))) return rc;
        if ((rc = apply_core(m))) return rc;
        if (S.d_trace) { shard_stamp_kernel<<<1, 1, 0, m->stream>>>(S.d_trace + 2 * (kBarriers - 1) + 1); m->launches++; }   // before END
        if ((rc = barrier(m, BAR_END))) return rc;
    }
    return WD_OK;
}

// Collective eval finish: every rank's metric accumulator summed in rank order into S.d_msum.  Multi-process ranks meet at a flag
// barrier before the sum (every accumulator final) and after it (no rank resets or adds to its accumulator while a peer still
// reads it); ranks of one process are ordered by the caller (wd_shard_local_sync after the last accumulate).
int shard_metrics_reduce(WdModel* m) {
    ShardState& S = m->shard;
    int rc;
    if ((rc = barrier(m, BAR_END))) return rc;
    PeerMetrics peers{};
    for (int r = 0; r < S.world; ++r) peers.acc[r] = reinterpret_cast<const double*>(S.peer_seg[r] + S.off_metrics);
    shard_metrics_reduce_kernel<<<2, 256, 0, m->stream>>>(peers, S.world, S.d_msum);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return barrier(m, BAR_END);
}

}  // namespace wd

using namespace wd;

// ================================================================================================== C-ABI
extern "C" int wd_shard_info(WdModel* m, int32_t* world, int32_t* rank, int64_t* seg_bytes) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    if (world) *world = m->shard.world;
    if (rank) *rank = m->shard.rank;
    if (seg_bytes) *seg_bytes = m->shard.seg_bytes;
    return WD_OK;
}

// debugging aid (not part of the public header): enter / leave stamps (ns, globaltimer) of the last step's flag barriers, WD_SHARD_TRACE=1
extern "C" int wd_debug_shard_trace(WdModel* m, unsigned long long* out) {
    if (!m || !m->shard.d_trace) return -1;
    cudaDeviceSynchronize();
    return cudaMemcpy(out, m->shard.d_trace, sizeof(unsigned long long) * 2 * kBarriers, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

extern "C" int wd_shard_ipc_handle(WdModel* m, void* handle_out64) {
    if (!m || !handle_out64) { set_error("null argument"); return WD_EINVAL; }
    if (m->shard.world <= 1 || !m->shard.seg) { set_error("model has no sharded tables (shard_world <= 1)"); return WD_ESTATE; }
    WD_CUDA(cudaSetDevice(m->device));
    cudaIpcMemHandle_t h;
    WD_CUDA(cudaIpcGetMemHandle(&h, m->shard.seg));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle_out64, &h, 64);
    return WD_OK;
}

// Maps every peer's exchange segment into this process.  wd_model_destroy closes these mappings and frees this rank's segment,
// which its peers write into: ranks should destroy their models only after their last collective call.
extern "C" int wd_shard_connect_ipc(WdModel* m, const void* handles, int32_t n_ranks) {
    if (!m || !handles) { set_error("null argument"); return WD_EINVAL; }
    ShardState& S = m->shard;
    if (n_ranks != S.world) { set_error("wd_shard_connect_ipc: %d handles for shard_world %d", n_ranks, S.world); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    for (int r = 0; r < S.world; ++r) {
        if (r == S.rank) { S.peer_seg[r] = S.seg; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const uint8_t*)handles + (size_t)r * 64, 64);
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { set_error("cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e)); return WD_ECUDA; }
        S.peer_seg[r] = (uint8_t*)p;
    }
    S.ipc = true;
    return shard_finish_connect(m);
}

extern "C" int wd_shard_connect_local(WdModel** models, int32_t n_ranks) {
    if (!models || n_ranks < 1) { set_error("bad arguments"); return WD_EINVAL; }
    for (int r = 0; r < n_ranks; ++r) {
        WdModel* m = models[r];
        if (!m || m->shard.world != n_ranks || m->shard.rank != r) { set_error("wd_shard_connect_local: handle %d is not rank %d of %d", r, r, n_ranks); return WD_EINVAL; }
        if (m->shard.seg_bytes != models[0]->shard.seg_bytes) { set_error("exchange segments differ between ranks (plans differ)"); return WD_EINVAL; }
    }
    for (int r = 0; r < n_ranks; ++r) {
        WdModel* m = models[r];
        WD_CUDA(cudaSetDevice(m->device));
        for (int q = 0; q < n_ranks; ++q) {
            m->shard.peer_seg[q] = models[q]->shard.seg;
            if (models[q]->device != m->device) {
                cudaError_t e = cudaDeviceEnablePeerAccess(models[q]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { set_error("cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e)); return WD_ECUDA; }
                cudaGetLastError();
            }
        }
        m->shard.ipc = false;
        int rc = shard_finish_connect(m);
        if (rc) return rc;
    }
    return WD_OK;
}

// every stream of every handle waits for everything enqueued so far on all of them (device side only): the "barrier" between
// phases when all ranks are driven by one process
extern "C" int wd_shard_local_sync(WdModel** models, int32_t n_ranks) {
    if (!models) { set_error("null argument"); return WD_EINVAL; }
    std::vector<cudaEvent_t> evs;
    for (int r = 0; r < n_ranks; ++r) {
        WdModel* m = models[r];
        WD_CUDA(cudaSetDevice(m->device));
        for (cudaStream_t st : {m->stream, m->sstream[0], m->sstream[1], m->shard.aux}) {
            if (!st) continue;
            cudaEvent_t ev;
            WD_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            WD_CUDA(cudaEventRecord(ev, st));
            evs.push_back(ev);
        }
    }
    for (int r = 0; r < n_ranks; ++r) {
        WdModel* m = models[r];
        WD_CUDA(cudaSetDevice(m->device));
        for (cudaStream_t st : {m->stream, m->sstream[0], m->sstream[1], m->shard.aux})
            if (st) for (cudaEvent_t ev : evs) WD_CUDA(cudaStreamWaitEvent(st, ev, 0));
    }
    for (cudaEvent_t ev : evs) cudaEventDestroy(ev);
    return WD_OK;
}
