// Device primitives for the sparse backward: exclusive scan and a stable LSD radix sort of (key, value)
// pairs whose length lives in DEVICE memory (no host sync between the id stage and the backward).
//
// The sort groups the step's (row id -> occurrence) pairs so that every touched table row gets exactly
// one optimizer update from the ordered sum of its gradients — TensorFlow's "sum duplicates, apply once"
// semantics for IndexedSlices (SURVEY.md A.8) — without float atomics (bit-reproducible run to run).
#include <stdlib.h>

#include "common.cuh"

namespace wd {

constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_ITEMS = 4;
constexpr int SCAN_CHUNK = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ int warp_incl_scan(int v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, d);
        if ((threadIdx.x & 31) >= d) v += t;
    }
    return v;
}

// block-wide exclusive scan of one int per thread (blockDim.x multiple of 32, <= 1024); returns exclusive
// prefix, *total = block sum.  smem: 33 ints.
__device__ __forceinline__ int block_excl_scan(int v, int* smem, int* total) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int inc = warp_incl_scan(v);
    if (lane == 31) smem[w] = inc;
    __syncthreads();
    if (w == 0) {
        int s = lane < nw ? smem[lane] : 0;
        int si = warp_incl_scan(s);
        smem[lane] = si - s;
        if (lane == 31) smem[32] = si;
    }
    __syncthreads();
    int r = inc - v + smem[w];
    *total = smem[32];
    __syncthreads();
    return r;
}

// Phase 1: per-chunk exclusive scan in place + chunk totals; the last block to finish scans the totals.
__global__ void __launch_bounds__(SCAN_THREADS) scan_chunks_kernel(int32_t* data, int64_t n, int32_t* chunk_sums,
                                                                   int32_t* counter) {
    __shared__ int sm[33];
    __shared__ bool is_last;
    int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = (base + i < n) ? data[base + i] : 0;
        s += v[i];
    }
    int tot;
    int ex = block_excl_scan(s, sm, &tot);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < n) data[base + i] = ex;
        ex += v[i];
    }
    if (threadIdx.x == 0) {
        chunk_sums[blockIdx.x] = tot;
        __threadfence();
        int t = atomicAdd(counter, 1);
        is_last = (t == (int)gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // scan chunk_sums[0..gridDim.x) in place (exclusive), total at chunk_sums[gridDim.x]
    int carry = 0;
    for (int off = 0; off < (int)gridDim.x; off += SCAN_THREADS) {
        int i = off + threadIdx.x;
        int x = i < (int)gridDim.x ? ((volatile int32_t*)chunk_sums)[i] : 0;
        int t2;
        int e = block_excl_scan(x, sm, &t2);
        if (i < (int)gridDim.x) chunk_sums[i] = e + carry;
        carry += t2;
    }
    if (threadIdx.x == 0) {
        chunk_sums[gridDim.x] = carry;
        *counter = 0;
    }
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_add_kernel(int32_t* data, int64_t n, const int32_t* chunk_sums,
                                                                int nchunks, int32_t* total_out) {
    int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int add = chunk_sums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i)
        if (base + i < n) data[base + i] += add;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int tot = chunk_sums[nchunks];
        data[n] = tot;                 // CSR sentinel
        if (total_out) *total_out = tot;
    }
}

// In-place exclusive scan of data[0..n) (n known on host); data[n] and *total_out receive the total.
int exclusive_scan_i32(WdModel* m, int32_t* data, int64_t n, int32_t* total_out) {
    int nchunks = (int)((n + SCAN_CHUNK - 1) / SCAN_CHUNK);
    if (nchunks < 1) nchunks = 1;
    const SortScratch& sc = m->scratch[m->scratch_sel];
    scan_chunks_kernel<<<nchunks, SCAN_THREADS, 0, m->stream>>>(data, n, sc.scan, sc.counter);
    scan_add_kernel<<<nchunks, SCAN_THREADS, 0, m->stream>>>(data, n, sc.scan, nchunks, total_out);
    m->launches += 2;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ------------------------------------------------------------------------- fused scans of the grouping stage
// The two scans of the grouping stage take their input from a formula instead of an array, and the first one's add pass is also
// the compaction: 4 launches where (flag kernel, scan, scan-add, compact kernel, chunk-count kernel, scan, scan-add) were 7.
//   GEN 0: value(i) = 1 where the sorted key i starts a new valid segment (segment heads -> unique rows)
//   GEN 1: value(u) = chunks of unique row u if it is a multi-chunk (hot) row, else 0; also pads urow[u >= nuniq] with kInvalidRow
struct ScanGen { const int32_t* d_n; const uint32_t* keys; uint32_t invalid; const int32_t* ustart; uint32_t* urow; int chunk; };
template <int GEN>
__device__ __forceinline__ int scan_gen_value(const ScanGen& g, int64_t i, int n) {
    if (GEN == 0) {
        if (i >= n) return 0;
        const uint32_t k = g.keys[i];
        return (k != g.invalid && (i == 0 || g.keys[i - 1] != k)) ? 1 : 0;
    }
    if (i < n) {
        const int len = g.ustart[i + 1] - g.ustart[i];
        return len > g.chunk ? (len + g.chunk - 1) / g.chunk : 0;
    }
    g.urow[i] = kInvalidRow;
    return 0;
}
template <int GEN>
__global__ void __launch_bounds__(SCAN_THREADS) scan_gen_chunks_kernel(ScanGen g, int32_t* data, int64_t cap, int32_t* chunk_sums, int32_t* counter) {
    __shared__ int sm[33];
    __shared__ bool is_last;
    const int n = *g.d_n;
    int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = (base + i < cap) ? scan_gen_value<GEN>(g, base + i, n) : 0;
        s += v[i];
    }
    int tot;
    int ex = block_excl_scan(s, sm, &tot);
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < cap) data[base + i] = ex;
        ex += v[i];
    }
    if (threadIdx.x == 0) {
        chunk_sums[blockIdx.x] = tot;
        __threadfence();
        int t = atomicAdd(counter, 1);
        is_last = (t == (int)gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    int carry = 0;
    for (int off = 0; off < (int)gridDim.x; off += SCAN_THREADS) {
        int i = off + threadIdx.x;
        int x = i < (int)gridDim.x ? ((volatile int32_t*)chunk_sums)[i] : 0;
        int t2;
        int e = block_excl_scan(x, sm, &t2);
        if (i < (int)gridDim.x) chunk_sums[i] = e + carry;
        carry += t2;
    }
    if (threadIdx.x == 0) {
        chunk_sums[gridDim.x] = carry;
        *counter = 0;
    }
}
// add pass of the segment-head scan + compaction: head i goes to slot pos(i) of (ustart, urow); the end of the last valid segment
// closes the list; *d_nuniq = number of heads
__global__ void __launch_bounds__(SCAN_THREADS) seg_add_compact_kernel(ScanGen g, const int32_t* __restrict__ pos, const int32_t* __restrict__ chunk_sums,
                                                                       int nchunks, int32_t* __restrict__ ustart, uint32_t* __restrict__ urow,
                                                                       int32_t* __restrict__ d_nuniq) {
    const int n = *g.d_n;
    const int add = chunk_sums[blockIdx.x], total = chunk_sums[nchunks];
    int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        const int64_t i = base + j;
        if (i >= n) continue;
        const uint32_t k = g.keys[i];
        if (k == g.invalid) continue;
        if (i == 0 || g.keys[i - 1] != k) {
            const int p = pos[i] + add;
            ustart[p] = (int32_t)i;
            urow[p] = k;
        }
        if (i == n - 1 || g.keys[i + 1] == g.invalid) ustart[total] = (int32_t)i + 1;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *d_nuniq = total;
}

// unique rows of the sorted keys: (ustart, urow, *d_nuniq); `pos` = scratch of `cap` ints
int seg_heads(WdModel* m, const int32_t* d_n, const uint32_t* keys, uint32_t invalid, int32_t* pos, int64_t cap, int32_t* ustart, uint32_t* urow,
              int32_t* d_nuniq) {
    int nchunks = (int)((cap + SCAN_CHUNK - 1) / SCAN_CHUNK);
    if (nchunks < 1) nchunks = 1;
    const SortScratch& sc = m->scratch[m->scratch_sel];
    const ScanGen g{d_n, keys, invalid, nullptr, nullptr, 0};
    scan_gen_chunks_kernel<0><<<nchunks, SCAN_THREADS, 0, m->stream>>>(g, pos, cap, sc.scan, sc.counter);
    seg_add_compact_kernel<<<nchunks, SCAN_THREADS, 0, m->stream>>>(g, pos, sc.scan, nchunks, ustart, urow, d_nuniq);
    m->launches += 2;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
// hot-row chunk layout: choff = exclusive scan of the chunk counts of the unique rows (0 for rows summed directly), choff[cap] and
// *d_nchunks = total; pads urow beyond the unique rows with kInvalidRow
int chunk_offsets(WdModel* m, const int32_t* d_nuniq, const int32_t* ustart, uint32_t* urow, int32_t* choff, int64_t cap, int chunk, int32_t* d_nchunks) {
    int nchunks = (int)((cap + SCAN_CHUNK - 1) / SCAN_CHUNK);
    if (nchunks < 1) nchunks = 1;
    const SortScratch& sc = m->scratch[m->scratch_sel];
    const ScanGen g{d_nuniq, nullptr, 0u, ustart, urow, chunk};
    scan_gen_chunks_kernel<1><<<nchunks, SCAN_THREADS, 0, m->stream>>>(g, choff, cap, sc.scan, sc.counter);
    scan_add_kernel<<<nchunks, SCAN_THREADS, 0, m->stream>>>(choff, cap, sc.scan, nchunks, d_nchunks);
    m->launches += 2;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ------------------------------------------------------------------------------------------ radix sort
constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
// Keys per tile (template parameter TILE of the three kernels): kSortTile = 1024 for the lists of a few 100 K keys (short blocks,
// enough of them to fill the SMs); RS_BIG_TILE for lists of millions of keys, where the per-tile overhead (clearing and scanning
// RS_WARPS x bins counters, the bin-base scan: ~10 shared-memory operations per key at 1024 keys) is what a pass costs.
constexpr int RS_BIG_TILE = 4096;

// Per-tile digit histogram -> hist[tile * bins + bin] (tile-major, coalesced) and global per-bin totals gtot[bin].
template <int RS_TILE>
__global__ void __launch_bounds__(RS_THREADS) rs_hist_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ d_n,
                                                             int shift, int bins, int32_t* __restrict__ hist, int32_t* __restrict__ gtot) {
    extern __shared__ int sh[];           // bins
    const int n = *d_n;
    const int ntiles = (n + RS_TILE - 1) / RS_TILE;
    const int tile = blockIdx.x;
    if (tile >= ntiles) return;
    for (int i = threadIdx.x; i < bins; i += RS_THREADS) sh[i] = 0;
    __syncthreads();
    const int base = tile * RS_TILE;
    for (int i = threadIdx.x; i < RS_TILE; i += RS_THREADS) {
        int j = base + i;
        if (j < n) atomicAdd(&sh[(keys[j] >> shift) & (bins - 1)], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < bins; i += RS_THREADS) {
        hist[(int64_t)tile * bins + i] = sh[i];
    }
}

// Column scan: one warp per bin turns the per-tile counts hist[tile][bin] into exclusive prefixes over tiles
// (32 tiles per shuffle scan); the last lane leaves the bin total in gtot[bin].
template <int RS_TILE>
__global__ void __launch_bounds__(256) rs_colscan_kernel(const int32_t* __restrict__ d_n, int bins, int32_t* __restrict__ hist, int32_t* __restrict__ gtot) {
    const int n = *d_n;
    const int ntiles = (n + RS_TILE - 1) / RS_TILE;
    const int bin = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (bin >= bins) return;
    int carry = 0;
    for (int t0 = 0; t0 < ntiles; t0 += 128) {              // 4 independent loads in flight per lane, then 4 shuffle scans
        int v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int t = t0 + i * 32 + lane;
            v[i] = t < ntiles ? hist[(int64_t)t * bins + bin] : 0;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int t = t0 + i * 32 + lane;
            int inc = v[i];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { int x = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += x; }
            if (t < ntiles) hist[(int64_t)t * bins + bin] = carry + inc - v[i];
            carry += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
    if (lane == 0) gtot[bin] = carry;
}

// Stable scatter of one tile.  Output base of (tile, bin) = exclusive scan over bins of the bin totals + the tile's
// prefix inside the bin (both precomputed by rs_colscan_kernel).
// LOCAL (the big-list instance): a key's 4-byte store into its bin's run is one store transaction per key whatever L2 does with
// the sector afterwards, and at ~0.4 such transactions per clock and SM that rate is what a pass of a 5 M-key list costs.  So the tile is first reordered in shared memory (position = the bin's tile-local base + the key's offset inside the
// tile's run) and then written out in that order: consecutive threads hold consecutive addresses of a run, a warp's store covers
// whole runs (4096 / bins keys each) instead of 32 unrelated sectors.
template <int RS_TILE, bool LOCAL>
__global__ void __launch_bounds__(RS_THREADS) rs_scatter_kernel(const uint32_t* __restrict__ keys_in,
                                                                const uint32_t* __restrict__ vals_in,
                                                                uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
                                                                const int32_t* __restrict__ d_n, int shift, int bins,
                                                                const int32_t* __restrict__ hist, const int32_t* __restrict__ gtot) {
    extern __shared__ int wh[];           // [RS_WARPS][bins], tilebase[bins]; LOCAL: + lbase[bins], skey[RS_TILE], sval[RS_TILE]
    __shared__ int sm[33];
    constexpr int RS_ITEMS_PER_WARP = RS_TILE / RS_WARPS;
    const int n = *d_n;
    const int ntiles = (n + RS_TILE - 1) / RS_TILE;
    const int tile = blockIdx.x;
    if (tile >= ntiles) return;
    int* tilebase = wh + RS_WARPS * bins;
    int* lbase = tilebase + bins;
    uint32_t* skey = reinterpret_cast<uint32_t*>(lbase + bins);
    uint32_t* sval = skey + RS_TILE;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int per = bins / RS_THREADS > 0 ? bins / RS_THREADS : 1;           // bins is a power of two >= 256
    const int b0 = threadIdx.x * per;
    {
        int tot[4] = {0, 0, 0, 0};
        int s = 0;
        if (b0 < bins)
            for (int k = 0; k < per; ++k) { tot[k] = gtot[b0 + k]; s += tot[k]; }
        int blocktot;
        int run = block_excl_scan(s, sm, &blocktot);
        if (b0 < bins)
            for (int k = 0; k < per; ++k) { tilebase[b0 + k] = run + hist[(int64_t)tile * bins + b0 + k]; run += tot[k]; }
    }
    for (int i = threadIdx.x; i < RS_WARPS * bins; i += RS_THREADS) wh[i] = 0;
    __syncthreads();
    const int wbase = tile * RS_TILE + w * RS_ITEMS_PER_WARP;
    int* my = wh + w * bins;
    // the warp's keys and values, all loads in flight at once: the rounds below are ordered (a round's ranks depend on the counters
    // the previous round left), so loading inside them would put one global-memory round trip on every round of both phases
    constexpr int RS_ROUNDS = RS_ITEMS_PER_WARP / 32;
    uint32_t kreg[RS_ROUNDS], vreg[RS_ROUNDS];
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        const int j = wbase + r * 32 + lane;
        kreg[r] = j < n ? keys_in[j] : 0u;
        vreg[r] = j < n ? vals_in[j] : 0u;
    }
    // phase A: per-warp histogram
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        const int j = wbase + r * 32 + lane;
        if (j < n) atomicAdd(&my[(kreg[r] >> shift) & (bins - 1)], 1);
    }
    __syncthreads();
    // phase B: warp bases = tile base + counts of earlier warps
    for (int b = threadIdx.x; b < bins; b += RS_THREADS) {
        int run = tilebase[b];
#pragma unroll
        for (int ww = 0; ww < RS_WARPS; ++ww) {
            int c = wh[ww * bins + b];
            wh[ww * bins + b] = run;
            run += c;
        }
        if (LOCAL) lbase[b] = run - tilebase[b];                              // keys of this tile in bin b
    }
    __syncthreads();
    if (LOCAL) {                                                              // lbase = exclusive scan over bins of the tile's counts
        int tot[4] = {0, 0, 0, 0};
        int s = 0;
        if (b0 < bins)
            for (int k = 0; k < per; ++k) { tot[k] = lbase[b0 + k]; s += tot[k]; }
        int blocktot;
        int run = block_excl_scan(s, sm, &blocktot);
        if (b0 < bins)
            for (int k = 0; k < per; ++k) { lbase[b0 + k] = run; run += tot[k]; }
        __syncthreads();
    }
    // phase C: ordered rounds; rank inside a round by match_any
#pragma unroll
    for (int r = 0; r < RS_ROUNDS; ++r) {
        const int j = wbase + r * 32 + lane;
        const bool valid = j < n;
        const uint32_t k = kreg[r], v = vreg[r];
        int d = valid ? (int)((k >> shift) & (bins - 1)) : bins;    // invalid lanes get a digit nobody shares
        // lanes holding the same digit: one ballot per digit bit (match.any.sync costs ~5 issue cycles per key and SM here, which
        // was what a pass of a long list took; ten votes and twenty logic operations are several times cheaper)
        unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
        for (int bit = 0; bit < 10; ++bit) {                        // bins <= 1024; bits above the digit are 0 in every valid lane
            const bool one = (d >> bit) & 1;
            const unsigned mask = __ballot_sync(0xffffffffu, one);
            peers &= one ? mask : ~mask;
        }
        int rank = __popc(peers & ((1u << lane) - 1u));
        int pos = 0;
        if (valid) pos = my[d] + rank;
        __syncwarp();
        if (valid && rank == 0) my[d] += __popc(peers);
        __syncwarp();
        if (valid) {
            if (LOCAL) {
                const int lp = lbase[d] + (pos - tilebase[d]);
                skey[lp] = k;
                sval[lp] = v;
            } else {
                keys_out[pos] = k;
                vals_out[pos] = v;
            }
        }
    }
    if (LOCAL) {
        __syncthreads();
        const int nt = min(RS_TILE, n - tile * RS_TILE);
        for (int i = threadIdx.x; i < nt; i += RS_THREADS) {
            const uint32_t k = skey[i];
            const int d = (int)((k >> shift) & (bins - 1));
            const int o = tilebase[d] + (i - lbase[d]);
            keys_out[o] = k;
            vals_out[o] = sval[i];
        }
    }
}

// Sort pairs (*keys, *vals) of length *d_n by the low `bits` bits of the key, with (*keys2, *vals2) as the ping-pong buffers.
// On return the sorted pairs are in (*keys, *vals) (the pointers are swapped as needed).  Scratch: the current stream's set.
int radix_sort_pairs(WdModel* m, uint32_t** keys, uint32_t** vals, uint32_t** keys2, uint32_t** vals2, int bits, const int32_t* d_n) {
    if (bits < 1) bits = 1;
    // Lists of millions of keys (the wide-only workload: 5.4 M keys per step): 4096-key tiles reordered in shared memory before
    // they are written (rs_scatter_kernel<.., true>; on an H100 80GB HBM3 at 700 W the wide workload trains at 89 M examples/s
    // with the reorder and at 71 M without it).  (Without that reorder narrower digits do not help: every key stays one store
    // transaction.)  WD_SORT_DIGIT_BITS=8|9|10 fixes the digit width (the tests use it to reach the 1024-bin kernels with small
    // tables).
    const bool big = m->max_nnz >= (int64_t)2 << 20;
    int passes = (bits + 9) / 10;
    int per = (bits + passes - 1) / passes;
    if (per < 8) per = 8;                                   // bins >= 256 so every thread owns at least one bin
    if (const char* e = getenv("WD_SORT_DIGIT_BITS")) {
        const int v = atoi(e);
        if (v >= 8 && v <= 10) { per = v; passes = (bits + per - 1) / per; }
    }
    int bins = 1 << per;
    const int tile = big ? RS_BIG_TILE : kSortTile;
    int ntiles_cap = (int)((m->max_nnz + tile - 1) / tile);
    if ((int64_t)bins * ntiles_cap + 4 * 1024 > m->sort_hist_cap) {
        set_error("radix sort histogram capacity too small");
        return WD_ESTATE;
    }
    int32_t* hist = m->scratch[m->scratch_sel].hist;
    int32_t* gtot = hist + (int64_t)bins * ntiles_cap;                  // [passes][bins]
    for (int p = 0; p < passes; ++p) {
        int shift = p * per;
        const size_t sh_h = bins * sizeof(int), sh_s = (RS_WARPS + 1) * bins * sizeof(int);
        const size_t sh_l = (RS_WARPS + 2) * bins * sizeof(int) + 2 * RS_BIG_TILE * sizeof(uint32_t);    // + lbase, skey, sval
        const int gcs = (bins * 32 + 255) / 256;
        if (big) {
            if (!m->sort_smem_opt_in) {                                 // 72 KB of dynamic shared memory at 1024 bins (per device: once per handle)
                WD_CUDA(cudaFuncSetAttribute(rs_scatter_kernel<RS_BIG_TILE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
                m->sort_smem_opt_in = true;
            }
            rs_hist_kernel<RS_BIG_TILE><<<ntiles_cap, RS_THREADS, sh_h, m->stream>>>(*keys, d_n, shift, bins, hist, gtot + p * bins);
            rs_colscan_kernel<RS_BIG_TILE><<<gcs, 256, 0, m->stream>>>(d_n, bins, hist, gtot + p * bins);
            rs_scatter_kernel<RS_BIG_TILE, true><<<ntiles_cap, RS_THREADS, sh_l, m->stream>>>(
                *keys, *vals, *keys2, *vals2, d_n, shift, bins, hist, gtot + p * bins);
        } else {
            rs_hist_kernel<kSortTile><<<ntiles_cap, RS_THREADS, sh_h, m->stream>>>(*keys, d_n, shift, bins, hist, gtot + p * bins);
            rs_colscan_kernel<kSortTile><<<gcs, 256, 0, m->stream>>>(d_n, bins, hist, gtot + p * bins);
            rs_scatter_kernel<kSortTile, false><<<ntiles_cap, RS_THREADS, sh_s, m->stream>>>(
                *keys, *vals, *keys2, *vals2, d_n, shift, bins, hist, gtot + p * bins);
        }
        m->launches += 3;
        std::swap(*keys, *keys2);
        std::swap(*vals, *vals2);
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

}  // namespace wd
