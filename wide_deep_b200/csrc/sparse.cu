// Sparse half of the step: wide linear logit, multihot embedding gather + mean-pool, and the backward
// scatter of both fused with their per-row optimizers.
//
//   wide_fwd_kernel        tf.feature_column.linear_model(sparse_combiner='sum')   (reference linear.py:29-36)
//   emb_pool_fwd_kernel    embedding_column(combiner='mean') inside input_layer     (reference dnn.py:88-90;
//                          safe_embedding_lookup_sparse: empty bag -> zeros, SURVEY A.7)
//   seg_* / *_apply        SparseSegmentMeanGrad + SparseApplyAdagrad / SparseApplyFtrl (reference
//                          joint.py:234-247 minimize(); SURVEY A.8-A.9): one update per touched row from the
//                          ordered sum of its gradients.
// HBM-bound kernels: 16-byte vector loads through the read-only path, several rows in flight per lane
// group, rows are 16..256 B records {w | optimizer slots} so forward touches one line and backward one
// contiguous record.
#include "common.cuh"
#include "sparse_dev.cuh"

namespace wd {


// ------------------------------------------------------------------------------------------- wide forward
// one warp per example: sum of w[row] over the example's wide ids (+ bias)
__global__ void __launch_bounds__(256) wide_fwd_kernel(int B, int C, const int32_t* __restrict__ offs,
                                                       const uint32_t* __restrict__ e_wide, const float4* __restrict__ wide,
                                                       const float* __restrict__ bias, float* __restrict__ out) {
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int nwarps = (gridDim.x * blockDim.x) >> 5;
    float b0 = bias[0];
    for (int b = warp; b < B; b += nwarps) {
        int s = offs[(int64_t)b * C], e = offs[(int64_t)(b + 1) * C];
        float acc = 0.f;
        for (int j = s + lane; j < e; j += 32) {
            uint32_t r = e_wide[j];
            if (r != kInvalidRow) acc += __ldg(&wide[r].x);
        }
        acc = warp_sum(acc);
        if (lane == 0) out[b] = acc + b0;
    }
}

// --------------------------------------------------------------------------------------- embedding forward
// All tables of one width D (G = D/4 lanes per bag, float4 per lane), desc[k] = table k of the width (gather view).  Bag =
// (example b, table k).  Long multihot bags: a full warp per bag, the 32/G lane groups take interleaved ids, then a shuffle tree
// combines them.
template <int G>
__global__ void __launch_bounds__(256) emb_pool_fwd_kernel(int B, int C, int ntab, const TabDesc* __restrict__ desc,
                                                           const int32_t* __restrict__ offs, const uint32_t* __restrict__ e_emb,
                                                           float* __restrict__ X0, int ld) {
    constexpr int GROUPS = 32 / G;
    const int lane = threadIdx.x & 31, lig = lane % G, grp = lane / G;
    const int64_t nbags = (int64_t)B * ntab;
    const int64_t gwarp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarp = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t bag = gwarp; bag < nbags; bag += nwarp) {
        const int b = (int)(bag / ntab);
        const TabDesc d = desc[bag % ntab];
        int s = offs[(int64_t)b * C + d.col], e = offs[(int64_t)b * C + d.col + 1];
        const float* base = d.data + lig * 4;
        const int stride = d.stride;
        const int64_t rb = d.row_base;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        // 32 ids of the bag per round trip (one per lane), then the rows of the chunk that belong to this lane group eight at a
        // time back to back: the chain offsets -> ids -> rows is 2 + ceil(rows / (8 GROUPS)) dependent round trips per 32 ids
        // instead of one per four rows.  (Sixteen in flight was measured slower: 120 registers -> 2 blocks per SM -> 3.5 waves
        // of the 8192 bags, 25.6 us against 20 us.)  Group grp still sums rows grp, grp + GROUPS, ... in that order (the result
        // is bit-identical to the sequential walk).
        constexpr int STEPS = 32 / GROUPS, RND = STEPS < 8 ? STEPS : 8;
        for (int j0 = s; j0 < e; j0 += 32) {
            const int cnt = min(32, e - j0);
            const uint32_t my = lane < cnt ? e_emb[j0 + lane] : 0u;
#pragma unroll
            for (int k0 = 0; k0 < STEPS; k0 += RND) {
                if (k0 * GROUPS >= cnt) break;
                float4 v[RND];
#pragma unroll
                for (int u = 0; u < RND; ++u) {
                    const int r = (k0 + u) * GROUPS + grp;
                    const uint32_t id = __shfl_sync(0xffffffffu, my, r & 31);
                    v[u] = r < cnt ? ldg_nc_f4(base + (int64_t)(id - rb) * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int u = 0; u < RND; ++u) {
                    if ((k0 + u) * GROUPS + grp < cnt) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
                }
            }
        }
#pragma unroll
        for (int d = G; d < 32; d <<= 1) {                  // segmented (per lane-in-group) shuffle reduction
            acc.x += __shfl_xor_sync(0xffffffffu, acc.x, d);
            acc.y += __shfl_xor_sync(0xffffffffu, acc.y, d);
            acc.z += __shfl_xor_sync(0xffffffffu, acc.z, d);
            acc.w += __shfl_xor_sync(0xffffffffu, acc.w, d);
        }
        int n = e - s;
        if (n > 1) {
            float inv = 1.f / (float)n;
            acc.x *= inv; acc.y *= inv; acc.z *= inv; acc.w *= inv;
        }
        if (grp == 0) *reinterpret_cast<float4*>(X0 + (int64_t)b * ld + d.x0 + lig * 4) = acc;
    }
}

// Warp per example (short bags).  The warp walks the example's bags of this width in rounds of 32/G bags and
// issues the loads of RMAX rounds back to back: offsets, then first ids, then first rows — every lane group keeps
// RMAX independent 16-byte row loads in flight instead of one dependent chain at a time.
template <int G, int RMAX>
__global__ void __launch_bounds__(256, 4) emb_pool_fwd_rows_kernel(int B, int C, int ntab, const TabDesc* __restrict__ desc,
                                                                const int32_t* __restrict__ offs, const uint32_t* __restrict__ e_emb,
                                                                float* __restrict__ X0, int ld) {
    constexpr int GROUPS = 32 / G;
    const int lane = threadIdx.x & 31, lig = lane % G, grp = lane / G;
    const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarp = (gridDim.x * blockDim.x) >> 5;
    for (int b = gwarp; b < B; b += nwarp) {
        const int32_t* orow = offs + (int64_t)b * C;
        float* xrow = X0 + (int64_t)b * ld;
        for (int k0 = 0; k0 < ntab; k0 += GROUPS * RMAX) {
            TabDesc d[RMAX];
            int s[RMAX], n[RMAX];
            float4 acc[RMAX];
#pragma unroll
            for (int r = 0; r < RMAX; ++r) {
                const int k = k0 + r * GROUPS + grp;
                n[r] = -1;
                if (k < ntab) {
                    d[r] = desc[k];
                    s[r] = orow[d[r].col];
                    n[r] = orow[d[r].col + 1] - s[r];
                }
            }
            uint32_t id0[RMAX];
#pragma unroll
            for (int r = 0; r < RMAX; ++r) id0[r] = n[r] > 0 ? e_emb[s[r]] : 0u;
#pragma unroll
            for (int r = 0; r < RMAX; ++r) {
                acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (n[r] > 0) acc[r] = ldg_nc_f4(d[r].data + (int64_t)(id0[r] - d[r].row_base) * d[r].stride + lig * 4);
            }
#pragma unroll
            for (int r = 0; r < RMAX; ++r) {
                if (n[r] > 1) {                                  // multihot bag: remaining rows, then the mean
                    for (int j = 1; j < n[r]; ++j) {
                        float4 v = ldg_nc_f4(d[r].data + (int64_t)(e_emb[s[r] + j] - d[r].row_base) * d[r].stride + lig * 4);
                        acc[r].x += v.x; acc[r].y += v.y; acc[r].z += v.z; acc[r].w += v.w;
                    }
                    const float inv = 1.f / (float)n[r];
                    acc[r].x *= inv; acc[r].y *= inv; acc[r].z *= inv; acc[r].w *= inv;
                }
                if (n[r] >= 0) *reinterpret_cast<float4*>(xrow + d[r].x0 + lig * 4) = acc[r];
            }
        }
    }
}

template <int G>
static void launch_emb_fwd(WdModel* m, int di, bool widebag) {
    const int ntab = m->dim_ntables[di];
    if (!widebag) {
        constexpr int RMAX = 4;                       // 4 rounds in flight per lane group at <= 64 registers: 32 warps per SM
        int grid = grid_for((int64_t)m->dbatch.B * 32, 256, kNumSms * 8);
        emb_pool_fwd_rows_kernel<G, RMAX><<<grid, 256, 0, m->stream>>>(m->dbatch.B, m->n_columns, ntab, m->d_dim_desc[di], m->d_col_offs,
                                                                        m->d_g_emb, m->d_X0, m->d0_phys);
    } else {
        const int64_t nbags = (int64_t)m->dbatch.B * ntab;            // one warp per bag
        int grid = grid_for(nbags * 32, 256, kNumSms * 8);
        emb_pool_fwd_kernel<G><<<grid, 256, 0, m->stream>>>(m->dbatch.B, m->n_columns, ntab, m->d_dim_desc[di], m->d_col_offs,
                                                             m->d_g_emb, m->d_X0, m->d0_phys);
    }
    m->launches++;
}

// the wide half of the forward (independent of the deep half until the head adds the logits)
int sparse_forward_wide(WdModel* m) {
    const int B = m->dbatch.B;
    if (m->use_wide) {
        wide_fwd_kernel<<<grid_for((int64_t)B * 32, 256), 256, 0, m->stream>>>(B, m->n_columns, m->d_col_offs, m->d_e_wide,
                                                                              m->d_wide, m->d_P + m->dense[0].off, m->d_wide_logit);
        m->launches++;
        mark(m, "wide_fwd");
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int sparse_forward_emb(WdModel* m);
int sparse_forward(WdModel* m) {
    int rc = sparse_forward_wide(m);
    return rc ? rc : sparse_forward_emb(m);
}
int sparse_forward_emb(WdModel* m) {
    if (m->use_deep) {
        // heuristic: average bag length from the key count of the batch decides narrow vs full-warp bags
        bool widebag = m->max_nnz > 0 && (m->keys_cap / (int64_t)(m->max_batch * (m->n_cat_fields > 0 ? m->n_cat_fields : 1))) >= 8;
        for (int di = 0; di < m->n_dims; ++di) {
            switch (m->dims[di] / 4) {
                case 1: launch_emb_fwd<1>(m, di, false); break;
                case 2: launch_emb_fwd<2>(m, di, widebag); break;
                case 4: launch_emb_fwd<4>(m, di, widebag); break;
                case 8: launch_emb_fwd<8>(m, di, widebag); break;
                case 16: launch_emb_fwd<16>(m, di, widebag); break;
                case 32: launch_emb_fwd<32>(m, di, true); break;
                default: set_error("unsupported embedding width %d (supported: 4,8,16,32,64,128)", m->dims[di]); return WD_EUNSUPPORTED;
            }
        }
        mark(m, "emb_fwd");
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ------------------------------------------------------------------------------------ backward: grouping
// (key, value) pairs for the two sorts (which = 0 embedding rows, 1 wide rows): key = row — non-participating entries get the key
// `invalid` (= 1 << bits), so they sort behind every real row —, value = val_src[i], or the entry's index i without val_src.
// The batch's own lists carry the entry's cell index bc = b * C + c (e_bc) as the value: that is all the gradient sums need to
// find an occurrence's gradient, so they read it straight from the sorted list instead of chasing e_bc[index] per occurrence.
__global__ void sort_keys_kernel(const int32_t* __restrict__ d_nnz, const uint32_t* __restrict__ e_row, uint32_t invalid,
                                 uint32_t* keys, uint32_t* vals, const int32_t* __restrict__ val_src) {
    int n = *d_nnz;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint32_t r = e_row[i];
        keys[i] = r == kInvalidRow ? invalid : r;
        vals[i] = val_src ? (uint32_t)val_src[i] : (uint32_t)i;
    }
}


// ---- per-row gradient sums of the batch's own lists (emb_grad_sum_kernel / wide_grad_sum_kernel, sparse_dev.cuh).  The sorted
// values are the occurrences' cell indices bc = b * C + c: that is all a sum needs to find an occurrence's gradient.
// embedding rows: occurrence bc contributes dX0[b, x0 : x0 + dim] / bag_size(b, c), x0 and dim of column c's table
// (the sources' arrays are read-only during the sums: loaded through the read-only path, as restrict kernel arguments would be)
struct LocalEmb {
    const uint32_t* sbc;
    const int32_t* offs;
    int C;
    const int32_t* col_table;
    const int32_t* tab_dim;
    const int32_t* tab_x0;
    const float* dX0;
    int ld;
    __device__ __forceinline__ uint32_t key(int j) const { return __ldg(sbc + j); }
    __device__ __forceinline__ void layout(uint32_t k, int& t, int& dim, int& x0) const {
        t = __ldg(col_table + (int)k % C);
        dim = __ldg(tab_dim + t); x0 = __ldg(tab_x0 + t);
    }
    __device__ __forceinline__ float4 row(uint32_t k, int x0, int q, float& inv) const {
        const int bc = (int)k;
        const float4 v = __ldg(reinterpret_cast<const float4*>(dX0 + (int64_t)(bc / C) * ld + x0 + q * 4));
        inv = 1.f / (float)(__ldg(offs + bc + 1) - __ldg(offs + bc));
        return v;
    }
};
// wide rows: occurrence bc contributes dlogit[b]
struct LocalWide {
    const uint32_t* sbc;
    int C;
    const float* dlogit;
    __device__ __forceinline__ uint32_t key(int j) const { return __ldg(sbc + j); }
    __device__ __forceinline__ float row(uint32_t k) const { return __ldg(dlogit + k / (uint32_t)C); }
};

// ugrad[u] = sum of the row's chunk partials (multi-chunk rows only).  Each lane checks one unique row; the (rare)
// multi-chunk rows of a warp are combined by the whole warp: lane groups add chunks g, g+NG, ... and a fixed-order shuffle
// tree adds the group sums, so the result does not depend on scheduling.  Hot rows are neighbours in row order (they are the
// rows of the small tables), so a warp takes every NW-th group of rows (lane l of warp w checks row (it * 32 + l) * NW + w):
// neighbouring hot rows land in different warps and their long chunk lists are walked concurrently, not one after the other.
// KIND 0: the sum goes to ugrad.  KIND 1 / 2 (single-GPU step, row-local optimizer): the hot row's optimizer update follows its
// sum here (1: embedding record, tables of ra.rec in row order, width a power of two in [4, 128]; 2: wide record, width 1) —
// together with the APPLY variants of the gradient-sum kernels this leaves no separate optimizer launch for the list.
template <int KIND>
__global__ void __launch_bounds__(256) chunk_combine_kernel(const int32_t* __restrict__ d_nuniq, const int32_t* __restrict__ choff,
                                                            const float* __restrict__ cpart, float* __restrict__ ugrad, int width, RowApply ra) {
    const int nu = *d_nuniq;
    const int lane = threadIdx.x & 31;
    const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t it = 0; it * 32 * nw < nu; ++it) {
        const int64_t u = (it * 32 + lane) * nw + w0;
        int c0 = 0, c1 = 0;
        if (u < nu) { c0 = choff[u]; c1 = choff[u + 1]; }
        unsigned multi = __ballot_sync(0xffffffffu, c1 > c0);
        while (multi) {
            const int src = __ffs(multi) - 1;
            multi &= multi - 1;
            const int b0 = __shfl_sync(0xffffffffu, c0, src), b1 = __shfl_sync(0xffffffffu, c1, src);
            const int64_t uu = (it * 32 + src) * nw + w0;          // the unique row being combined
            const int G = width >> 2;
            if (width >= 4 && (G & (G - 1)) == 0 && G <= 32) {
                // G lanes cover one chunk's row (float4 each), 32/G chunks in flight per step, 4 steps unrolled;
                // fixed-order tree over the chunk groups
                const int lq = lane % G, cg = lane / G, NG = 32 / G;
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                int c = b0 + cg;
                for (; c + 3 * NG < b1; c += 4 * NG) {
                    const float4 v0 = *reinterpret_cast<const float4*>(cpart + (int64_t)c * width + lq * 4);
                    const float4 v1 = *reinterpret_cast<const float4*>(cpart + (int64_t)(c + NG) * width + lq * 4);
                    const float4 v2 = *reinterpret_cast<const float4*>(cpart + (int64_t)(c + 2 * NG) * width + lq * 4);
                    const float4 v3 = *reinterpret_cast<const float4*>(cpart + (int64_t)(c + 3 * NG) * width + lq * 4);
                    acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
                    acc.x += v1.x; acc.y += v1.y; acc.z += v1.z; acc.w += v1.w;
                    acc.x += v2.x; acc.y += v2.y; acc.z += v2.z; acc.w += v2.w;
                    acc.x += v3.x; acc.y += v3.y; acc.z += v3.z; acc.w += v3.w;
                }
                for (; c < b1; c += NG) {
                    const float4 v = *reinterpret_cast<const float4*>(cpart + (int64_t)c * width + lq * 4);
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                }
                for (int d = G; d < 32; d <<= 1) {
                    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, d); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, d);
                    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, d); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, d);
                }
                if (KIND == 1) {
                    if (cg == 0) {
                        const int64_t row = ra.urow[uu];
                        const int t = table_of(ra.rec.row_base, ra.rec.ntab, row);
                        const int dim = ra.rec.dim[t];
                        if (lq * 4 < dim) update_record4(ra.o, record(ra.rec, t, ra.urow, uu) + lq * 4, dim, kind_nslots(ra.o.kind), acc);
                    }
                } else if (cg == 0) *reinterpret_cast<float4*>(ugrad + uu * width + lq * 4) = acc;
            } else {
                for (int q = 0; q < width; ++q) {
                    float acc = 0.f;
                    for (int c = b0 + lane; c < b1; c += 32) acc += cpart[(int64_t)c * width + q];
#pragma unroll
                    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
                    if (lane == 0) {
                        if (KIND == 2) update_wide(ra.o, ra.wide + ra.urow[uu], acc);     // width == 1
                        else ugrad[uu * width + q] = acc;
                    }
                }
            }
        }
    }
}

// --------------------------------------------------------------------------------------------- optimizers

// embedding rows: record = [w[dim] | s1[dim] | s2[dim]], tables of rr in row order
__global__ void __launch_bounds__(256) emb_apply_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow,
                                                        const float* __restrict__ ugrad, int width, RowRecords rr, OptParams op) {
    const OptParams o = with_lr_t(op);
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int nu = *d_nuniq;
    const int64_t g0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4 + grp;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    for (int64_t u = g0; u < nu; u += gstep) {
        const int64_t row = urow[u];
        const int t = table_of(rr.row_base, rr.ntab, row);
        const int dim = rr.dim[t], nslots = kind_nslots(o.kind);
        float* rec = record(rr, t, urow, u);
        for (int q = lig; q * 4 < dim; q += 8)
            update_record4(o, rec + q * 4, dim, nslots, *reinterpret_cast<const float4*>(ugrad + (int64_t)u * width + q * 4));
        if (lig == 0) mark_touched(o, row);
    }
}

// wide rows: record {w, s1, s2, -}; also the bias record (dense gradient = sum of dlogit)
__global__ void wide_apply_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow,
                                  const float* __restrict__ ugrad, float4* __restrict__ wide, OptParams op) {
    const OptParams o = with_lr_t(op);
    const int nu = *d_nuniq;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += gridDim.x * blockDim.x) {
        update_wide(o, wide + urow[u], ugrad[u]);
        mark_touched(o, urow[u]);
    }
}

// Adam, untouched pass over the embedding records of one set (adam_untouched_emb): one warp per 32-bit word of the bitmap, i.e. per
// 32 rows; lane groups of 8 take rows grp, grp + 4, ..., each lane float4 chunks lig, lig + 8, ... of the row.  The warp clears the
// word once every row of it has read its bit.
__global__ void __launch_bounds__(256) adam_untouched_emb_kernel(RowRecords rr, const int64_t* __restrict__ rows, int64_t nbits, OptParams op) {
    const OptParams o = with_lr_t(op);
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int64_t nwords = (nbits + 31) >> 5;
    for (int64_t wd = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wd < nwords; wd += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const uint32_t bits = o.touched[wd];
        for (int k = grp; k < 32; k += 4) {
            const int64_t row = wd * 32 + k;
            if (row >= nbits || ((bits >> k) & 1u)) continue;
            const int t = table_of(rr.row_base, rr.ntab, row);
            const int64_t local = row - rr.row_base[t];
            if (local >= rows[t]) continue;                        // (a row-sharded space: past this rank's share of table t)
            const int dim = rr.dim[t];
            float* rec = rr.data[t] + local * rr.stride[t];
            for (int q = lig; q * 4 < dim; q += 8) adam_untouched4(o, rec + q * 4, dim);
        }
        __syncwarp();
        if (lane == 0 && bits) o.touched[wd] = 0u;
    }
}
// ... over the wide records {w, m, v, -}: one thread per row, a warp per word
__global__ void __launch_bounds__(256) adam_untouched_wide_kernel(float4* __restrict__ wide, int64_t nbits, OptParams op) {
    const OptParams o = with_lr_t(op);
    const int64_t npad = (nbits + 31) & ~(int64_t)31;              // warp-uniform trip count
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npad; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t bits = o.touched[i >> 5];
        if (i < nbits && !((bits >> (i & 31)) & 1u)) {
            float4 r = wide[i];
            adam_decay(o, r.y, r.z);
            adam_step(o, r.x, r.y, r.z);
            wide[i] = r;
        }
        __syncwarp();
        if ((i & 31) == 0 && bits) o.touched[i >> 5] = 0u;
    }
}


static int bits_for(int64_t n) {
    int b = 1;
    while ((1ll << b) < n) ++b;
    return b;
}

int list_alloc(WdModel* m, int L, int64_t rows, int width, bool sort_only) {
    RowList& l = m->lists[L];
    const int64_t n = m->max_nnz + 8;
    l.bits = bits_for(rows);
    l.width = width;
    int rc;
    for (uint32_t** p : {&l.keys, &l.vals, &l.keys2, &l.vals2})
        if ((rc = dev_alloc(m, p, n))) return rc;
    if (sort_only) return WD_OK;
    if ((rc = dev_alloc(m, &l.urow, n))) return rc;
    if ((rc = dev_alloc(m, &l.ustart, n))) return rc;
    if ((rc = dev_alloc(m, &l.ugrad, n * width))) return rc;
    if ((rc = dev_alloc(m, &l.nuniq, 4))) return rc;
    if (L < 2 && (rc = dev_alloc(m, &l.nubig, 4))) return rc;     // (only the replicated lists hand rows to the small-table block)
    if ((rc = dev_alloc(m, &l.nvalid, 4))) return rc;
    if ((rc = dev_alloc(m, &l.choff, n))) return rc;
    if ((rc = dev_alloc(m, &l.nchunks, 4))) return rc;
    return dev_alloc(m, &l.cpart, chunk_cap(m->max_nnz) * width);
}

// sort (row, occurrence) pairs by row and find the unique rows; e_row: per-occurrence row ids (kInvalidRow = skip)
static int group_tail(WdModel* m, RowList& l, const int32_t* d_n);
static int group_rows(WdModel* m, RowList& l, const int32_t* d_n, const uint32_t* e_row, const int32_t* val_src = nullptr) {
    int g = grid_for(m->max_nnz, 256);
    sort_keys_kernel<<<g, 256, 0, m->stream>>>(d_n, e_row, 1u << l.bits, l.keys, l.vals, val_src);
    m->launches++;
    int rc = radix_sort_pairs(m, &l.keys, &l.vals, &l.keys2, &l.vals2, l.bits + 1, d_n);
    if (rc) return rc;
    return group_tail(m, l, d_n);
}
// unique rows + segment starts of the sorted (row, occurrence) pairs in keys / vals
static int group_tail(WdModel* m, RowList& l, const int32_t* d_n) {
    int32_t* pos = (int32_t*)l.keys2;                          // ping-pong buffer is free after the sort
    return seg_heads(m, d_n, l.keys, 1u << l.bits, pos, m->max_nnz, l.ustart, l.urow, l.nuniq);
}

// out[u] = sum over the segment of in[sv[j]] (rows of `width` floats); one thread per (unique row, float4 chunk)
__global__ void merged_sum_kernel(const int32_t* __restrict__ d_nuniq, const int32_t* __restrict__ ustart, const uint32_t* __restrict__ svals,
                                  const float* __restrict__ in, float* __restrict__ out, int width) {
    const int nu = *d_nuniq;
    const int64_t total = (int64_t)nu * width;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        int u = (int)(t / width), q = (int)(t % width);
        float acc = 0.f;
        for (int j = ustart[u]; j < ustart[u + 1]; ++j) acc += in[(int64_t)svals[j] * width + q];
        out[t] = acc;
    }
}

__global__ void set_count_kernel(int32_t* dst, int32_t v) { *dst = v; }

// Replace the gradient list `which` by the row-wise sum of an external (rows, grads) list, e.g. the
// all-gathered lists of every rank: keeps "sum duplicates, apply once" across data-parallel replicas.
int merge_sparse(WdModel* m, int which, const void* rows, const void* grads, int64_t n) {
    RowList& l = m->lists[which];
    if (n > m->max_nnz) { set_error("merged sparse list has %lld rows, capacity %lld", (long long)n, (long long)m->max_nnz); return WD_EINVAL; }
    set_count_kernel<<<1, 1, 0, m->stream>>>(l.nvalid, (int32_t)n);     // (a kernel, not a memcpy: capturable into a graph)
    m->launches++;
    int rc = group_rows(m, l, l.nvalid, (const uint32_t*)rows);
    if (rc) return rc;
    merged_sum_kernel<<<grid_for(std::max<int64_t>(n, 1) * l.width, 256), 256, 0, m->stream>>>(l.nuniq, l.ustart, l.vals, (const float*)grads,
                                                                                              l.ugrad, l.width);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// Merge of G lists that are each sorted ascending, duplicate-free and padded with kInvalidRow (what wd_sparse_grads hands out, so
// what a fixed-size all-gather of it yields): no sort — every element finds its position in the stable merged order with one
// binary search per list (own list: its index), one kernel; then the usual unique-row / segment pass and the ordered sums.
__global__ void __launch_bounds__(256) merge_rank_kernel(const uint32_t* __restrict__ rows, int G, int K, uint32_t* __restrict__ keys,
                                                         uint32_t* __restrict__ vals, int32_t* __restrict__ d_nvalid) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int n = 0;
        for (int r = 0; r < G; ++r) n += lower_bound_u32(rows + (int64_t)r * K, K, kInvalidRow);
        *d_nvalid = n;
    }
    const int64_t total = (int64_t)G * K;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t x = rows[e];
        if (x == kInvalidRow) continue;
        const int r = (int)(e / K);
        int pos = (int)(e - (int64_t)r * K);                        // earlier entries of the own list are all smaller
        for (int q = 0; q < G; ++q) {
            if (q == r) continue;
            const uint32_t* lst = rows + (int64_t)q * K;
            pos += q < r ? upper_bound_u32(lst, K, x) : lower_bound_u32(lst, K, x);   // ties: lower list index first (stable)
        }
        keys[pos] = x;
        vals[pos] = (uint32_t)e;
    }
}
// this rank touched more unique rows than the fixed exchange length: its tail was NOT exchanged -> fail the step loudly (flag 8)
__global__ void list_len_check_kernel(const int32_t* __restrict__ d_nuniq, int64_t list_len, int32_t* __restrict__ flags) {
    if ((int64_t)*d_nuniq > list_len) atomicOr(flags, 8);
}
int merge_sparse_sorted(WdModel* m, int which, const void* rows, const void* grads, int n_lists, int64_t list_len) {
    RowList& l = m->lists[which];
    const int64_t n = (int64_t)n_lists * list_len;
    if (n_lists < 1 || list_len < 1 || list_len > 0x7fffffff) { set_error("merge: bad list shape"); return WD_EINVAL; }
    if (n > m->max_nnz) { set_error("merged sparse list has %lld rows, capacity %lld", (long long)n, (long long)m->max_nnz); return WD_EINVAL; }
    list_len_check_kernel<<<1, 1, 0, m->stream>>>(l.nuniq, list_len, m->d_flags);   // (nuniq still holds the local count)
    m->launches++;
    merge_rank_kernel<<<grid_for(n, 256), 256, 0, m->stream>>>((const uint32_t*)rows, n_lists, (int)list_len, l.keys, l.vals, l.nvalid);
    m->launches++;
    int rc = group_tail(m, l, l.nvalid);
    if (rc) return rc;
    merged_sum_kernel<<<grid_for(std::max<int64_t>(n, 1) * l.width, 256), 256, 0, m->stream>>>(l.nuniq, l.ustart, l.vals, (const float*)grads,
                                                                                              l.ugrad, l.width);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// sort + per-row gradient sums for both tables; leaves (urow, ugrad, nuniq) ready for exchange / apply
// Stage 1 of the sparse backward: group the step's (row, occurrence) pairs by row for both table spaces and lay out
// the hot-row chunks.  Depends only on the ids of the batch (not on any gradient), so api.cu runs it on a side stream
// concurrently with the towers' forward/backward.
int sparse_group_which(WdModel* m, int which) {
    int rc;
    RowList& l = m->lists[which];
    const bool present = which == 0 ? (m->use_deep && !m->tables.empty()) : m->use_wide;
    if (present) {
        if ((rc = group_rows(m, l, m->d_nnz, which == 0 ? m->d_e_emb : m->d_e_wide, m->d_e_bc))) return rc;     // values = cell indices
        if ((rc = chunk_offsets(m, l.nuniq, l.ustart, l.urow, l.choff, m->max_nnz, kChunk, l.nchunks))) return rc;
        mark(m, which == 0 ? "emb_group" : "wide_group");
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// Stage 2: per-row gradient sums; leaves (urow, ugrad, nuniq) ready for exchange / apply.
// Single-GPU step (train_eager: nothing exchanges the sums between backward and optimizer) with a row-local optimizer (everything
// but Adam, whose moments decay over whole tables): the rows are updated inside these two launches and sparse_apply_which has
// nothing left to launch for the list (RowList::fused).
static bool fuse_row_apply(const WdModel* m, const WdOptimizer& o) {
    return m->fuse_dense && o.kind != WD_OPT_ADAM && m->gs_count == 0;
}
int sparse_reduce_emb(WdModel* m) {
    const int g = grid_for(m->max_nnz, 256);
    if (m->use_deep && !m->tables.empty()) {
        RowList& l = m->lists[0];
        const int width = l.width, G4 = width >> 2;
        const int ge = grid_for((m->max_nnz + chunk_cap(m->max_nnz)) * 8, 256);
        // the hot rows' update lives in the lane-group branch of chunk_combine_kernel: widths 4, 8, ..., 128
        const bool fused = fuse_row_apply(m, m->dnn_opt) && width >= 4 && (G4 & (G4 - 1)) == 0 && G4 <= 32;
        // the direct rows' records by table in plan order (a sum knows its table from the column), the hot rows' by table in row
        // order; host tables: the fused updates go to the staged records, host_tables_write_back copies them home after the list's apply
        const OptParams o = make_opt(m->dnn_opt);
        const RowApply ra{l.urow, m->tabs.rec, nullptr, o};
        const RowApply ha{l.urow, m->rtabs.rec, nullptr, o};
        const LocalEmb src{l.vals, m->d_col_offs, m->n_columns, m->dplan.col_emb_table, m->tabs.rec.dim, m->tabs.x0, m->d_dX0, m->d0_phys};
        if (fused) {
            emb_grad_sum_kernel<LocalEmb, true><<<ge, 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad, l.cpart, width, ra);
            chunk_combine_kernel<1><<<g, 256, 0, m->stream>>>(l.nuniq, l.choff, l.cpart, l.ugrad, width, ha);
        } else {
            emb_grad_sum_kernel<LocalEmb, false><<<ge, 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad, l.cpart, width, ra);
            chunk_combine_kernel<0><<<g, 256, 0, m->stream>>>(l.nuniq, l.choff, l.cpart, l.ugrad, width, ha);
        }
        l.fused = fused;
        m->launches += 2;
        mark(m, "emb_grad_sum");
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int sparse_reduce_wide(WdModel* m) {
    const int g = grid_for(m->max_nnz, 256);
    if (m->use_wide) {
        RowList& l = m->lists[1];
        const bool fused = fuse_row_apply(m, m->lin_opt);
        const RowApply ra{l.urow, RowRecords{}, m->d_wide, make_opt(m->lin_opt)};
        const LocalWide src{l.vals, m->n_columns, m->d_dlogit};
        const int gw = grid_for(m->max_nnz + chunk_cap(m->max_nnz), 256);
        if (fused) {
            wide_grad_sum_kernel<LocalWide, true><<<gw, 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad, l.cpart, ra);
            chunk_combine_kernel<2><<<g, 256, 0, m->stream>>>(l.nuniq, l.choff, l.cpart, l.ugrad, 1, ra);
        } else {
            wide_grad_sum_kernel<LocalWide, false><<<gw, 256, 0, m->stream>>>(l.nuniq, l.nchunks, l.ustart, l.choff, src, l.ugrad, l.cpart, ra);
            chunk_combine_kernel<0><<<g, 256, 0, m->stream>>>(l.nuniq, l.choff, l.cpart, l.ugrad, 1, ra);
        }
        l.fused = fused;
        m->launches += 2;
        mark(m, "wide_grad_sum");
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// ------------------------------------------------------------------------- dense exchange of small tables
// Rows of the small tables sit at the end of the global row space, so they are the tail of the sorted unique-row list.  Their summed
// gradients move into the dense block behind the dense gradient arena (all-reduced with it in data-parallel runs) and leave the
// list: the tail is overwritten with kInvalidRow and the list length becomes the number of large-table rows.
__global__ void __launch_bounds__(256) small_scatter_emb_kernel(const int32_t* __restrict__ d_nuniq, uint32_t* __restrict__ urow,
                                                                const float* __restrict__ ugrad, int width, uint32_t small_base, int ntab,
                                                                const int64_t* __restrict__ rtab_row_base, const int32_t* __restrict__ rtab_dim,
                                                                const int64_t* __restrict__ rtab_gs_off, float* __restrict__ Gs,
                                                                float* __restrict__ touched, int32_t* __restrict__ d_nubig) {
    const int nu = *d_nuniq;
    const int lb = lower_bound_u32(urow, nu, small_base);        // (a concurrently invalidated tail entry still compares >= small_base)
    if (blockIdx.x == 0 && threadIdx.x == 0) *d_nubig = lb;
    const int lane = threadIdx.x & 31, lig = lane & 7, grp = lane >> 3;
    const int64_t g0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4 + grp;
    const int64_t gstep = (((int64_t)gridDim.x * blockDim.x) >> 5) * 4;
    for (int64_t u = lb + g0; u < nu; u += gstep) {
        const int64_t row = urow[u];
        const int t = table_of(rtab_row_base, ntab, row);
        const int dim = rtab_dim[t];
        float* dst = Gs + rtab_gs_off[t] + (row - rtab_row_base[t]) * dim;
        for (int q = lig; q * 4 < dim; q += 8)
            *reinterpret_cast<float4*>(dst + q * 4) = *reinterpret_cast<const float4*>(ugrad + u * width + q * 4);
        __syncwarp();
        if (lig == 0) {
            touched[row - small_base] = 1.f;                      // "this rank touched the row" (summed over ranks with the block)
            urow[u] = kInvalidRow;
        }
    }
}
__global__ void __launch_bounds__(256) small_scatter_wide_kernel(const int32_t* __restrict__ d_nuniq, uint32_t* __restrict__ urow,
                                                                 const float* __restrict__ ugrad, uint32_t small_base, float* __restrict__ Gs,
                                                                 float* __restrict__ touched, int32_t* __restrict__ d_nubig) {
    const int nu = *d_nuniq;
    const int lb = lower_bound_u32(urow, nu, small_base);
    if (blockIdx.x == 0 && threadIdx.x == 0) *d_nubig = lb;
    for (int64_t u = lb + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < nu; u += (int64_t)gridDim.x * blockDim.x) {
        Gs[urow[u] - small_base] = ugrad[u];
        touched[urow[u] - small_base] = 1.f;
        urow[u] = kInvalidRow;
    }
}
__global__ void copy_count_kernel(int32_t* dst, const int32_t* src) { *dst = *src; }

int small_scatter(WdModel* m, int which) {
    if (m->gs_count == 0) return WD_OK;
    const RowList& l = m->lists[which];
    float* block = m->d_G + m->dense_count;
    if (which == 0) {
        if (m->n_small_tab == 0 || !(m->use_deep && !m->tables.empty())) return WD_OK;
        small_scatter_emb_kernel<<<grid_for(m->max_nnz * 8, 256, kNumSms * 8), 256, 0, m->stream>>>(l.nuniq, l.urow, l.ugrad, l.width,
            (uint32_t)m->small_base[0], m->rtabs.rec.ntab, m->rtabs.rec.row_base, m->rtabs.rec.dim, m->rtabs.gs_off, block,
            block + m->gs_touch_off[0], l.nubig);
    } else {
        if (!m->use_wide || m->small_base[1] >= m->wide_rows) return WD_OK;
        small_scatter_wide_kernel<<<grid_for(m->max_nnz, 256, kNumSms * 8), 256, 0, m->stream>>>(l.nuniq, l.urow, l.ugrad,
            (uint32_t)m->small_base[1], block + m->gs_emb_floats, block + m->gs_touch_off[1], l.nubig);
    }
    copy_count_kernel<<<1, 1, 0, m->stream>>>(l.nuniq, l.nubig);
    m->launches += 2;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

// optimizer over the dense block: one update per small-table row that ANY rank touched this step.  "Touched" travels with the
// block as a per-row count (summed by the same all-reduce), not as "gradient != 0": a touched row whose summed gradient is
// exactly zero (saturated sigmoids give dlogit == 0.0) still takes its optimizer step in TensorFlow — FTRL then rebuilds w from
// (z, n) and RMSProp decays its mean square.
__global__ void __launch_bounds__(256) small_apply_emb_kernel(const float* __restrict__ Gs, const float* __restrict__ touched, int64_t n4, int ntab,
                                                              int first_small, int64_t small_base, const int64_t* __restrict__ rtab_row_base,
                                                              const int64_t* __restrict__ rtab_gs_off, float* const* __restrict__ rtab_data,
                                                              const int32_t* __restrict__ rtab_dim, const int32_t* __restrict__ rtab_stride, OptParams op) {
    const OptParams o = with_lr_t(op);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        // small tables are the last entries, offsets ascending
        const int t = first_small + table_of(rtab_gs_off + first_small, ntab - first_small, i * 4);
        const int dim = rtab_dim[t], stride = rtab_stride[t];
        const int64_t local = i * 4 - rtab_gs_off[t];
        if (touched[rtab_row_base[t] - small_base + local / dim] == 0.f) continue;
        const float4 g = *reinterpret_cast<const float4*>(Gs + i * 4);
        update_record4(o, rtab_data[t] + (local / dim) * stride + (local % dim), dim, kind_nslots(o.kind), g);
        if (local % dim == 0) mark_touched(o, rtab_row_base[t] + local / dim);
    }
}
// (wide: the small wide rows from global row row0)
__global__ void __launch_bounds__(256) small_apply_wide_kernel(const float* __restrict__ Gs, const float* __restrict__ touched, int64_t n,
                                                               float4* __restrict__ wide, int64_t row0, OptParams op) {
    const OptParams o = with_lr_t(op);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (touched[i] == 0.f) continue;
        update_wide(o, wide + row0 + i, Gs[i]);
        mark_touched(o, row0 + i);
    }
}
int small_apply(WdModel* m) {
    if (m->gs_count == 0) return WD_OK;
    const float* block = m->d_G + m->dense_count;
    if (m->gs_emb_floats > 0) {
        const RecordSet& rs = m->rtabs;
        small_apply_emb_kernel<<<grid_for(m->gs_emb_floats / 4, 256), 256, 0, m->stream>>>(block, block + m->gs_touch_off[0], m->gs_emb_floats / 4, rs.rec.ntab,
            rs.rec.ntab - m->n_small_tab, m->small_base[0], rs.rec.row_base, rs.gs_off, rs.rec.data, rs.rec.dim, rs.rec.stride,
            space_opt(m, 0, m->d_adam_touched[0]));
        m->launches++;
    }
    const int64_t nw = m->use_wide ? m->wide_rows - m->small_base[1] : 0;
    if (nw > 0) {
        small_apply_wide_kernel<<<grid_for(nw, 256), 256, 0, m->stream>>>(block + m->gs_emb_floats, block + m->gs_touch_off[1], nw,
            m->d_wide, m->small_base[1], space_opt(m, 1, m->d_adam_touched[1]));
        m->launches++;
    }
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

OptParams space_opt(const WdModel* m, int space, uint32_t* touched) {
    const WdOptimizer& o = space == 0 ? m->dnn_opt : m->lin_opt;
    const bool adam = o.kind == WD_OPT_ADAM;
    return make_opt(o, adam ? m->d_bpow + (space == 0 ? 2 : 0) : nullptr, adam ? touched : nullptr);
}
// the records of a set in place, none staged (the unfused updates write host records through their mapped pointers)
static RowRecords in_place(RowRecords r) {
    r.stage = nullptr;
    return r;
}

int sparse_apply_which(WdModel* m, int which) {
    int rc;
    RowList& l = m->lists[which];
    // rows already updated by the gradient-sum / combine launches of this step (single-GPU step)
    const bool done = l.fused;
    l.fused = false;
    // the fused updates of host-table rows went to their staged copies: copy those home (the unfused kernels below update host
    // records in place, through their mapped pointers)
    if (done) return (which == 0 && m->n_host_tab > 0) ? host_tables_write_back(m) : WD_OK;
    // deferred Adam host tables (the only host tables Adam allows): their rows were staged and caught up by this step's stage-in,
    // so the update goes to the staged records, which then go home as after the fused updates
    if (which == 0 && m->n_host_tab > 0 && m->dnn_opt.kind == WD_OPT_ADAM) {
        if ((rc = list_apply_emb(m, l, m->rtabs.rec, space_opt(m, 0, m->d_adam_touched[0])))) return rc;
        return host_tables_write_back(m);
    }
    if (which == 0 && m->hcache.slots > 0) {       // the unfused updates below would write host records behind the cache's back
        set_error("embedding rows of a model with a host-table cache are only updated by the fused single-GPU step");
        return WD_EUNSUPPORTED;
    }
    if (which == 0 && m->use_deep && !m->tables.empty() && (rc = list_apply_emb(m, l, in_place(m->rtabs.rec), space_opt(m, 0, m->d_adam_touched[0]))))
        return rc;
    if (which == 1 && m->use_wide && (rc = list_apply_wide(m, l, m->d_wide, space_opt(m, 1, m->d_adam_touched[1])))) return rc;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
// ---- wrappers used by shard.cu (rows this rank owns in a row-sharded table space)
// stable sort of (e_key[i], i) pairs, i < *d_n, by key; keys equal to kInvalidRow sort last; result in the list's keys / vals
int list_sort_by_key(WdModel* m, RowList& l, const int32_t* d_n, const uint32_t* e_key) {
    sort_keys_kernel<<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(d_n, e_key, 1u << l.bits, l.keys, l.vals, nullptr);
    m->launches++;
    return radix_sort_pairs(m, &l.keys, &l.vals, &l.keys2, &l.vals2, l.bits + 1, d_n);
}
int list_group(WdModel* m, RowList& l, const int32_t* d_n, const uint32_t* e_row) {
    int rc = group_rows(m, l, d_n, e_row);
    if (rc) return rc;
    if ((rc = chunk_offsets(m, l.nuniq, l.ustart, l.urow, l.choff, m->max_nnz, kChunk, l.nchunks))) return rc;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int list_chunk_combine(WdModel* m, const RowList& l) {
    chunk_combine_kernel<0><<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(l.nuniq, l.choff, l.cpart, l.ugrad, l.width, RowApply{});
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int list_apply_emb(WdModel* m, const RowList& l, const RowRecords& rec, const OptParams& o) {
    emb_apply_kernel<<<grid_for(m->max_nnz * 8, 256), 256, 0, m->stream>>>(l.nuniq, l.urow, l.ugrad, l.width, rec, o);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int list_apply_wide(WdModel* m, const RowList& l, float4* wide, const OptParams& o) {
    wide_apply_kernel<<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(l.nuniq, l.urow, l.ugrad, wide, o);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int adam_untouched_emb(WdModel* m, const RecordSet& set, int64_t nbits, const OptParams& o) {
    if (o.kind != WD_OPT_ADAM || set.rec.ntab == 0 || nbits <= 0) return WD_OK;
    adam_untouched_emb_kernel<<<grid_for(nbits, 256), 256, 0, m->stream>>>(in_place(set.rec), set.rows, nbits, o);    // (a warp per 32 rows)
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int adam_untouched_wide(WdModel* m, float4* wide, int64_t nbits, const OptParams& o) {
    if (o.kind != WD_OPT_ADAM || nbits <= 0) return WD_OK;
    adam_untouched_wide_kernel<<<grid_for(nbits, 256), 256, 0, m->stream>>>(wide, nbits, o);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
// Adam, the untouched passes of the replicated record sets: after both their lists and the dense block's small-table rows
int adam_untouched_replicated(WdModel* m) {
    int rc;
    if (m->use_deep && (rc = adam_untouched_emb(m, m->rtabs, m->emb_total_rows, space_opt(m, 0, m->d_adam_touched[0]))))
        return rc;
    return m->use_wide ? adam_untouched_wide(m, m->d_wide, m->wide_rows, space_opt(m, 1, m->d_adam_touched[1])) : WD_OK;
}

}  // namespace wd
