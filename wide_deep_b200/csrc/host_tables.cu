// Embedding tables in page-locked host memory (WdPlanDesc::table_placement).  The reference keeps its tables in host RAM: it
// trains on the CPU or spreads them over parameter servers (reference python/lib/build_estimator.py:211-214, joint.py:141-143).
//
// A host table's [w | slots] records live in mapped, page-locked host memory.  Every step already sorts its embedding ids into the
// unique-row list urow[0] / ustart[0] (sparse_group_which), and every touched row takes exactly one optimizer update, so one step
// moves exactly one record per unique host row each way over PCIe:
//   stage-in    host_rows_kernel<true>: record of unique row u (host tables only) -> HBM staging buffer row u
//   remap       host_remap_kernel: the gather reads ids in which a host-table entry carries u instead of its global row; the
//               gather kernels see the host tables as (data = staging buffer, row base 0, stride = staging stride)
//   apply       the fused updates (RowApply / HotApply in sparse.cu) address the staged record of u
//   write-back  host_rows_kernel<false>: staging buffer row u -> host record, after the list's apply, on its stream
// Every kernel downstream of the stage-in runs on bit-identical values in the same order, so the result equals the HBM-resident
// model's bit for bit.  Updates that do not go through the fused kernels (data-parallel lists: wd_step_backward + wd_step_apply)
// address the host records directly through their mapped pointers.
#include <algorithm>

#include "common.cuh"
#include "sparse_dev.cuh"

namespace wd {

// table (index in row order) of a global embedding row: tables are few, binary search over their row bases
__device__ __forceinline__ int rtab_of(const int64_t* __restrict__ rtab_row_base, int ntab, int64_t row) {
    int lo = 0, hi = ntab - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (rtab_row_base[mid] <= row) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// IN: host record of unique row u -> stage + u * S; !IN: the reverse.  One thread per float4 of a staged record, consecutive
// threads on consecutive float4 of a record (the PCIe transfers are whole records); each thread keeps kInFlight float4 in flight.
constexpr int kInFlight = 4;
template <bool IN>
__global__ void __launch_bounds__(256) host_rows_kernel(const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow, int ntab,
                                                        const int64_t* __restrict__ rtab_row_base, float* const* __restrict__ rtab_data,
                                                        const int32_t* __restrict__ rtab_stride, const int32_t* __restrict__ rtab_stage,
                                                        float* __restrict__ stage, int S) {
    const int q4 = S >> 2;
    const int64_t total = (int64_t)*d_nuniq * q4;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += T * kInFlight) {
        float4 v[kInFlight];
        float* dst[kInFlight];
#pragma unroll
        for (int k = 0; k < kInFlight; ++k) {
            dst[k] = nullptr;
            const int64_t i = i0 + k * T;
            if (i >= total) continue;
            const int64_t u = i / q4;
            const int q = (int)(i - u * q4);
            const int64_t row = urow[u];
            const int lo = rtab_of(rtab_row_base, ntab, row);
            const int stride = rtab_stride[lo];
            if (rtab_stage[lo] == 0 || q * 4 >= stride) continue;          // HBM table / beyond this table's record
            float* rec = rtab_data[lo] + (row - rtab_row_base[lo]) * stride + q * 4;
            float* st = stage + u * S + q * 4;
            if (IN) { v[k] = *reinterpret_cast<const float4*>(rec); dst[k] = st; }
            else { v[k] = *reinterpret_cast<const float4*>(st); dst[k] = rec; }
        }
#pragma unroll
        for (int k = 0; k < kInFlight; ++k)
            if (dst[k]) *reinterpret_cast<float4*>(dst[k]) = v[k];
    }
}

// gather ids: e_emb, with the entries of host tables replaced by their unique-row index u (urow[0..nu) is sorted ascending)
__global__ void __launch_bounds__(256) host_remap_kernel(const int32_t* __restrict__ d_nnz, const uint32_t* __restrict__ e_emb,
                                                         const int32_t* __restrict__ d_nuniq, const uint32_t* __restrict__ urow, int ntab,
                                                         const int64_t* __restrict__ rtab_row_base, const int32_t* __restrict__ rtab_stage,
                                                         uint32_t* __restrict__ g_emb) {
    const int n = *d_nnz, nu = *d_nuniq;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t r = e_emb[i];
        uint32_t g = r;
        if (r != kInvalidRow && rtab_stage[rtab_of(rtab_row_base, ntab, r)] != 0) g = (uint32_t)lower_bound_u32(urow, nu, r);
        g_emb[i] = g;
    }
}

int host_tables_stage_in(WdModel* m) {
    host_rows_kernel<true><<<grid_for(m->max_nnz * (m->stage_stride / 4) / kInFlight, 256), 256, 0, m->stream>>>(
        m->d_nuniq[0], m->d_urow[0], m->n_rtab, m->d_rtab_row_base, m->d_rtab_data, m->d_rtab_stride, m->d_rtab_stage, m->d_stage, m->stage_stride);
    host_remap_kernel<<<grid_for(m->max_nnz, 256), 256, 0, m->stream>>>(m->d_nnz, m->d_e_emb, m->d_nuniq[0], m->d_urow[0], m->n_rtab,
                                                                        m->d_rtab_row_base, m->d_rtab_stage, m->d_g_emb);
    m->launches += 2;
    mark(m, "stage_in");
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int host_tables_write_back(WdModel* m) {
    host_rows_kernel<false><<<grid_for(m->max_nnz * (m->stage_stride / 4) / kInFlight, 256), 256, 0, m->stream>>>(
        m->d_nuniq[0], m->d_urow[0], m->n_rtab, m->d_rtab_row_base, m->d_rtab_data, m->d_rtab_stride, m->d_rtab_stage, m->d_stage, m->stage_stride);
    m->launches++;
    mark(m, "write_back");
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

template <typename T>
static int upload(WdModel* m, T** dst, const std::vector<T>& h) {
    int rc = dev_alloc(m, dst, (int64_t)h.size(), false);
    if (rc) return rc;
    WD_CUDA(cudaMemcpyAsync(*dst, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, m->stream));
    return WD_OK;
}
template <typename T>
static int overwrite(WdModel* m, T* dst, const std::vector<T>& h) {
    WD_CUDA(cudaMemcpyAsync(dst, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, m->stream));
    return WD_OK;
}

// Allocates every embedding table — in HBM (WD_PLACE_HBM, and WD_PLACE_AUTO tables while they fit, largest first, with
// `hbm_reserve` bytes held back for the buffers allocated after wd_model_create) or in mapped page-locked host memory — and fills
// in the table pointers of the descriptors build_model uploaded, plus the staging buffer and the gather / apply descriptors of the
// host tables.
int place_tables(WdModel* m, int64_t hbm_reserve) {
    const int nt = (int)m->tables.size();
    const bool host_ok = m->shard.world <= 1 && m->dense_exchange_max_rows <= 0 && m->dnn_opt.kind != WD_OPT_ADAM;
    for (int t = 0; t < nt; ++t)
        if (m->tables[t].place == WD_PLACE_HOST && !host_ok) {
            set_error("table %d: host placement is not supported with row-sharded tables, dense_exchange_max_rows > 0 or the Adam "
                      "dnn optimizer (its sparse update decays the whole table every step)", t);
            return WD_EUNSUPPORTED;
        }
    auto bytes_of = [&](int t) { return m->tables[t].arows * (int64_t)m->tables[t].stride * 4; };
    int rc;
    std::vector<int> autos;
    for (int t = 0; t < nt; ++t) {
        EmbTable& tb = m->tables[t];
        tb.host = tb.place == WD_PLACE_HOST;
        if (tb.place == WD_PLACE_AUTO && host_ok) autos.push_back(t);
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
        m->n_host_tab++;
        m->stage_stride = std::max(m->stage_stride, tb.stride);
    }

    // table pointers of the descriptors build_model uploaded before the tables existed
    std::vector<float*> data(nt), rdata;
    for (int t = 0; t < nt; ++t) data[t] = m->tables[t].data;
    for (int t : m->rtab_order) rdata.push_back(m->tables[t].data);
    if ((rc = overwrite(m, m->d_tab_data, data))) return rc;
    if (!rdata.empty() && (rc = overwrite(m, m->d_rtab_data, rdata))) return rc;
    // what the gather kernels / fused updates address: host tables through the staging buffer
    std::vector<float*> gdata(data), rgdata(rdata);
    std::vector<int32_t> gstride(nt), stage(nt, 0), rstage;
    std::vector<int64_t> grb(nt);
    for (int t = 0; t < nt; ++t) {
        const EmbTable& tb = m->tables[t];
        gstride[t] = tb.host ? m->stage_stride : tb.stride;
        grb[t] = tb.host ? 0 : tb.row_base;
        stage[t] = tb.host ? m->stage_stride : 0;
    }
    for (size_t i = 0; i < m->rtab_order.size(); ++i) {
        const bool h = m->tables[m->rtab_order[i]].host;
        rstage.push_back(h ? m->stage_stride : 0);
    }
    if (m->n_host_tab > 0) {
        if ((rc = dev_alloc(m, &m->d_stage, m->max_nnz * (int64_t)m->stage_stride, true))) return rc;
        if ((rc = dev_alloc(m, &m->d_g_emb, m->max_nnz, true))) return rc;
        for (int t = 0; t < nt; ++t) if (m->tables[t].host) gdata[t] = m->d_stage;
        for (size_t i = 0; i < m->rtab_order.size(); ++i) if (rstage[i]) rgdata[i] = m->d_stage;
        if ((rc = upload(m, &m->d_gtab_data, gdata))) return rc;
        if ((rc = upload(m, &m->d_gtab_stride, gstride))) return rc;
        if ((rc = upload(m, &m->d_gtab_row_base, grb))) return rc;
        if ((rc = upload(m, &m->d_tab_stage, stage))) return rc;
        if ((rc = upload(m, &m->d_rtab_gdata, rgdata))) return rc;
        if ((rc = upload(m, &m->d_rtab_stage, rstage))) return rc;
    } else {                                 // nothing on the host: the step addresses the tables' own arrays
        m->d_g_emb = m->d_e_emb;
        m->d_gtab_data = m->d_tab_data; m->d_gtab_stride = m->d_tab_stride; m->d_gtab_row_base = m->d_tab_row_base;
        m->d_rtab_gdata = m->d_rtab_data;
    }
    for (int i = 0; i < m->n_dims; ++i) {    // per-width descriptors of the short-bag gather (table ids ascending, as build_model)
        std::vector<TabDesc> descs;
        for (int t = 0; t < nt; ++t) {
            const EmbTable& tb = m->tables[t];
            if (tb.dim != m->dims[i] || tb.sharded) continue;
            descs.push_back(TabDesc{gdata[t], grb[t], gstride[t], tb.x0_off, tb.col, tb.dim});
        }
        if ((rc = overwrite(m, m->d_dim_desc[i], descs))) return rc;
    }
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

}  // namespace wd
