// Layer summaries of a train step (reference python/lib/utils/model_util.py:15-17 add_layer_summary): per segment of the step's
// layer values, the histogram TensorFlow's SummaryHistoOp builds (tensorflow/core/lib/histogram/histogram.cc, default buckets)
// and the counts behind tf.nn.zero_fraction.
//
// A segment is one tensor the towers produce, read once:
//   deep input X0        [B, d0_phys], only its logical columns (WdModelExtra::x0_real: no table padding, no alignment gap)
//   hidden layer (t, l)  [B, N], rebuilt from the post-activation values A: dropout multiplier and BN affine of this step
//                        (drop_mult / bn_out, shared with the forward), so it equals the fp32 layer output H bit for bit
//   tower t's logits     [B]
//   wide logit           [B]
// A summary tag concatenates segments (connected modes, wide_deep_b200/summary.py); the host adds their counts and sums.
//
// One launch per armed step, on the main stream after the head (before any optimizer: the values depend on gamma / beta and on
// the step's dropout key).  A block walks a fixed share of one segment, bins each value (as a double) into a shared-memory
// histogram by binary search over the 1551 limits in shared memory, and adds the histogram to the segment's counts with integer
// atomics.  Sums, sums of squares, min and max leave as per-block partials that wd_summary_read adds in block order: no float
// atomics, the same bytes on every run (DESIGN section 3).
#include <float.h>

#include <algorithm>
#include <memory>

#include "common.cuh"
#include "gemm.cuh"

namespace wd {

// TensorFlow's default histogram limits (histogram.cc InitDefaultBucketsInner): 1e-12 * 1.1^k below 1e20 and DBL_MAX, mirrored,
// with 0 between the halves; ascending
static std::vector<double> default_limits() {
    std::vector<double> pos;
    double v = 1.0e-12;
    while (v < 1.0e20) {
        pos.push_back(v);
        v *= 1.1;
    }
    pos.push_back(DBL_MAX);
    std::vector<double> out;
    for (auto it = pos.rbegin(); it != pos.rend(); ++it) out.push_back(-*it);
    out.push_back(0.0);
    out.insert(out.end(), pos.begin(), pos.end());
    return out;
}

__global__ void __launch_bounds__(kSummaryThreads) summary_stats_kernel(const SummarySeg* __restrict__ segs, int nseg, int B,
                                                                       const double* __restrict__ limits, unsigned long long seed,
                                                                       const unsigned int* __restrict__ step,
                                                                       unsigned long long* __restrict__ counts, double* __restrict__ part,
                                                                       long long* __restrict__ ipart) {
    __shared__ double lim[WD_SUMMARY_BUCKETS];
    __shared__ unsigned int hist[WD_SUMMARY_BUCKETS];
    __shared__ double rs[4][kSummaryThreads / 32];
    __shared__ long long ri[3][kSummaryThreads / 32];
    int s = 0;
    while (s + 1 < nseg && (int)blockIdx.x >= segs[s + 1].blk0) ++s;
    const SummarySeg sg = segs[s];
    for (int i = threadIdx.x; i < WD_SUMMARY_BUCKETS; i += blockDim.x) { lim[i] = limits[i]; hist[i] = 0u; }
    __syncthreads();

    const bool hidden = sg.kind == WD_SEG_HIDDEN;
    const bool drop = hidden && sg.drop_rate > 0.f;
    const unsigned long long key = drop ? drop_key(DropArgs{sg.drop_rate, seed, step, sg.layer_id, sg.drop_row0}) : 0ull;
    const float inv_keep = drop ? 1.f / (1.f - sg.drop_rate) : 1.f;
    double sum = 0.0, sumsq = 0.0, mn = DBL_MAX, mx = -DBL_MAX;
    long long num = 0, zeros = 0, bad = 0;
    const int64_t total = (int64_t)B * sg.cols;
    const int64_t stride = (int64_t)sg.nblk * blockDim.x;
    for (int64_t e = (int64_t)(blockIdx.x - sg.blk0) * blockDim.x + threadIdx.x; e < total; e += stride) {
        const unsigned ue = (unsigned)e, row = ue / (unsigned)sg.cols, col = ue - row * (unsigned)sg.cols;   // (summary_prepare: < 2^31)
        if (sg.mask && !sg.mask[col]) continue;
        float v = sg.ptr[(int64_t)row * sg.ld + col];
        if (hidden) {
            if (drop) v *= drop_mult(key, sg.drop_row0 + row, col, sg.drop_rate, inv_keep);
            v = bn_out(v, sg.gamma, sg.beta, col, sg.bn);
        }
        ++num;
        if (!isfinite(v)) { ++bad; continue; }
        const double d = (double)v;
        sum += d;
        sumsq += d * d;
        mn = fmin(mn, d);
        mx = fmax(mx, d);
        if (d == 0.0) { ++zeros; continue; }          // (+0 and -0: one fixed bucket, added below without contention)
        int lo = 0, hi = WD_SUMMARY_BUCKETS;         // upper_bound: first limit > d
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (lim[mid] > d) hi = mid; else lo = mid + 1;
        }
        atomicAdd(&hist[lo], 1u);
    }
    // block partials in a fixed order: warp butterfly, then the warps in index order
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sumsq += __shfl_xor_sync(0xffffffffu, sumsq, o);
        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        num += __shfl_xor_sync(0xffffffffu, num, o);
        zeros += __shfl_xor_sync(0xffffffffu, zeros, o);
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if (lane == 0) {
        rs[0][w] = sum; rs[1][w] = sumsq; rs[2][w] = mn; rs[3][w] = mx;
        ri[0][w] = num; ri[1][w] = zeros; ri[2][w] = bad;
    }
    __syncthreads();
    unsigned long long* c = counts + (int64_t)s * WD_SUMMARY_BUCKETS;
    for (int i = threadIdx.x; i < WD_SUMMARY_BUCKETS; i += blockDim.x)
        if (hist[i]) atomicAdd(c + i, (unsigned long long)hist[i]);
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0, lo = DBL_MAX, hi = -DBL_MAX;
        long long n = 0, z = 0, nf = 0;
        for (int i = 0; i < kSummaryThreads / 32; ++i) {
            a += rs[0][i]; b += rs[1][i]; lo = fmin(lo, rs[2][i]); hi = fmax(hi, rs[3][i]);
            n += ri[0][i]; z += ri[1][i]; nf += ri[2][i];
        }
        double* p = part + (int64_t)blockIdx.x * 4;
        p[0] = a; p[1] = b; p[2] = lo; p[3] = hi;
        long long* q = ipart + (int64_t)blockIdx.x * 3;
        q[0] = n; q[1] = z; q[2] = nf;
        if (z) atomicAdd(c + kSummaryZeroBucket, (unsigned long long)z);
    }
}

// Segments in wd_summary_segments order: the deep input, then per tower its hidden layers and its logits, then the wide logit.
// Built on first use; every pointer is fixed for the model's life (the arena, the layer buffers, the head's outputs).
int summary_prepare(WdModel* m, const std::vector<uint8_t>& x0_real) {
    if (m->summ) return WD_OK;
    std::unique_ptr<SummaryState> own(new SummaryState());
    SummaryState* S = own.get();
    const int64_t Bm = m->max_batch;
    // blocks of a segment: one per 16 values per thread at the largest batch, at most two waves of the SMs
    auto add = [&](int kind, int tower, int layer, const float* ptr, int ld, int cols) {
        if (Bm * cols >= (1ll << 31)) { set_error("layer summaries: a segment of %lld values", (long long)(Bm * cols)); return WD_EUNSUPPORTED; }
        SummarySeg g{};
        g.kind = kind; g.ptr = ptr; g.ld = ld; g.cols = cols; g.blk0 = S->blocks;
        g.nblk = (int)std::min<int64_t>(std::max<int64_t>((Bm * cols + 16 * kSummaryThreads - 1) / (16 * kSummaryThreads), 1), 2 * kNumSms);
        S->blocks += g.nblk;
        S->h.push_back(g);
        S->kind.push_back(kind); S->tower.push_back(tower); S->layer.push_back(layer);
        return WD_OK;
    };
    int rc;
    if (m->use_deep) {
        if ((rc = add(WD_SEG_DEEP_INPUT, -1, -1, m->d_X0, m->d0_phys, m->d0_phys))) return rc;
        if ((rc = upload(m, &S->d_mask, x0_real.data(), m->d0_phys))) return rc;
        S->h.back().mask = S->d_mask;
        for (size_t t = 0; t < m->towers.size(); ++t) {
            Tower& tw = m->towers[t];
            for (int l = 0; l < tw.n_hidden; ++l) {
                const Layer& L = tw.layers[l];
                if ((rc = add(WD_SEG_HIDDEN, (int)t, l, L.A, L.N_phys, L.N))) return rc;
                SummarySeg& g = S->h.back();
                g.bn = m->batch_norm;
                g.gamma = L.t_gamma >= 0 ? m->d_P + m->dense[L.t_gamma].off : nullptr;
                g.beta = L.t_beta >= 0 ? m->d_P + m->dense[L.t_beta].off : nullptr;
                g.drop_rate = m->dropout_rate;
                g.layer_id = (int)t * 64 + l;                              // as mlp_forward's DropArgs
                g.drop_row0 = drop_row0(m);
            }
            if ((rc = add(WD_SEG_TOWER_LOGITS, (int)t, -1, tw.logit, 1, 1))) return rc;
        }
    }
    if (m->use_wide && (rc = add(WD_SEG_WIDE_LOGIT, -1, -1, m->d_wide_logit, 1, 1))) return rc;
    const int n = (int)S->h.size();
    if ((rc = upload(m, &S->d_seg, S->h))) return rc;
    if ((rc = upload(m, &S->d_limits, default_limits()))) return rc;
    if ((rc = dev_alloc(m, &S->d_counts, (int64_t)n * WD_SUMMARY_BUCKETS))) return rc;
    if ((rc = dev_alloc(m, &S->d_part, (int64_t)S->blocks * 4))) return rc;
    if ((rc = dev_alloc(m, &S->d_ipart, (int64_t)S->blocks * 3))) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    m->summ = own.release();
    return WD_OK;
}

// the statistics of the current train step (armed by wd_summary_arm); main stream, after the head
int summary_launch(WdModel* m) {
    SummaryState* S = m->summ;
    const int n = (int)S->h.size();
    m->summary_armed = false;
    if (n == 0) { m->summary_ready = true; return WD_OK; }
    WD_CUDA(cudaMemsetAsync(S->d_counts, 0, (size_t)n * WD_SUMMARY_BUCKETS * sizeof(unsigned long long), m->stream));
    summary_stats_kernel<<<S->blocks, kSummaryThreads, 0, m->stream>>>(S->d_seg, n, m->dbatch.B, S->d_limits, m->dropout_seed, m->d_step,
                                                                      S->d_counts, S->d_part, S->d_ipart);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    mark(m, "summary");
    m->summary_ready = true;
    return WD_OK;
}
}  // namespace wd

using namespace wd;

extern "C" int wd_summary_limits(double* out, int32_t cap) {
    const std::vector<double> lim = default_limits();
    if (out) {
        if (cap < (int32_t)lim.size()) { set_error("wd_summary_limits: buffer of %d, need %d", cap, (int)lim.size()); return WD_EINVAL; }
        std::copy(lim.begin(), lim.end(), out);
    }
    return (int)lim.size();
}

extern "C" int wd_summary_read(WdModel* m, int64_t* counts, int64_t* ints, double* reals, int32_t n_segments) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    if (!m->summary_ready) { set_error("no armed train step since the last wd_summary_read (wd_summary_arm before the step)"); return WD_ESTATE; }
    SummaryState* S = m->summ;
    const int n = (int)S->h.size();
    if (n_segments != n || !counts || !ints || !reals) { set_error("wd_summary_read: the model has %d segments, caller passed %d", n, n_segments); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    std::vector<double> part((size_t)S->blocks * 4);
    std::vector<long long> ipart((size_t)S->blocks * 3);
    WD_CUDA(cudaMemcpy(counts, S->d_counts, (size_t)n * WD_SUMMARY_BUCKETS * sizeof(int64_t), cudaMemcpyDeviceToHost));
    WD_CUDA(cudaMemcpy(part.data(), S->d_part, part.size() * sizeof(double), cudaMemcpyDeviceToHost));
    WD_CUDA(cudaMemcpy(ipart.data(), S->d_ipart, ipart.size() * sizeof(long long), cudaMemcpyDeviceToHost));
    for (int s = 0; s < n; ++s) {
        const SummarySeg& g = S->h[s];
        double sum = 0.0, sumsq = 0.0, mn = DBL_MAX, mx = -DBL_MAX;
        long long num = 0, zeros = 0, bad = 0;
        for (int b = g.blk0; b < g.blk0 + g.nblk; ++b) {                  // block order: the same sums on every run
            sum += part[4 * b]; sumsq += part[4 * b + 1];
            mn = std::min(mn, part[4 * b + 2]); mx = std::max(mx, part[4 * b + 3]);
            num += ipart[3 * b]; zeros += ipart[3 * b + 1]; bad += ipart[3 * b + 2];
        }
        ints[3 * s] = num; ints[3 * s + 1] = zeros; ints[3 * s + 2] = bad;
        reals[4 * s] = mn; reals[4 * s + 1] = mx; reals[4 * s + 2] = sum; reals[4 * s + 3] = sumsq;
    }
    m->summary_ready = false;
    return WD_OK;
}
