// Parameter initialisation (TensorFlow initialisers) and streaming eval metrics of the binary head.
//   embeddings  truncated_normal(stddev = 1/sqrt(dim))      (embedding_column default initializer, SURVEY A.7)
//   wide        zeros                                       (linear_model, A.7)
//   metrics     accuracy / auc(200 thresholds) / ...        (reference joint.py:402-406 head; SURVEY A.10)
#include "common.cuh"
#include "sparse_dev.cuh"

namespace wd {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
__device__ __forceinline__ float trunc_normal(uint64_t seed, uint64_t idx) {
    for (int attempt = 0; attempt < 16; ++attempt) {
        uint64_t r = splitmix64(seed ^ splitmix64(idx * 16 + attempt));
        float u1 = ((uint32_t)(r >> 40) + 1u) * (1.f / 16777217.f);     // (0,1]
        float u2 = (uint32_t)((r >> 8) & 0xFFFFFF) * (1.f / 16777216.f);
        float z = sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
        if (fabsf(z) <= 2.f) return z;
    }
    return 0.f;
}

__global__ void emb_init_kernel(float* data, int64_t rows, int dim, int dim_logical, int stride, float slot1, uint64_t seed, int random_w) {
    int64_t total = rows * stride;
    float sd = rsqrtf((float)dim_logical);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = i / stride;
        int c = (int)(i % stride);
        float v;
        if (c < dim) v = (random_w && c < dim_logical) ? sd * trunc_normal(seed, r * dim + c) : 0.f;
        else if (c < 2 * dim) v = slot1;
        else v = 0.f;
        data[i] = v;
    }
}
__global__ void wide_init_kernel(float4* w, int64_t rows, float slot1) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x)
        w[i] = make_float4(0.f, slot1, 0.f, 0.f);
}

static uint64_t splitmix64_host(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// random_w = 0: weights zero, optimizer slots at their initial accumulator value (state of a freshly created model,
// so padding entries never see a 0/sqrt(0) update)
int init_sparse_tables(WdModel* m, uint64_t seed, int random_w) {
    float s_dnn = slot1_init(m->dnn_opt);
    for (size_t t = 0; t < m->tables.size(); ++t) {
        auto& tb = m->tables[t];
        // (a shard draws from its own stream: rank r of a sharded table uses seed + 7919 * r)
        emb_init_kernel<<<grid_for(tb.arows * tb.stride, 256, kNumSms * 32), 256, 0, m->stream>>>(tb.data, tb.arows, tb.dim, tb.dim_logical, tb.stride, s_dnn,
                                                                                           splitmix64_host(seed + 1000 + t + (tb.sharded ? 7919ull * m->shard.rank : 0ull)), random_w);
        m->launches++;
    }
    if (m->use_wide && m->wide_rows > 0) {
        float s_lin = slot1_init(m->lin_opt);
        wide_init_kernel<<<grid_for(m->wide_rows, 256, kNumSms * 32), 256, 0, m->stream>>>(m->d_wide, m->wide_rows, s_lin);
        m->launches++;
    }
    if (m->use_wide && m->shard.sp[1].on) {
        float s_lin = slot1_init(m->lin_opt);
        wide_init_kernel<<<grid_for(m->shard.sp[1].local_rows, 256, kNumSms * 32), 256, 0, m->stream>>>(m->shard.sp[1].d_wide, m->shard.sp[1].local_rows, s_lin);
        m->launches++;
    }
    WD_CUDA(cudaGetLastError());
    return host_cache_sync(m, false, true);                     // the host records were rewritten: cached copies are stale
}

// ----------------------------------------------------------------------------------------------- metrics
// accumulator layout (doubles): [0,201) positive-label histogram over the threshold index, [201,402) negative,
// then 8 scalars: sum w, sum w*loss, sum w*label, sum w*pred, sum w*correct, tp, fp, fn (threshold 0.5 <=> logit > 0)
constexpr int kNumThr = 200;
__constant__ float c_thr[kNumThr];

__global__ void __launch_bounds__(256) metrics_kernel(int B, const float* __restrict__ logits, const float* __restrict__ label,
                                                     const float* __restrict__ weight, double* acc) {
    __shared__ double sh[2 * (kNumThr + 1) + 8];
    for (int i = threadIdx.x; i < 2 * (kNumThr + 1) + 8; i += blockDim.x) sh[i] = 0.0;
    __syncthreads();
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
        float x = logits[b], y = label[b], w = weight ? weight[b] : 1.f;
        float p = 1.f / (1.f + expf(-x));
        int lo = 0, hi = kNumThr;                     // k = number of thresholds strictly below p
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (c_thr[mid] < p) lo = mid + 1; else hi = mid;
        }
        atomicAdd(&sh[(y > 0.5f ? 0 : kNumThr + 1) + lo], (double)w);
        float l = fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
        float cls = x > 0.f ? 1.f : 0.f;
        double* s = sh + 2 * (kNumThr + 1);
        atomicAdd(&s[0], (double)w);
        atomicAdd(&s[1], (double)w * l);
        atomicAdd(&s[2], (double)w * y);
        atomicAdd(&s[3], (double)w * p);
        atomicAdd(&s[4], (double)w * (cls == y ? 1.0 : 0.0));
        atomicAdd(&s[5], (double)w * cls * y);
        atomicAdd(&s[6], (double)w * cls * (1.f - y));
        atomicAdd(&s[7], (double)w * (1.f - cls) * y);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * (kNumThr + 1) + 8; i += blockDim.x)
        if (sh[i] != 0.0) atomicAdd(&acc[i], sh[i]);
}

int metrics_setup() {
    float thr[kNumThr];
    thr[0] = (float)(0.0 - 1e-7);
    for (int i = 0; i < kNumThr - 2; ++i) thr[i + 1] = (float)((i + 1) * 1.0 / (kNumThr - 1));
    thr[kNumThr - 1] = (float)(1.0 + 1e-7);
    WD_CUDA(cudaMemcpyToSymbol(c_thr, thr, sizeof(thr)));
    WD_CUDA(cudaDeviceSynchronize());
    return WD_OK;
}

int metrics_accumulate(WdModel* m, int rows) {
    metrics_kernel<<<grid_for(rows, 256, kNumSms), 256, 0, m->stream>>>(rows, m->d_logits, m->dbatch.label, m->dbatch.weight, m->d_metrics);
    m->launches++;
    m->eval_batches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}

int metrics_finish(WdModel* m, const double* acc, double* out) {
    const int H = kNumThr + 1;
    double a[2 * H + 8];
    WD_CUDA(cudaStreamSynchronize(m->stream));
    WD_CUDA(cudaMemcpy(a, acc, sizeof(a), cudaMemcpyDeviceToHost));
    const double eps = 1e-7;
    double P = 0, Nn = 0;
    for (int k = 0; k < H; ++k) { P += a[k]; Nn += a[H + k]; }
    // tp[t] = sum_{k > t} pos[k]  (prediction > threshold t  <=>  t < k)
    double tp[kNumThr], fp[kNumThr];
    double cp = 0, cn = 0;
    for (int t = kNumThr - 1; t >= 0; --t) { cp += a[t + 1]; cn += a[H + t + 1]; tp[t] = cp; fp[t] = cn; }
    double auc = 0, aupr = 0;
    auto rec = [&](int t) { return (tp[t] + eps) / (P + eps); };               // tp + fn = P
    auto fpr = [&](int t) { return fp[t] / (Nn + eps); };                      // fp + tn = N
    auto prec = [&](int t) { return (tp[t] + eps) / (tp[t] + fp[t] + eps); };
    for (int t = 0; t < kNumThr - 1; ++t) {
        auc += (fpr(t) - fpr(t + 1)) * (rec(t) + rec(t + 1)) / 2.0;
        aupr += (rec(t) - rec(t + 1)) * (prec(t) + prec(t + 1)) / 2.0;
    }
    const double* s = a + 2 * H;
    double sw = s[0], lm = sw > 0 ? s[2] / sw : 0;
    out[0] = sw > 0 ? s[4] / sw : 0;                       // accuracy
    out[1] = lm > 1 - lm ? lm : 1 - lm;                    // accuracy_baseline
    out[2] = auc;
    out[3] = aupr;
    out[4] = sw > 0 ? s[1] / sw : 0;                       // average_loss
    out[5] = lm;                                           // label/mean
    out[6] = m->eval_batches > 0 ? s[1] / (double)m->eval_batches : 0;   // loss: mean over batches of the batch sum
    out[7] = (s[5] + s[6]) > 0 ? s[5] / (s[5] + s[6]) : 0; // precision
    out[8] = sw > 0 ? s[3] / sw : 0;                       // prediction/mean
    out[9] = (s[5] + s[7]) > 0 ? s[5] / (s[5] + s[7]) : 0; // recall
    return WD_OK;
}

}  // namespace wd

// ---- Adam's non-slot variables (beta1^t, beta2^t per optimizer) live in device memory so that a replayed CUDA graph advances them
namespace wd {
__global__ void adam_tick_kernel(float* bpow, uint32_t* step, float lb1, float lb2, float db1, float db2, int lin, int dnn) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        if (lin) { bpow[0] *= lb1; bpow[1] *= lb2; }
        if (dnn) { bpow[2] *= db1; bpow[3] *= db2; }
        *step += 1u;
    }
}
__global__ void step_tick_kernel(unsigned int* step) { if (threadIdx.x == 0 && blockIdx.x == 0) *step += 1u; }
int step_tick(WdModel* m) {
    step_tick_kernel<<<1, 32, 0, m->stream>>>(m->d_step);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
int adam_tick(WdModel* m) {
    adam_tick_kernel<<<1, 32, 0, m->stream>>>(m->d_bpow, m->d_adam_step, m->lin_opt.beta1, m->lin_opt.beta2, m->dnn_opt.beta1, m->dnn_opt.beta2,
                                             m->lin_opt.kind == WD_OPT_ADAM, m->dnn_opt.kind == WD_OPT_ADAM);
    m->launches++;
    WD_CUDA(cudaGetLastError());
    return WD_OK;
}
}  // namespace wd

// Restores the optimizers' step count (checkpoint resume): beta^(steps + 1), multiplied up in fp32 exactly as training does.  The
// Adam step count moves too; the stamps of deferred tables' rows stay (the rows then owe the steps in between).
extern "C" int wd_set_opt_step(WdModel* m, int64_t steps) {
    if (!m || steps < 0) { wd::set_error("wd_set_opt_step: bad arguments"); return WD_EINVAL; }
    if (m->n_defer_tab > 0 && steps > 0xFFFFFFFFll) { wd::set_error("wd_set_opt_step: deferred Adam tables stamp rows with 32-bit steps"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    float bp[4] = {m->lin_opt.beta1, m->lin_opt.beta2, m->dnn_opt.beta1, m->dnn_opt.beta2};
    const float b[4] = {m->lin_opt.beta1, m->lin_opt.beta2, m->dnn_opt.beta1, m->dnn_opt.beta2};
    for (int64_t s = 0; s < steps && s < 100000000; ++s)
        for (int i = 0; i < 4; ++i) bp[i] *= b[i];
    WD_CUDA(cudaMemcpyAsync(m->d_bpow, bp, sizeof(bp), cudaMemcpyHostToDevice, m->stream));
    const unsigned int st = (unsigned int)steps;                   // dropout counter
    WD_CUDA(cudaMemcpyAsync(m->d_step, &st, sizeof(st), cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaMemcpyAsync(m->d_adam_step, &st, sizeof(st), cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}
