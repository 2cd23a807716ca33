// C-ABI of libwd_b200 (include/wd_b200.h): model construction from the compiled plan, parameter IO,
// and the orchestration of one train / forward / eval step on the model's stream.
//
// A step replaces one sess.run(train_op) of the reference's Estimator.train loop (reference
// python/train.py:128-133 -> joint.py:81-269): ids -> sparse forward -> towers -> head -> backward ->
// optimizers.  Nothing here falls back to the CPU: without a CUDA device every entry point returns
// WD_ENODEVICE.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <random>

#include "common.cuh"
#include "farmhash.cuh"
#include "sparse_dev.cuh"

namespace wd {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int init_sparse_tables(WdModel* m, uint64_t seed, int random_w);
int refresh_weight_copies(WdModel* m);
int wide_bias_grad(WdModel* m);
int metrics_setup();
int merge_sparse(WdModel* m, int which, const void* rows, const void* grads, int64_t n);
int shard_step(WdModel* m, bool train, int seg);

static int pad_to(int n, int k) { return (n + k - 1) / k * k; }

// sources of each layer input, in concat order (reference dnn.py:92-193); -1 = deep input x
static std::vector<std::vector<int>> layer_sources(int mode, int L) {
    std::vector<std::vector<int>> out;
    for (int l = 0; l < L; ++l) {
        std::vector<int> s;
        if (l == 0) s = {-1};
        else if (mode == WD_MODE_SIMPLE || mode == WD_MODE_LAST_DENSE) s = {l - 1};
        else if (mode == WD_MODE_FIRST_DENSE) s = {l - 1, -1};
        else if (mode == WD_MODE_DENSE) { s.push_back(-1); for (int j = 0; j < l; ++j) s.push_back(j); }
        else { for (int j = l - 1; j >= 0; --j) s.push_back(j); s.push_back(-1); }
        out.push_back(s);
    }
    std::vector<int> last;
    if (L == 0) last = {-1};
    else if (mode == WD_MODE_SIMPLE) last = {L - 1};
    else if (mode == WD_MODE_FIRST_DENSE) last = {L - 1, -1};
    else if (mode == WD_MODE_LAST_DENSE || mode == WD_MODE_DENSE) { last.push_back(-1); for (int j = 0; j < L; ++j) last.push_back(j); }
    else { for (int j = L - 1; j >= 0; --j) last.push_back(j); last.push_back(-1); }
    out.push_back(last);
    return out;
}
}  // namespace wd

using namespace wd;

static int ensure_slot(WdModel* m, int s);

extern "C" const char* wd_last_error(void) { return wd::g_err; }
extern "C" int wd_version(void) { return WD_API_VERSION; }
extern "C" int wd_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
extern "C" uint64_t wd_fingerprint64(const uint8_t* bytes, size_t n) { return wd::fingerprint64(bytes, n); }
extern "C" uint64_t wd_fingerprint_cat64(uint64_t a, uint64_t b) { return wd::fingerprint_cat64(a, b); }

namespace wd { void tc_map_cache_clear(); }

extern "C" int wd_model_destroy(WdModel* m) {
    if (!m) return WD_OK;
    cudaSetDevice(m->device);
    for (cudaStream_t s : m->streams) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (cudaEvent_t e : m->events) cudaEventDestroy(e);
    tc_map_cache_clear();
    for (auto& sl : m->slots) {
        sl.train.destroy();
        sl.bwd.destroy();
        sl.shard.destroy();
        sl.shard_eval.destroy();
    }
    for (auto& g : m->merge_graph) g.destroy();
    tsv_dev_destroy(m);
    const ShardState& S = m->shard;
    if (S.ipc)                                               // the peers' segments wd_shard_connect_ipc mapped
        for (int r = 0; r < S.world; ++r)
            if (r != S.rank && S.peer_seg[r]) cudaIpcCloseMemHandle(S.peer_seg[r]);
    for (const DevAlloc& a : m->allocs) cudaFree(a.p);
    for (void* p : m->host_allocs) cudaFreeHost(p);
    if (m->h_loss_pinned) cudaFreeHost(m->h_loss_pinned);
    delete m->summ;
    delete m;
    return WD_OK;
}

// optimizer slots of the dense arena start at the initial accumulator value everywhere (padding included)
static int init_dense_slots(WdModel* m) {
    if (m->dense_count == 0) return WD_OK;
    std::vector<float> S1(m->dense_count, 0.f);
    for (size_t i = 0; i < m->dense.size(); ++i) {
        const WdOptimizer& o = (m->use_wide && i == 0) ? m->lin_opt : m->dnn_opt;
        float s1 = slot1_init(o);
        int64_t end = i + 1 < m->dense.size() ? m->dense[i + 1].off : m->dense_count;
        for (int64_t j = m->dense[i].off; j < end; ++j) S1[j] = s1;
    }
    WD_CUDA(cudaMemcpyAsync(m->d_S1, S1.data(), S1.size() * 4, cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

static int build_model(const WdPlanDesc* d, WdModel* m) {
    int rc;
    m->use_wide = d->model_type & 1;
    m->use_deep = (d->model_type & 2) != 0;
    m->n_cat_fields = d->n_cat_fields; m->n_dense_fields = d->n_dense_fields; m->n_columns = d->n_columns;
    const int C = d->n_columns;
    m->col_kind.assign(d->col_kind, d->col_kind + C);
    m->col_field.assign(d->col_field, d->col_field + C);
    m->col_buckets.assign(d->col_buckets, d->col_buckets + C);
    m->col_wide_base.assign(d->col_wide_base, d->col_wide_base + C);
    m->col_emb_table.assign(d->col_emb_table, d->col_emb_table + C);
    m->col_ind_off.assign(d->col_ind_off, d->col_ind_off + C);
    m->n_numeric = d->n_numeric;
    m->d0_phys = d->d0_phys; m->wide_rows = d->wide_rows;
    // crelu(z) = [relu(z) | relu(-z)]: the layer is built twice as wide with relu, its kernel / bias columns n + u tied to minus
    // columns n (exact: every product and sum just changes sign); see crelu_fold / crelu_mirror in mlp.cu
    m->crelu = d->activation == WD_ACT_CRELU;
    m->activation = m->crelu ? WD_ACT_RELU : d->activation; m->batch_norm = d->batch_norm;
    m->dropout_rate = d->dropout_rate; m->dropout_seed = d->dropout_seed;
    if (!(m->dropout_rate >= 0.f && m->dropout_rate < 1.f)) { set_error("dnn_dropout %g outside [0, 1)", m->dropout_rate); return WD_EINVAL; }
    m->lin_opt = d->lin_opt; m->dnn_opt = d->dnn_opt;
    m->max_batch = d->max_batch; m->max_batch_pad = pad_to(d->max_batch, 128);
    m->ldt = m->max_batch_pad;
    m->row_tiles = m->max_batch_pad / 128;
    m->gemm_engine = d->gemm_engine == WD_GEMM_AUTO ? WD_GEMM_TC3X : d->gemm_engine;
    m->operands = m->gemm_engine == WD_GEMM_BF16X3 ? kBf16Operands : kFp32Operands;
    const bool fp32_ops = m->operands == kFp32Operands;
    m->dense_exchange_max_rows = d->dense_exchange_max_rows > 0 ? d->dense_exchange_max_rows : 0;
    m->small_base[1] = (m->dense_exchange_max_rows > 0 && d->wide_small_base >= 0 && d->wide_small_base <= d->wide_rows) ? d->wide_small_base : d->wide_rows;
    m->max_nnz = d->max_nnz > 0 ? d->max_nnz : (int64_t)d->max_batch * std::max(C, 1) * 2;
    const int G = d->shard_world > 1 ? d->shard_world : 1;
    m->shard.world = G; m->shard.rank = G > 1 ? d->shard_rank : 0;
    if (G > 1) {
        if (d->shard_rank < 0 || d->shard_rank >= G) { set_error("shard_rank %d outside [0, %d)", d->shard_rank, G); return WD_EINVAL; }
        // as an owner a rank can receive more ids than it routes itself (skewed ids): all per-entry scratch is sized for that
        const int64_t route = d->shard_capacity > 0 ? d->shard_capacity : m->max_nnz;
        const double slack = d->shard_slack >= 1.f ? d->shard_slack : 2.0;
        m->max_nnz = std::max<int64_t>(m->max_nnz, (int64_t)(route * slack));
    }
    m->keys_cap = d->max_keys > 0 ? d->max_keys : (int64_t)d->max_batch * std::max(d->n_cat_fields, 1) * 4;
    if (m->lin_opt.kind == WD_OPT_FTRL && m->lin_opt.lr_power != -0.5f) { set_error("FTRL: only learning_rate_power=-0.5 is supported"); return WD_EUNSUPPORTED; }
    if (m->dnn_opt.kind == WD_OPT_FTRL && m->dnn_opt.lr_power != -0.5f) { set_error("FTRL: only learning_rate_power=-0.5 is supported"); return WD_EUNSUPPORTED; }
    for (int c = 0; c < C; ++c)
        if (d->col_kind[c] == WD_COL_CROSS && d->col_aux_n[c] > 8) { set_error("cross with more than 8 keys"); return WD_EUNSUPPORTED; }

    // ---- plan tables on the device
    DevPlan& p = m->dplan;
    p.n_cat_fields = d->n_cat_fields; p.n_dense_fields = d->n_dense_fields; p.n_columns = C; p.d0_phys = d->d0_phys;
    if ((rc = upload(m, &p.field_is_string, d->cat_field_is_string, d->n_cat_fields))) return rc;
    if ((rc = upload(m, &p.col_kind, d->col_kind, C))) return rc;
    if ((rc = upload(m, &p.col_field, d->col_field, C))) return rc;
    if ((rc = upload(m, &p.col_buckets, d->col_buckets, C))) return rc;
    if ((rc = upload(m, &p.col_aux_off, d->col_aux_off, C))) return rc;
    if ((rc = upload(m, &p.col_aux_n, d->col_aux_n, C))) return rc;
    if ((rc = upload(m, &p.col_norm_kind, d->col_norm_kind, C))) return rc;
    if ((rc = upload(m, &p.col_norm_a, d->col_norm_a, C))) return rc;
    if ((rc = upload(m, &p.col_norm_b, d->col_norm_b, C))) return rc;
    if ((rc = upload(m, &p.col_wide_base, d->col_wide_base, C))) return rc;
    if ((rc = upload(m, &p.col_emb_table, d->col_emb_table, C))) return rc;
    if ((rc = upload(m, &p.col_ind_off, d->col_ind_off, C))) return rc;
    if ((rc = upload(m, &p.vocab_fp, d->vocab_fp, d->n_vocab_fp))) return rc;
    if ((rc = upload(m, &p.boundaries, d->boundaries, d->n_boundaries))) return rc;
    if ((rc = upload(m, &p.cross_key_type, d->cross_key_type, d->n_cross_keys))) return rc;
    if ((rc = upload(m, &p.cross_key_idx, d->cross_key_idx, d->n_cross_keys))) return rc;
    if ((rc = upload(m, &m->d_num_field, d->num_field, d->n_numeric))) return rc;
    if ((rc = upload(m, &m->d_num_norm_kind, d->num_norm_kind, d->n_numeric))) return rc;
    if ((rc = upload(m, &m->d_num_x0_off, d->num_x0_off, d->n_numeric))) return rc;
    if ((rc = upload(m, &m->d_num_a, d->num_norm_a, d->n_numeric))) return rc;
    if ((rc = upload(m, &m->d_num_b, d->num_norm_b, d->n_numeric))) return rc;

    // ---- batch slot 0
    const int64_t Bm = m->max_batch;
    if ((rc = ensure_slot(m, 0))) return rc;
    if ((rc = dev_alloc(m, &m->d_col_offs, Bm * std::max(C, 1) + 2))) return rc;
    if ((rc = dev_alloc(m, &m->d_e_wide, m->max_nnz))) return rc;
    if ((rc = dev_alloc(m, &m->d_e_emb, m->max_nnz))) return rc;
    if ((rc = dev_alloc(m, &m->d_e_bc, m->max_nnz))) return rc;
    if ((rc = dev_alloc(m, &m->d_e_id, m->max_nnz))) return rc;
    if ((rc = dev_alloc(m, &m->d_nnz, 4))) return rc;
    if ((rc = dev_alloc(m, &m->d_flags, 4))) return rc;
    m->sort_hist_cap = 1024 * ((m->max_nnz + kSortTile - 1) / kSortTile + 1) + 4 * 1024 + 64;
    for (SortScratch& sc : m->scratch) {
        if ((rc = dev_alloc(m, &sc.counter, 4))) return rc;
        if ((rc = dev_alloc(m, &sc.scan, std::max<int64_t>(Bm * std::max(C, 1) + 2, m->max_nnz + 2) / 4096 + 8))) return rc;
        if ((rc = dev_alloc(m, &sc.hist, m->sort_hist_cap))) return rc;
    }
    if ((rc = dev_alloc(m, &m->d_logits, Bm))) return rc;
    if (G == 1 && (rc = dev_alloc(m, &m->d_dlogit, Bm))) return rc;
    if ((rc = dev_alloc(m, &m->d_loss_part, 512))) return rc;
    if ((rc = dev_alloc(m, &m->d_loss, 4))) return rc;
    if ((rc = dev_alloc(m, &m->d_head_counter, 4))) return rc;
    if (getenv("WD_STEP_TRACE") && (rc = dev_alloc(m, &m->d_step_trace, 16))) return rc;
    if ((rc = dev_alloc(m, &m->d_step, 4))) return rc;
    if ((rc = dev_alloc(m, &m->d_bpow, 4))) return rc;
    if ((rc = dev_alloc(m, &m->d_adam_step, 1))) return rc;
    {
        const float bp[4] = {m->lin_opt.beta1, m->lin_opt.beta2, m->dnn_opt.beta1, m->dnn_opt.beta2};     // beta^1: state before the first step
        WD_CUDA(cudaMemcpyAsync(m->d_bpow, bp, sizeof(bp), cudaMemcpyHostToDevice, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
    }
    if (G == 1 && (rc = dev_alloc(m, &m->d_metrics, kMetricsDoubles))) return rc;   // (sharded: in the exchange segment, shard_build)
    WD_CUDA(cudaMallocHost(&m->h_loss_pinned, 64));

    // ---- dense tensors
    auto add_dense = [&](int rows, int cols, int gparts, int g_rowtiles, int64_t gstride, bool transpose) {
        DenseTensor t{};
        t.off = m->dense_count; t.count = (int64_t)rows * cols; t.rows = rows; t.cols = cols;
        t.gpart_off = m->gpart_count; t.gparts = gparts; t.g_rowtiles = g_rowtiles; t.gstride = gstride;
        t.wt_off = transpose ? m->wt_count : -1;
        m->dense_count += (t.count + 3) / 4 * 4;
        m->gpart_count += (int64_t)gparts * gstride;
        if (transpose) m->wt_count += t.count;
        m->dense.push_back(t);
        return (int)m->dense.size() - 1;
    };
    if (m->use_wide) {
        add_dense(1, 1, m->row_tiles, 1, 4, false);            // [0] wide bias
        if ((rc = dev_alloc(m, &m->d_wide, m->wide_rows))) return rc;
        if (m->lin_opt.kind == WD_OPT_ADAM && (rc = dev_alloc(m, &m->d_adam_touched[1], (m->wide_rows + 31) / 32))) return rc;
        if ((rc = dev_alloc(m, &m->d_wide_logit, Bm))) return rc;
    }

    // ---- deep part
    m->x0_real.assign(std::max(d->d0_phys, 1), 0);
    if (m->use_deep) {
        int64_t row_base = 0;
        const int nslots = opt_nslots(m->dnn_opt);
        for (int t = 0; t < d->n_tables; ++t) {
            EmbTable tb{};
            tb.rows = d->table_rows[t]; tb.dim = d->table_dim[t]; tb.x0_off = d->table_x0_off[t];
            tb.dim_logical = d->table_dim_logical[t];
            if (tb.dim_logical < 1 || tb.dim_logical > tb.dim) { set_error("table %d: bad logical width", t); return WD_EINVAL; }
            const int place = d->table_placement ? d->table_placement[t] : WD_PLACE_HBM;
            tb.place = place & ~WD_PLACE_DEFER_ADAM;
            if (tb.place < WD_PLACE_HBM || tb.place > WD_PLACE_AUTO) { set_error("table %d: placement %d is not a WD_PLACE_*", t, place); return WD_EINVAL; }
            tb.defer = (place & WD_PLACE_DEFER_ADAM) && tb.place != WD_PLACE_HBM && m->dnn_opt.kind == WD_OPT_ADAM;
            tb.row_base = 0; tb.gs_off = -1; tb.stride = tb.dim * (1 + nslots) + (tb.defer ? 4 : 0); tb.col = -1;
            tb.sharded = G > 1 && d->table_sharded && d->table_sharded[t];
            tb.arows = tb.sharded ? (tb.rows - m->shard.rank + G - 1) / G : tb.rows;
            if (tb.dim % 4 || tb.x0_off % 4) { set_error("table %d: dim and deep-input offset must be multiples of 4", t); return WD_EINVAL; }
            for (int c = 0; c < C; ++c) if (d->col_emb_table[c] == t) tb.col = c;
            if (tb.col < 0) { set_error("table %d has no producing column", t); return WD_EINVAL; }
            tb.data = nullptr;                                       // allocated by place_tables, after every other buffer of the model
            for (int i = 0; i < tb.dim_logical; ++i) m->x0_real[tb.x0_off + i] = 1;
            m->emb_max_dim = std::max(m->emb_max_dim, tb.dim);
            m->tables.push_back(tb);
        }
        // global row space: large tables first, then the small (dense-exchanged) ones, each group in table order; the small ones'
        // gradients in the same order in the small-table block
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 1) m->small_base[0] = row_base;
            for (int t = 0; t < d->n_tables; ++t) {
                EmbTable& tb = m->tables[t];
                if (tb.sharded) continue;                            // rows live in the sharded space (shard.cu), not here
                const bool small = m->dense_exchange_max_rows > 0 && tb.rows <= m->dense_exchange_max_rows;
                if (small != (pass == 1)) continue;
                if (small) {
                    m->n_small_tab++;
                    tb.gs_off = m->gs_emb_floats;
                    m->gs_emb_floats += tb.rows * tb.dim;
                }
                tb.row_base = row_base;
                row_base += tb.rows;
                m->rtab_order.push_back(t);
            }
        }
        m->emb_total_rows = row_base;
        if (m->dnn_opt.kind == WD_OPT_ADAM && (rc = dev_alloc(m, &m->d_adam_touched[0], (row_base + 31) / 32))) return rc;
        if (row_base >= (1ll << 31)) { set_error("more than 2^31 embedding rows on one device"); return WD_EUNSUPPORTED; }
        for (int i = 0; i < d->n_numeric; ++i) m->x0_real[d->num_x0_off[i]] = 1;
        for (int c = 0; c < C; ++c)
            if (d->col_ind_off[c] >= 0) for (int64_t i = 0; i < d->col_buckets[c]; ++i) m->x0_real[d->col_ind_off[c] + i] = 1;
        for (auto v : m->x0_real) m->d0_logical += v;
        const int nt = (int)m->tables.size();
        // group the replicated tables by width (the gather view, build_record_sets)
        for (int t = 0; t < nt; ++t) {
            if (m->tables[t].sharded) continue;                      // gathered by their owners, not by the local gather kernels
            int di = -1;
            for (int i = 0; i < m->n_dims; ++i) if (m->dims[i] == m->tables[t].dim) di = i;
            if (di < 0) {
                if (m->n_dims == kMaxDims) { set_error("more than %d distinct embedding widths", kMaxDims); return WD_EUNSUPPORTED; }
                di = m->n_dims++; m->dims[di] = m->tables[t].dim; m->dim_ntables[di] = 0;
            }
            m->dim_ntables[di]++;
        }
        const int64_t actn = (int64_t)m->max_batch_pad * d->d0_phys;
        if ((rc = dev_alloc(m, &m->d_X0, actn))) return rc;
        if (fp32_ops && (rc = dev_alloc(m, &m->d_X0T, actn))) return rc;
        if (G == 1 && (rc = dev_alloc(m, &m->d_dX0, actn))) return rc;      // (sharded runs: inside the exchange segment, peers read it)
        if (!fp32_ops)
            for (int part = 0; part < 2; ++part) {
                if ((rc = dev_alloc(m, &m->d_X0s[part], actn))) return rc;
            }

        // towers
        if (d->n_towers > kMaxTowers) { set_error("more than %d towers", kMaxTowers); return WD_EUNSUPPORTED; }
        int hu_off = 0, did = 0;
        for (int t = 0; t < d->n_towers; ++t) {
            Tower tw{};
            tw.n_hidden = d->tower_nlayers[t]; tw.mode = d->tower_mode[t];
            std::vector<int> hu(d->hidden_units + hu_off, d->hidden_units + hu_off + tw.n_hidden);
            hu_off += tw.n_hidden;
            const std::vector<int> units = hu;                         // the conf's units per layer
            if (m->crelu) for (int& h : hu) h *= 2;                    // features a layer hands on
            auto srcs = layer_sources(tw.mode, tw.n_hidden);
            for (int l = 0; l <= tw.n_hidden; ++l) {
                Layer L{};
                if ((int)srcs[l].size() > kMaxSegs) { set_error("layer with more than %d concatenated inputs", kMaxSegs); return WD_EUNSUPPORTED; }
                L.n_in_segs = (int)srcs[l].size();
                int koff = 0, klog = 0;
                for (int s = 0; s < L.n_in_segs; ++s) {
                    int src = srcs[l][s];
                    Seg sg{};
                    sg.src = src;
                    sg.width = src < 0 ? m->d0_logical : hu[src];
                    sg.width_phys = src < 0 ? d->d0_phys : pad_to(hu[src], 32);
                    sg.k_off = koff;
                    koff += sg.width_phys; klog += sg.width;
                    L.segs[s] = sg;
                }
                L.K = klog; L.K_phys = koff;
                const bool hidden = l < tw.n_hidden;
                L.N = hidden ? hu[l] : 1;
                L.N_phys = hidden ? pad_to(hu[l], 32) : 1;
                L.N_param = hidden ? units[l] : 1;
                L.t_gamma = L.t_beta = -1;
                bool logits_reads = false;
                for (int src : srcs[tw.n_hidden]) if (src == l) logits_reads = true;
                std::vector<int> idx(4, -1);
                if (hidden) {
                    // split-K factor of the weight gradient: enough (tile x split) work items to fill one wave of SMs,
                    // each split still at least 512 batch rows long
                    {
                        const int tiles = ((L.K_phys + 127) / 128) * ((L.N_phys + 127) / 128);     // both engines: 128 x 128 tiles
                        int num_sms = kNumSms;
                        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, m->device);
                        int sp = m->wgrad_splits;
                        while (sp < 32 && tiles * sp * 2 <= num_sms && m->max_batch_pad / (sp * 2) >= 512) sp *= 2;   // double only while one wave still holds it
                        L.wgrad_splits = sp;
                    }
                    L.t_kernel = add_dense(L.K_phys, L.N_phys, L.wgrad_splits, 0, (int64_t)L.K_phys * L.N_phys, true);
                    L.t_bias = add_dense(1, L.N_phys, m->row_tiles, 1, L.N_phys, false);
                    if (m->crelu) m->dense[L.t_kernel].mirror_u = m->dense[L.t_bias].mirror_u = L.N_param;
                    if (m->batch_norm) {
                        L.t_gamma = add_dense(1, L.N_phys, m->row_tiles, 1, L.N_phys, false);
                        L.t_beta = add_dense(1, L.N_phys, m->row_tiles, 1, L.N_phys, false);
                    }
                    const int64_t n = (int64_t)m->max_batch_pad * L.N_phys;
                    // the bf16 family keeps the layer output in fp32 only where the logits layer (not a GEMM) reads it
                    if ((fp32_ops || logits_reads) && (rc = dev_alloc(m, &L.H, n))) return rc;
                    // post-activation values are kept apart from the layer output whenever something sits between them (BN affine, dropout)
                    if (m->batch_norm || m->dropout_rate > 0.f || !L.H) { if ((rc = dev_alloc(m, &L.A, n))) return rc; } else L.A = L.H;
                    if (fp32_ops && (rc = dev_alloc(m, &L.HT, n))) return rc;
                    if ((rc = dev_alloc(m, &L.dH, n))) return rc;
                    if (fp32_ops) {
                        if ((rc = dev_alloc(m, &L.dZ, n))) return rc;
                        if ((rc = dev_alloc(m, &L.dZT, n))) return rc;
                    } else
                        for (int part = 0; part < 2; ++part) {
                            if ((rc = dev_alloc(m, &L.Hs[part], n))) return rc;
                            if ((rc = dev_alloc(m, &L.dZs[part], n))) return rc;
                        }
                } else {
                    L.t_kernel = add_dense(L.K_phys, 1, m->row_tiles, 1, L.K_phys, false);
                    L.t_bias = add_dense(1, 1, m->row_tiles, 1, 4, false);
                }
                idx[WD_D_KERNEL] = L.t_kernel; idx[WD_D_BIAS] = L.t_bias; idx[WD_D_GAMMA] = L.t_gamma; idx[WD_D_BETA] = L.t_beta;
                m->dense_index.push_back(idx);
                m->did_tower.push_back(t); m->did_layer.push_back(l);
                ++did;
                tw.layers.push_back(L);
            }
            if ((rc = dev_alloc(m, &tw.logit, Bm))) return rc;
            m->towers.push_back(tw);
        }
    }
    {
        // block layout: [embedding gradients | wide gradients | touched counts of the small embedding rows | ... of the small wide rows]
        const int64_t nw_small = m->use_wide ? m->wide_rows - m->small_base[1] : 0;
        const int64_t ne_small = (m->use_deep && m->n_small_tab > 0) ? m->emb_total_rows - m->small_base[0] : 0;
        const int64_t grads = m->gs_emb_floats + nw_small;
        m->gs_touch_off[0] = grads;
        m->gs_touch_off[1] = grads + ne_small;
        m->gs_count = grads > 0 ? grads + ne_small + nw_small : 0;
    }
    if (m->dense_count > 0) {
        if ((rc = dev_alloc(m, &m->d_P, m->dense_count))) return rc;
        if ((rc = dev_alloc(m, &m->d_S1, m->dense_count))) return rc;
        if ((rc = dev_alloc(m, &m->d_S2, m->dense_count))) return rc;
        if (G == 1 && (rc = dev_alloc(m, &m->d_G, m->dense_count + m->gs_count))) return rc;
        if ((rc = dev_alloc(m, &m->d_gpart, m->gpart_count))) return rc;
        if (fp32_ops) {
            if ((rc = dev_alloc(m, &m->d_Wt, m->wt_count))) return rc;
            float* split;                                            // the four tf32 splits share one allocation
            if ((rc = dev_alloc(m, &split, 4 * m->wt_count))) return rc;
            m->d_W_hi = split; m->d_W_lo = split + m->wt_count; m->d_Wt_hi = split + 2 * m->wt_count; m->d_Wt_lo = split + 3 * m->wt_count;
        } else {
            if ((rc = dev_alloc(m, &m->d_Wq_hi, m->wt_count))) return rc;
            if ((rc = dev_alloc(m, &m->d_Wq_lo, m->wt_count))) return rc;
        }
        if ((rc = upload(m, &m->d_dense_desc, m->dense))) return rc;
    }

    // ---- sparse backward scratch: lists 0 (embedding rows) and 1 (wide rows); a row-sharded model's lists 2 - 5 in shard_build
    if (std::max(m->emb_total_rows, m->wide_rows) > (1ll << 30)) { set_error("more than 2^30 rows in one table space on one device"); return WD_EUNSUPPORTED; }
    if (m->use_deep && !m->tables.empty() && (rc = list_alloc(m, 0, m->emb_total_rows, m->emb_max_dim, false))) return rc;
    if (m->use_wide && (rc = list_alloc(m, 1, m->wide_rows, 1, false))) return rc;
    if (G > 1 && (rc = shard_build(m, d))) return rc;
    // Embedding tables come last, so an auto-placed table competes only with what is allocated after wd_model_create returns.
    if (m->use_deep && (rc = place_tables(m, hbm_reserve_bytes(m)))) return rc;
    if ((rc = build_record_sets(m))) return rc;               // every table, staging buffer and shard row base is final now
    if (G > 1) {
        DevPlan& dp = m->dplan;
        dp.sh_world = G;
        for (int sx = 0; sx < 2; ++sx) {
            ShardSpace& sp = m->shard.sp[sx];
            if (!sp.on) continue;
            if (sx == 0) { dp.sh_col_emb = sp.d_col_slot; dp.sh_base_emb = sp.set.rec.row_base; dp.sh_own_emb = sp.d_own; dp.sh_lrow_emb = sp.d_lrow; }
            else { dp.sh_col_wide = sp.d_col_slot; dp.sh_base_wide = sp.set.rec.row_base; dp.sh_own_wide = sp.d_own; dp.sh_lrow_wide = sp.d_lrow; }
        }
    }
    if ((rc = metrics_setup())) return rc;
    if ((rc = init_sparse_tables(m, 0, 0))) return rc;           // slots = initial accumulator, weights 0
    if ((rc = init_dense_slots(m))) return rc;
    for (auto& e : m->timer.ev) WD_CUDA(new_event(m, &e, cudaEventDefault));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

extern "C" int wd_model_create(const WdPlanDesc* d, int device, WdModel** out) {
    if (!d || !out) { set_error("null argument"); return WD_EINVAL; }
    if (d->api_version != WD_API_VERSION) { set_error("plan api_version %d != library %d", d->api_version, WD_API_VERSION); return WD_EINVAL; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_error("no CUDA device: libwd_b200 has no CPU fallback");
        return WD_ENODEVICE;
    }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d devices)", device, ndev); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(device));
    WdModel* m = new WdModel();
    m->device = device;
    cudaError_t e = cudaSuccess;
    for (cudaStream_t* s : {&m->stream, &m->stream_up, &m->sstream[0], &m->sstream[1]})
        if (e == cudaSuccess) e = new_stream(m, s);
    for (cudaEvent_t* ev : {&m->ev_grouped[0], &m->ev_grouped[1], &m->ev_done[0], &m->ev_done[1], &m->ev_ids, &m->ev_wide_fwd,
                            &m->ev_wgrad_rest, &m->ev_head, &m->ev_dx0, &m->ev_bwd_done})
        if (e == cudaSuccess) e = new_event(m, ev, cudaEventDisableTiming);
    if (e != cudaSuccess) { set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); wd_model_destroy(m); return WD_ECUDA; }
    m->graphs_enabled = getenv("WD_NO_GRAPH") == nullptr;
    int rc = build_model(d, m);
    if (rc) { wd_model_destroy(m); return rc; }
    *out = m;
    return WD_OK;
}

namespace wd {
// HBM kept free for what is allocated after the embedding tables (see ensure_slot, place_tables and the step graphs): the auto
// tables are placed with it held back, and wd_host_cache_enable refuses a cache that would eat into it.
//   kReserveSlots batch slots beyond slot 0 (cat offsets, keys, dense, label, weight each; bench.py and the estimator use at most 10),
//   the staging buffer + gather ids of the host tables (at most max_nnz records of the widest table), or a row-sharded model's
//   owner staging buffer of its host shards (max_nnz + 1 records, inside the same bound), and the record sets
//   (build_record_sets: a few hundred bytes per table, inside the kGraphReserve margin),
//   kGraphReserve for the instantiated step graphs (one train and one backward graph per slot) and the runtime's growth.
int64_t hbm_reserve_bytes(const WdModel* m) {
    constexpr int kReserveSlots = 16;
    constexpr int64_t kGraphReserve = 256ll << 20;
    const int64_t Bm = m->max_batch;
    const int64_t slot_bytes = (Bm * std::max(m->n_cat_fields, 1) + 1) * 4 + m->keys_cap * 8 + Bm * std::max(m->n_dense_fields, 1) * 4 + 2 * Bm * 4;
    int max_stride = 0;
    for (auto& tb : m->tables) max_stride = std::max(max_stride, tb.stride);
    const int64_t stage_bytes = m->max_nnz * ((int64_t)max_stride + 1) * 4 + 64 * (int64_t)m->tables.size() + 4096;
    return kReserveSlots * slot_bytes + stage_bytes + kGraphReserve;
}
}  // namespace wd

// glorot-uniform kernels / zero biases / gamma 1 / beta 0 built on the host (dense part is ~1.5M floats)
static int init_dense(WdModel* m, uint64_t seed) {
    if (m->dense_count == 0) return WD_OK;
    std::vector<float> P(m->dense_count, 0.f), S1(m->dense_count, 0.f), S2(m->dense_count, 0.f);
    std::mt19937_64 rng(seed * 7919 + 17);
    std::uniform_real_distribution<float> U(-1.f, 1.f);
    for (size_t ti = 0; ti < m->towers.size(); ++ti) {
        Tower& tw = m->towers[ti];
        for (int l = 0; l <= tw.n_hidden; ++l) {
            Layer& L = tw.layers[l];
            const DenseTensor& tk = m->dense[L.t_kernel];
            const float lim = std::sqrt(6.f / (float)(L.K + L.N_param));          // glorot_uniform over the variable's shape [K, N_param]
            for (int s = 0; s < L.n_in_segs; ++s) {
                const Seg& sg = L.segs[s];
                for (int j = 0; j < sg.width_phys; ++j) {
                    bool real = sg.src < 0 ? (m->x0_real[j] != 0) : (j < sg.width);
                    if (!real) continue;
                    float* prow = &P[tk.off + (int64_t)(sg.k_off + j) * L.N_phys];
                    for (int n = 0; n < L.N_param; ++n) {
                        prow[n] = lim * U(rng);
                        if (tk.mirror_u) prow[n + tk.mirror_u] = -prow[n];
                    }
                }
            }
            if (L.t_gamma >= 0) for (int n = 0; n < L.N; ++n) P[m->dense[L.t_gamma].off + n] = 1.f;
        }
    }
    for (size_t i = 0; i < m->dense.size(); ++i) {
        const WdOptimizer& o = (m->use_wide && i == 0) ? m->lin_opt : m->dnn_opt;
        float s1 = slot1_init(o);
        for (int64_t j = 0; j < m->dense[i].count; ++j) S1[m->dense[i].off + j] = s1;
    }
    WD_CUDA(cudaMemcpyAsync(m->d_P, P.data(), P.size() * 4, cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaMemcpyAsync(m->d_S1, S1.data(), S1.size() * 4, cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaMemcpyAsync(m->d_S2, S2.data(), S2.size() * 4, cudaMemcpyHostToDevice, m->stream));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return refresh_weight_copies(m);
}

extern "C" int wd_model_init(WdModel* m, uint64_t seed) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    int rc = init_sparse_tables(m, seed, 1);
    if (rc) return rc;
    rc = init_dense(m, seed);
    if (rc) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    m->initialized = true;
    return WD_OK;
}

// ---------------------------------------------------------------------------------------------- tensor IO
static int resolve_dense(WdModel* m, int did, int sub, int* out) {
    if (did < 0 || did >= (int)m->dense_index.size() || sub < 0 || sub > 3 || m->dense_index[did][sub] < 0) {
        set_error("no dense tensor (%d, %d)", did, sub);
        return WD_EINVAL;
    }
    *out = m->dense_index[did][sub];
    return WD_OK;
}

extern "C" int64_t wd_tensor_size(WdModel* m, int kind, int index, int sub) {
    if (!m) return WD_EINVAL;
    if (kind == WD_T_WIDE_COL) {
        if (index < 0 || index >= m->n_columns) return WD_EINVAL;
        const ShardSpace& sw = m->shard.sp[1];
        if (sw.on && sw.h_col_slot[index] >= 0) return (m->col_buckets[index] - m->shard.rank + m->shard.world - 1) / m->shard.world;   // this rank's rows
        return m->col_wide_base[index] >= 0 ? m->col_buckets[index] : WD_EINVAL;
    }
    if (kind == WD_T_WIDE_BIAS) return m->use_wide ? 1 : WD_EINVAL;
    if (kind == WD_T_EMB_TABLE) return (index >= 0 && index < (int)m->tables.size()) ? m->tables[index].arows * m->tables[index].dim_logical : WD_EINVAL;
    if (kind == WD_T_DENSE) {
        int di;
        if (resolve_dense(m, index, sub, &di)) return WD_EINVAL;
        Layer& L = m->towers[m->did_tower[index]].layers[m->did_layer[index]];
        return sub == WD_D_KERNEL ? (int64_t)L.K * L.N_param : (sub == WD_D_BIAS ? L.N_param : L.N);
    }
    return WD_EINVAL;
}

extern "C" int wd_memory_usage(WdModel* m, int64_t* device_bytes, int64_t* host_bytes) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    if (device_bytes) *device_bytes = m->bytes_allocated;
    if (host_bytes) *host_bytes = m->host_bytes;
    return WD_OK;
}

extern "C" int wd_tensor_io(WdModel* m, int kind, int index, int sub, int slot, void* host, int64_t count, int to_device) {
    if (!m || !host) { set_error("null argument"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    int64_t want = wd_tensor_size(m, kind, index, sub);
    if (want < 0 || want != count) { set_error("tensor (%d,%d,%d): size %lld, caller passed %lld", kind, index, sub, (long long)want, (long long)count); return WD_EINVAL; }
    if (slot < 0 || slot > 2) { set_error("slot out of range"); return WD_EINVAL; }
    const cudaMemcpyKind dir = to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
    if (kind == WD_T_WIDE_COL) {
        const ShardSpace& sw = m->shard.sp[1];
        float* dev = (sw.on && sw.h_col_slot[index] >= 0)
                         ? reinterpret_cast<float*>(sw.d_wide + sw.h_slot_base[sw.h_col_slot[index]]) + slot     // rows r = rank, rank + G, ...
                         : reinterpret_cast<float*>(m->d_wide + m->col_wide_base[index]) + slot;
        if (to_device) WD_CUDA(cudaMemcpy2DAsync(dev, 16, host, 4, 4, count, dir, m->stream));
        else WD_CUDA(cudaMemcpy2DAsync(host, 4, dev, 16, 4, count, dir, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
        return WD_OK;
    }
    if (kind == WD_T_EMB_TABLE) {
        EmbTable& tb = m->tables[index];
        if (slot * tb.dim >= tb.stride) { set_error("table has no optimizer slot %d", slot); return WD_EINVAL; }
        float* dev = tb.data + slot * tb.dim;
        const size_t lw = (size_t)tb.dim_logical * 4;
        // host records cached in HBM (one GPU, or this rank's host shards): dirty slots go home before either direction; a write
        // then empties the cache
        if (tb.host) {
            const int rc = host_cache_sync(m, true, to_device != 0);
            if (rc) return rc;
        }
        // a deferred table's rows are brought up to the current step before a read; a write makes them current
        if (deferred(tb) && !to_device) {
            const int rc = deferred_adam_settle(m, tb, 0, tb.arows, false);
            if (rc) return rc;
        }
        const cudaMemcpyKind dir = tb.host ? cudaMemcpyDefault : (to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost);
        if (to_device) WD_CUDA(cudaMemcpy2DAsync(dev, (size_t)tb.stride * 4, host, lw, lw, tb.arows, dir, m->stream));
        else WD_CUDA(cudaMemcpy2DAsync(host, lw, dev, (size_t)tb.stride * 4, lw, tb.arows, dir, m->stream));
        if (deferred(tb) && to_device) {
            const int rc = deferred_adam_settle(m, tb, 0, tb.arows, true);
            if (rc) return rc;
        }
        WD_CUDA(cudaStreamSynchronize(m->stream));
        return WD_OK;
    }
    float* arena = slot == 0 ? m->d_P : (slot == 1 ? m->d_S1 : m->d_S2);
    if (kind == WD_T_WIDE_BIAS) {
        WD_CUDA(cudaMemcpyAsync(to_device ? (void*)(arena + m->dense[0].off) : host, to_device ? host : (void*)(arena + m->dense[0].off), 4, dir, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
        return WD_OK;
    }
    int di;
    int rc = resolve_dense(m, index, sub, &di);
    if (rc) return rc;
    const DenseTensor& t = m->dense[di];
    Layer& L = m->towers[m->did_tower[index]].layers[m->did_layer[index]];
    std::vector<float> phys(t.count, 0.f);
    float* h = (float*)host;
    if (!to_device || slot > 0) {
        WD_CUDA(cudaMemcpyAsync(phys.data(), arena + t.off, t.count * 4, cudaMemcpyDeviceToHost, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
    }
    if (sub == WD_D_KERNEL) {
        int64_t lk = 0;
        for (int s = 0; s < L.n_in_segs; ++s) {
            const Seg& sg = L.segs[s];
            for (int j = 0; j < sg.width_phys; ++j) {
                bool real = sg.src < 0 ? (m->x0_real[j] != 0) : (j < sg.width);
                if (!real) continue;
                for (int n = 0; n < L.N_param; ++n) {
                    float& pv = phys[(int64_t)(sg.k_off + j) * L.N_phys + n];
                    if (to_device) {
                        pv = h[lk * L.N_param + n];
                        if (t.mirror_u) (&pv)[t.mirror_u] = slot == 0 ? -pv : pv;       // tied half: minus the weight, same slot value
                    } else h[lk * L.N_param + n] = pv;
                }
                ++lk;
            }
        }
        if (lk != L.K) { set_error("internal: logical K mismatch %lld vs %d", (long long)lk, L.K); return WD_ESTATE; }
    } else {
        const int nn = sub == WD_D_BIAS ? L.N_param : L.N;
        for (int n = 0; n < nn; ++n) {
            if (to_device) {
                phys[n] = h[n];
                if (t.mirror_u) phys[n + t.mirror_u] = slot == 0 ? -h[n] : h[n];
            } else h[n] = phys[n];
        }
    }
    if (to_device) {
        // all copies go through the model stream: a pageable cudaMemcpy on the NULL stream may still be in flight when a
        // kernel on this (non-blocking) stream starts
        WD_CUDA(cudaMemcpyAsync(arena + t.off, phys.data(), t.count * 4, cudaMemcpyHostToDevice, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
        if (slot == 0 && t.wt_off >= 0) return refresh_weight_copies(m);
    }
    return WD_OK;
}

extern "C" int wd_tensor_io_rows(WdModel* m, int kind, int index, int sub, int slot, int64_t row0, int64_t nrows, void* host, int to_device) {
    if (!m || !host) { set_error("null argument"); return WD_EINVAL; }
    if (kind != WD_T_EMB_TABLE && kind != WD_T_WIDE_COL) { set_error("wd_tensor_io_rows: tensor kind %d has no rows", kind); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    const int64_t size = wd_tensor_size(m, kind, index, sub);
    if (size < 0) { set_error("no tensor (%d,%d,%d)", kind, index, sub); return WD_EINVAL; }
    const int64_t rows = kind == WD_T_EMB_TABLE ? m->tables[index].arows : size;
    if (row0 < 0 || nrows < 0 || row0 > rows - nrows) {
        set_error("tensor (%d,%d,%d): rows [%lld, %lld) outside its %lld rows", kind, index, sub, (long long)row0, (long long)(row0 + nrows),
                  (long long)rows);
        return WD_EINVAL;
    }
    if (slot < 0 || slot > 2) { set_error("slot out of range"); return WD_EINVAL; }
    if (nrows == 0) return WD_OK;
    if (kind == WD_T_WIDE_COL) {
        const ShardSpace& sw = m->shard.sp[1];
        float4* base = (sw.on && sw.h_col_slot[index] >= 0) ? sw.d_wide + sw.h_slot_base[sw.h_col_slot[index]] : m->d_wide + m->col_wide_base[index];
        float* dev = reinterpret_cast<float*>(base + row0) + slot;
        if (to_device) WD_CUDA(cudaMemcpy2DAsync(dev, 16, host, 4, 4, nrows, cudaMemcpyHostToDevice, m->stream));
        else WD_CUDA(cudaMemcpy2DAsync(host, 4, dev, 16, 4, nrows, cudaMemcpyDeviceToHost, m->stream));
        WD_CUDA(cudaStreamSynchronize(m->stream));
        return WD_OK;
    }
    EmbTable& tb = m->tables[index];
    if (slot * tb.dim >= tb.stride) { set_error("table has no optimizer slot %d", slot); return WD_EINVAL; }
    float* dev = tb.data + row0 * tb.stride + slot * tb.dim;
    const size_t lw = (size_t)tb.dim_logical * 4;
    int rc;
    // wd_tensor_io's guarantees, for the rows of the range only: their dirty cached records go home before either direction and a
    // write empties their slots; a deferred table's rows are settled before a read and stamped after a write
    if (tb.host && (rc = host_cache_sync_rows(m, tb, row0, nrows, to_device != 0))) return rc;
    if (deferred(tb) && !to_device && (rc = deferred_adam_settle(m, tb, row0, nrows, false))) return rc;
    const cudaMemcpyKind dir = tb.host ? cudaMemcpyDefault : (to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost);
    if (to_device) WD_CUDA(cudaMemcpy2DAsync(dev, (size_t)tb.stride * 4, host, lw, lw, nrows, dir, m->stream));
    else WD_CUDA(cudaMemcpy2DAsync(host, lw, dev, (size_t)tb.stride * 4, lw, nrows, dir, m->stream));
    if (deferred(tb) && to_device && (rc = deferred_adam_settle(m, tb, row0, nrows, true))) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

// -------------------------------------------------------------------------------------------------- steps
static int check_ready(WdModel* m) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    WD_CUDA(cudaSetDevice(m->device));
    return WD_OK;
}
static void timer_begin(WdModel* m) {
    if (!m->timer.enabled) return;
    m->timer.n = 0;
    mark(m, "start");
}

// allocates the buffers of batch slots up to `s` on first use
static int ensure_slot(WdModel* m, int s) {
    if (s < 0 || s >= 64) { set_error("batch slot %d out of range [0, 64)", s); return WD_EINVAL; }
    while ((int)m->slots.size() <= s) {
        BatchSlot b;
        int rc;
        const int64_t Bm = m->max_batch;
        if ((rc = dev_alloc(m, &b.off, Bm * std::max(m->n_cat_fields, 1) + 1))) return rc;
        if ((rc = dev_alloc(m, &b.keys, m->keys_cap))) return rc;
        if ((rc = dev_alloc(m, &b.dense, Bm * std::max(m->n_dense_fields, 1)))) return rc;
        if ((rc = dev_alloc(m, &b.label, Bm))) return rc;
        if ((rc = dev_alloc(m, &b.weight, Bm))) return rc;
        m->slots.push_back(b);
    }
    return WD_OK;
}
// make batch slot `s` current (allocating its buffers on first use)
static int select_slot(WdModel* m, int s) {
    int rc = ensure_slot(m, s);
    if (rc) return rc;
    BatchSlot& b = m->slots[s];
    m->cur_slot = s;
    if (b.filled) m->dbatch = b.view;
    if (b.up_pending) {                                     // a prefetch refilled this slot on the upload stream
        WD_CUDA(cudaStreamWaitEvent(m->stream, b.ev_up, 0));
        b.up_pending = false;
    }
    return WD_OK;
}
// the prologue of the entry points that run on a slot: makes `slot` current, refuses a slot never filled and, when the caller
// needs labels (`needs_labels` names what it does with them), a batch without
static int use_slot(WdModel* m, int slot, const char* needs_labels) {
    int rc = select_slot(m, slot);
    if (rc) return rc;
    if (!m->slots[slot].filled) { set_error("batch slot %d was never uploaded", slot); return WD_ESTATE; }
    if (needs_labels && !m->dbatch.label) { set_error("%s needs labels", needs_labels); return WD_EINVAL; }
    return WD_OK;
}
// slot `s` now holds batch `view`; `pending`: its copies were issued on the upload stream, which the next step on it waits for
static void fill_slot(WdModel* m, int s, const DevBatch& view, bool pending) {
    BatchSlot& sl = m->slots[s];
    sl.view = view;
    sl.filled = true;
    if (pending) sl.up_pending = true;
    if (s == m->cur_slot) m->dbatch = view;
}
// the model stream has consumed the current slot up to here (a later prefetch into it must wait for this point)
static int mark_slot_used(WdModel* m) {
    BatchSlot& b = m->slots[m->cur_slot];
    if (!b.ev_used) WD_CUDA(new_event(m, &b.ev_used, cudaEventDisableTiming));
    WD_CUDA(cudaEventRecord(b.ev_used, m->stream));
    b.used_recorded = true;
    return WD_OK;
}

// copies a host batch into the buffers of slot `sl` on stream `st`; fills the device view of the batch
static int upload_into(WdModel* m, BatchSlot& sl, const WdBatch* b, cudaStream_t st, DevBatch* view) {
    if (!b || b->batch_size <= 0 || b->batch_size > m->max_batch) { set_error("batch_size %d outside (0, %d]", b ? b->batch_size : -1, m->max_batch); return WD_EINVAL; }
    const int B = b->batch_size, F = m->n_cat_fields, Nd = m->n_dense_fields;
    int64_t nnz = b->cat_offsets ? b->nnz : (int64_t)B * F;
    if (nnz > m->keys_cap) { set_error("batch has %lld keys, capacity %lld (raise max_keys)", (long long)nnz, (long long)m->keys_cap); return WD_EINVAL; }
    if (F > 0) {
        if (b->cat_offsets) WD_CUDA(cudaMemcpyAsync(sl.off, b->cat_offsets, ((int64_t)B * F + 1) * 4, cudaMemcpyHostToDevice, st));
        if (nnz > 0) WD_CUDA(cudaMemcpyAsync(sl.keys, b->cat_keys, nnz * 8, cudaMemcpyHostToDevice, st));
    }
    if (Nd > 0) WD_CUDA(cudaMemcpyAsync(sl.dense, b->dense, (int64_t)B * Nd * 4, cudaMemcpyHostToDevice, st));
    if (b->label) WD_CUDA(cudaMemcpyAsync(sl.label, b->label, (int64_t)B * 4, cudaMemcpyHostToDevice, st));
    if (b->weight) WD_CUDA(cudaMemcpyAsync(sl.weight, b->weight, (int64_t)B * 4, cudaMemcpyHostToDevice, st));
    view->B = B;
    view->cat_offsets = (F > 0 && b->cat_offsets) ? sl.off : nullptr;
    view->cat_keys = sl.keys;
    view->dense = sl.dense;
    view->label = b->label ? sl.label : nullptr;
    view->weight = b->weight ? sl.weight : nullptr;
    return WD_OK;
}

static int upload_current(WdModel* m, const WdBatch* b) {
    DevBatch view{};
    int rc = upload_into(m, m->slots[m->cur_slot], b, m->stream, &view);
    if (rc) return rc;
    fill_slot(m, m->cur_slot, view, false);
    mark(m, "h2d");
    return WD_OK;
}

// Asynchronous refill of a batch slot: the copies run on the library's upload stream, behind the last step that read the slot
// and concurrently with whatever the model stream is doing (normally: the step on another slot).  The next step on this slot
// waits for them on the device.  Host buffers must stay untouched until that step has been issued and returned.
extern "C" int wd_batch_prefetch_slot(WdModel* m, int slot, const WdBatch* b) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = ensure_slot(m, slot))) return rc;
    BatchSlot& sl = m->slots[slot];
    if (!sl.ev_up) WD_CUDA(new_event(m, &sl.ev_up, cudaEventDisableTiming));
    if (sl.used_recorded) WD_CUDA(cudaStreamWaitEvent(m->stream_up, sl.ev_used, 0));
    DevBatch view{};
    if ((rc = upload_into(m, sl, b, m->stream_up, &view))) return rc;
    WD_CUDA(cudaEventRecord(sl.ev_up, m->stream_up));
    fill_slot(m, slot, view, true);
    return WD_OK;
}

// TSV text -> batch slot on the device (tsv.cu), ordered like wd_batch_prefetch_slot: behind the last step that read the slot, on
// the upload stream.  Waits for this parse only; a batch the device parser declines is parsed on the host and uploaded instead.
extern "C" int wd_tsv_parse_slot(WdModel* m, int slot, const WdTsvSpec* sp, const char* text, int64_t text_len, const int64_t* starts,
                                 int32_t n_lines) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (!sp || !text || !starts || n_lines < 0 || text_len < 0) { set_error("wd_tsv_parse_slot: bad arguments"); return WD_EINVAL; }
    if ((rc = ensure_slot(m, slot))) return rc;
    BatchSlot& sl = m->slots[slot];
    if (!sl.ev_up) WD_CUDA(new_event(m, &sl.ev_up, cudaEventDisableTiming));
    if (sl.used_recorded) WD_CUDA(cudaStreamWaitEvent(m->stream_up, sl.ev_used, 0));
    int status = 0;
    if ((rc = tsv_parse_device(m, sp, text, text_len, starts, n_lines, sl.off, sl.keys, sl.dense, sl.label, sl.weight, m->stream_up, &status))) return rc;
    DevBatch view{};
    if (status == 0) {
        view.B = n_lines;
        view.cat_offsets = m->n_cat_fields > 0 ? sl.off : nullptr;
        view.cat_keys = sl.keys;
        view.dense = sl.dense;
        view.label = sp->has_label ? sl.label : nullptr;
        view.weight = (sp->use_weight && sp->has_label) ? sl.weight : nullptr;
        m->tsv_device_batches++;
    } else {
        WdBatch hb{};
        if ((rc = tsv_parse_host(sp, text, starts, n_lines, &hb))) return rc;
        if ((rc = upload_into(m, sl, &hb, m->stream_up, &view))) return rc;
        m->tsv_host_batches++;
    }
    WD_CUDA(cudaEventRecord(sl.ev_up, m->stream_up));
    if (status != 0) WD_CUDA(cudaEventSynchronize(sl.ev_up));      // the host batch lives in per-thread buffers
    fill_slot(m, slot, view, true);
    return WD_OK;
}

extern "C" int wd_tsv_parse_stats(WdModel* m, int64_t* out, int32_t n, int32_t reset) {
    if (!m) { set_error("null model"); return WD_EINVAL; }
    const int64_t v[2] = {m->tsv_device_batches, m->tsv_host_batches};
    for (int i = 0; i < n && i < 2; ++i) out[i] = v[i];
    if (reset) m->tsv_device_batches = m->tsv_host_batches = 0;
    return WD_OK;
}

extern "C" int wd_batch_upload_slot(WdModel* m, int slot, const WdBatch* b) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = select_slot(m, slot))) return rc;
    return upload_current(m, b);
}
extern "C" int wd_batch_upload(WdModel* m, const WdBatch* b) { return wd_batch_upload_slot(m, 0, b); }

static int finish_step(WdModel* m, float* loss_out, float* logits_out) {
    int32_t* flags_host = reinterpret_cast<int32_t*>(m->h_loss_pinned + 4);
    WD_CUDA(cudaMemcpyAsync(m->h_loss_pinned, m->d_loss, 4, cudaMemcpyDeviceToHost, m->stream));
    WD_CUDA(cudaMemcpyAsync(flags_host, m->d_flags, 4, cudaMemcpyDeviceToHost, m->stream));
    if (logits_out) WD_CUDA(cudaMemcpyAsync(logits_out, m->d_logits, (int64_t)m->dbatch.B * 4, cudaMemcpyDeviceToHost, m->stream));
    mark(m, "d2h");
    WD_CUDA(cudaStreamSynchronize(m->stream));
    if (flags_host[0] & 1) {
        cudaMemsetAsync(m->d_flags, 0, 16, m->stream);
        set_error("categorical-column id capacity exceeded (max_nnz=%lld): recreate the model with a larger max_nnz", (long long)m->max_nnz);
        return WD_EINVAL;
    }
    if (flags_host[0] & 2) {
        cudaMemsetAsync(m->d_flags, 0, 16, m->stream);
        set_error("row-sharded exchange capacity exceeded (a rank received more than %lld ids): raise shard_slack / shard_capacity", (long long)m->max_nnz);
        return WD_EINVAL;
    }
    if (flags_host[0] & 8) {
        cudaMemsetAsync(m->d_flags, 0, 16, m->stream);
        set_error("data-parallel list exchange: this rank touched more unique rows than the fixed list length it exchanges (wd_sparse_set_sorted list_len); raise fixed_rows");
        return WD_EINVAL;
    }
    if (flags_host[0] & 4) {
        cudaMemsetAsync(m->d_flags, 0, 16, m->stream);
        set_error("row-sharded exchange: a peer rank did not reach a barrier within 20 s (ranks out of step, or a rank failed)");
        return WD_ESTATE;
    }
    if (loss_out) *loss_out = m->dbatch.label ? m->h_loss_pinned[0] : 0.f;
    if (m->timer.enabled) {
        PhaseTimer& t = m->timer;
        for (int i = 1; i < t.n; ++i) cudaEventElapsedTime(&t.ms[i], t.ev[i - 1], t.ev[i]);
        t.ms[0] = 0.f;
        if (t.n > 1) cudaEventElapsedTime(&t.ms[0], t.ev[0], t.ev[t.n - 1]);   // [0] = total
        t.n_last = t.n;
    }
    return WD_OK;
}

static bool list_present(const WdModel* m, int which) { return which == 0 ? (m->use_deep && !m->tables.empty()) : m->use_wide; }

// launch the id-only grouping of both sparse lists on their side streams (overlaps forward + backward of the towers)
// WD_STEP_TRACE=1: stamp i of the step timeline on whatever stream is current (captured into the step's graph like any kernel)
__global__ void step_stamp_kernel(unsigned long long* t) { unsigned long long v; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v)); *t = v; }
enum { ST_START = 0, ST_IDS, ST_GATHER, ST_HEAD, ST_BWD, ST_MAIN_END, ST_G0, ST_G1, ST_R0_BEG, ST_R0_END, ST_R1_BEG, ST_R1_END, ST_A0_END, ST_A1_END };
static void stamp(WdModel* m, int i) {
    if (!m->d_step_trace) return;
    step_stamp_kernel<<<1, 1, 0, m->stream>>>(m->d_step_trace + i);
    m->launches++;
}

// group_async, backward_core and apply_core are also pieces of the row-sharded rank-step (shard.cu)
namespace wd {
int group_async(WdModel* m) {
    if (m->timer.enabled) return WD_OK;                      // profiling: keep everything on one stream (done before the reduce)
    WD_CUDA(cudaEventRecord(m->ev_ids, m->stream));
    for (int w = 0; w < 2; ++w) {
        if (!list_present(m, w)) continue;
        WD_CUDA(cudaStreamWaitEvent(m->sstream[w], m->ev_ids, 0));
        int rc = on_side(m, w, [&] { int r = sparse_group_which(m, w); stamp(m, ST_G0 + w); return r; });
        if (rc) return rc;
        WD_CUDA(cudaEventRecord(m->ev_grouped[w], m->sstream[w]));
        m->side_pending[w] = true;
    }
    return WD_OK;
}

static int forward_core(WdModel* m, bool train) {
    int rc;
    m->stepped = true;
    stamp(m, ST_START);
    if ((rc = ids_prepare(m))) return rc;
    mark(m, "ids");
    stamp(m, ST_IDS);
    // training: the wide logit is needed only by the head, so it is computed on side stream 1, ahead of that stream's grouping work
    const bool wide_aside = train && !m->timer.enabled && m->use_wide && m->use_deep && list_present(m, 1);
    if (wide_aside) {
        WD_CUDA(cudaEventRecord(m->ev_ids, m->stream));
        WD_CUDA(cudaStreamWaitEvent(m->sstream[1], m->ev_ids, 0));
        if ((rc = on_side(m, 1, [&] { return sparse_forward_wide(m); }))) return rc;
        WD_CUDA(cudaEventRecord(m->ev_wide_fwd, m->sstream[1]));
    }
    if (train && (rc = group_async(m))) return rc;
    if (!wide_aside && (rc = sparse_forward_wide(m))) return rc;
    if (m->n_host_tab > 0) {
        // host tables: the gather reads the step's unique host rows from the staging buffer, so the embedding list is grouped first
        // (on side stream 0 when the train step put it there, else here; the backward then groups it once more only when profiling)
        if (m->side_pending[0]) WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_grouped[0], 0));
        else if ((rc = sparse_group_which(m, 0))) return rc;
        if ((rc = host_tables_stage_in(m, train))) return rc;
    }
    if ((rc = sparse_forward_emb(m))) return rc;
    stamp(m, ST_GATHER);
    if ((rc = mlp_forward(m, train))) return rc;
    mark(m, "mlp_other");
    if (wide_aside) WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_wide_fwd, 0));
    if ((rc = loss_forward(m, train))) return rc;
    mark(m, "head");
    stamp(m, ST_HEAD);
    if (train && (m->side_pending[0] || m->side_pending[1])) WD_CUDA(cudaEventRecord(m->ev_head, m->stream));
    if (train && m->summary_armed && (rc = summary_launch(m))) return rc;     // (after ev_head: the side streams do not wait for it)
    return WD_OK;
}

// Backward.  Main stream: towers (dgrad before wgrad per layer), dense gradient reduction.  Side streams (when the
// grouping already lives there): wide gradient sums as soon as dlogit exists, embedding gradient sums as soon as dX0
// exists — i.e. under the remaining weight-gradient GEMMs.
int backward_core(WdModel* m) {
    int rc;
    m->side_active[0] = m->side_active[1] = false;
    if (m->gs_count > 0) WD_CUDA(cudaMemsetAsync(m->d_G + m->dense_count, 0, (size_t)m->gs_count * sizeof(float), m->stream));
    if (m->side_pending[1]) {
        if (m->gs_count > 0) { WD_CUDA(cudaEventRecord(m->ev_head, m->stream)); }     // (re-recorded: also orders the memset above)
        WD_CUDA(cudaStreamWaitEvent(m->sstream[1], m->ev_head, 0));
        if ((rc = on_side(m, 1, [&] { stamp(m, ST_R1_BEG); int r = sparse_reduce_wide(m); if (!r) r = small_scatter(m, 1); stamp(m, ST_R1_END); return r; }))) return rc;
        m->side_active[1] = true;
    }
    m->record_dx0 = m->side_pending[0];
    m->dx0_recorded = false;
    // single-GPU fused step with the wide list on its side stream: the dense optimizer of everything but the first layer's kernel
    // runs there (after the wide rows' updates), under that kernel's weight-gradient GEMM
    m->dense_split_tensor = -1;
    m->record_wgrad_rest = m->fuse_dense && m->side_active[1] && m->operands == kBf16Operands && !m->timer.enabled && !m->crelu;
    if ((rc = mlp_backward(m))) return rc;
    m->record_dx0 = false;
    m->record_wgrad_rest = false;
    mark(m, "mlp_other");
    stamp(m, ST_BWD);
    if (m->side_pending[0] && m->dx0_recorded) {
        WD_CUDA(cudaStreamWaitEvent(m->sstream[0], m->ev_dx0, 0));
        if ((rc = on_side(m, 0, [&] { stamp(m, ST_R0_BEG); int r = sparse_reduce_emb(m); if (!r) r = small_scatter(m, 0); stamp(m, ST_R0_END); return r; }))) return rc;
        m->side_active[0] = true;
    }
    if ((rc = wide_bias_grad(m))) return rc;
    if ((rc = dense_reduce_grads(m))) return rc;
    mark(m, "dense_reduce");
    for (int w = 0; w < 2; ++w) {                           // lists that stay on the main stream
        if (m->side_active[w] || !list_present(m, w)) { m->side_pending[w] = false; continue; }
        if (m->side_pending[w]) WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_grouped[w], 0));
        else if ((rc = sparse_group_which(m, w))) return rc;
        m->side_pending[w] = false;
        if ((rc = (w == 0 ? sparse_reduce_emb(m) : sparse_reduce_wide(m)))) return rc;
        if ((rc = small_scatter(m, w))) return rc;
    }
    if (m->gs_count > 0)                                    // the dense block is read (all-reduced) on the main stream
        for (int w = 0; w < 2; ++w)
            if (m->side_active[w]) {
                WD_CUDA(cudaEventRecord(m->ev_done[w], m->sstream[w]));
                WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_done[w], 0));
            }
    m->grads_pending = true;
    return WD_OK;
}

// Optimizer.  A list whose sums live on its side stream is applied there (after its merge in data-parallel runs); the dense
// optimizer runs on the main stream meanwhile and the streams join at the end of the step.
int apply_core(WdModel* m) {
    int rc;
    const bool split_dense = m->fuse_dense && m->dense_split_tensor >= 0 && m->side_active[1];
    for (int w = 0; w < 2; ++w) {
        if (m->side_active[w]) {
            if ((rc = on_side(m, w, [&]() -> int {
                    int r = sparse_apply_which(m, w);
                    stamp(m, ST_A0_END + w);
                    if (!r && w == 1 && split_dense) {
                        WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_wgrad_rest, 0));
                        m->dense_part = 2;
                        r = dense_apply(m);
                        m->dense_part = 0;
                    }
                    return r;
                }))) return rc;
            WD_CUDA(cudaEventRecord(m->ev_done[w], m->sstream[w]));
        } else if ((rc = sparse_apply_which(m, w))) return rc;
    }
    mark(m, "sparse_apply");
    m->dense_part = split_dense ? 1 : 0;
    rc = dense_apply(m);
    m->dense_part = 0;
    if (rc) return rc;
    if ((rc = small_apply(m))) return rc;
    mark(m, "dense_apply");
    stamp(m, ST_MAIN_END);
    if (m->dropout_rate > 0.f && (rc = step_tick(m))) return rc;          // the dropout counter advances once per train step
    if (m->lin_opt.kind == WD_OPT_ADAM || m->dnn_opt.kind == WD_OPT_ADAM) {
        // Sparse Adam moves every row of a table each step, and each row exactly once (sparse_dev.cuh).  Per record set: first
        // every touched-row update of the step, then the set's untouched pass, on the stream that ran the last of those updates.
        // A replicated set is updated by its list (possibly on its side stream, after the data-parallel merge) and by the dense
        // block (small_apply, here): join the lists, then its pass runs here.  A row-sharded set is updated only by its owner,
        // whose pass follows on the owner's stream (shard.cu), which has joined this one by now.  AdamOptimizer._finish: the beta
        // powers advance once per step, after all of that.
        for (int w = 0; w < 2; ++w)
            if (m->side_active[w]) WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_done[w], 0));
        if ((rc = adam_untouched_replicated(m))) return rc;
        mark(m, "adam_untouched");
        if ((rc = adam_tick(m))) return rc;
    }
    for (int w = 0; w < 2; ++w)
        if (m->side_active[w]) { WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_done[w], 0)); m->side_active[w] = false; }
    m->grads_pending = false;
    return WD_OK;
}
}  // namespace wd

static int train_eager(WdModel* m) {
    int rc;
    // the whole step runs here, nothing exchanges the dense gradient arena between backward and optimizer: reduce the gradient
    // partials inside the optimizer kernel (mlp.cu dense_vec_kernel<2>)
    m->fuse_dense = true;
    rc = forward_core(m, true);
    if (!rc) rc = backward_core(m);
    if (!rc) rc = apply_core(m);
    m->fuse_dense = false;
    return rc;
}

enum class GraphRun { eager, captured, replayed };

// Issues step work through a CUDA graph.  issue(capturing) enqueues the work on `st`; under capture it joins every other stream it
// forks back into `st`.  The work runs eagerly twice, is then captured once and replayed for as long as `key` equals the key the
// capture baked in; a different key re-captures at once.  A replay removes the launch gaps between the work's many small kernels,
// and the host cost becomes one cudaGraphLaunch.  With WD_NO_GRAPH=1 or profiling on, or for good once a capture has failed,
// the work runs eagerly.  *how tells the caller which of the three happened.
template <class Key, class F>
static int run_graphed(WdModel* m, StepGraph<Key>& g, const Key& key, cudaStream_t st, F issue, GraphRun* how) {
    *how = GraphRun::eager;
    if (!m->graphs_enabled || m->timer.enabled) return issue(false);
    if (g.exec && g.key == key) {
        *how = GraphRun::replayed;
        m->graph_replays++;
    } else if (g.eager < 2) {
        const int rc = issue(false);
        if (rc == WD_OK) g.eager++;
        return rc;
    } else {
        g.destroy();
        const int64_t l0 = m->launches;
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            const int rc = issue(true);
            const cudaError_t e2 = cudaStreamEndCapture(st, &graph);
            if (rc == WD_OK && e2 == cudaSuccess && graph) e = cudaGraphInstantiate(&g.exec, graph, 0);
            else e = e2 != cudaSuccess ? e2 : cudaErrorUnknown;
            if (graph) cudaGraphDestroy(graph);
        }
        if (e != cudaSuccess || !g.exec) {                  // not capturable here: stay eager for good
            cudaGetLastError();
            g.exec = nullptr;
            m->graphs_enabled = false;
            return issue(false);
        }
        g.key = key;
        g.launches = m->launches - l0;                      // counted again on every launch of the graph
        m->launches = l0;
        *how = GraphRun::captured;
        m->graph_captures++;
    }
    WD_CUDA(cudaGraphLaunch(g.exec, st));
    m->launches += g.launches;
    return WD_OK;
}

// A train step through its slot's graph.  A step armed for layer summaries (wd_summary_arm) runs eagerly instead: it is one step
// in save_summary_steps (1000 in conf/train.yaml), and a second graph per slot would cost a capture and its device memory to save
// the launch gaps of that one step.  The plain step's graph stays the one every other step replays.
template <class Key, class F>
static int run_train_graphed(WdModel* m, StepGraph<Key>& g, const Key& key, F issue, GraphRun* how) {
    if (m->summary_armed) {
        *how = GraphRun::eager;
        return issue(false);
    }
    return run_graphed(m, g, key, m->stream, issue, how);
}

// After a graph ran in place of the issuing code, the host state that code leaves behind (a replay runs none of it): a whole step
// leaves nothing pending; the split step (`bwd`: its slot) leaves the lists' sums on the side streams the captured backward left
// them on, and those streams continue behind the graph.
static int after_graph(WdModel* m, GraphRun how, BatchSlot* bwd) {
    if (how == GraphRun::eager) return WD_OK;
    if (bwd && how == GraphRun::captured)
        for (int w = 0; w < 2; ++w) bwd->bwd_side_active[w] = m->side_active[w];
    if (bwd) WD_CUDA(cudaEventRecord(m->ev_bwd_done, m->stream));
    for (int w = 0; w < 2; ++w) {
        m->side_pending[w] = false;
        m->side_active[w] = bwd && bwd->bwd_side_active[w];
        if (m->side_active[w]) WD_CUDA(cudaStreamWaitEvent(m->sstream[w], m->ev_bwd_done, 0));
    }
    m->grads_pending = bwd != nullptr;
    return WD_OK;
}

// One whole train step on the current slot (three streams, ~55 kernels, no host sync), graphed per slot.
static int train_current(WdModel* m, float* loss_out) {
    GraphRun how;
    int rc = run_train_graphed(m, m->slots[m->cur_slot].train, m->dbatch, [&](bool) { return train_eager(m); }, &how);
    if (rc) return rc;
    if ((rc = after_graph(m, how, nullptr))) return rc;
    if ((rc = mark_slot_used(m))) return rc;
    if (loss_out) return finish_step(m, loss_out, nullptr);
    return WD_OK;
}

extern "C" int wd_train_step_slot(WdModel* m, int slot, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = use_slot(m, slot, "training"))) return rc;
    timer_begin(m);
    return train_current(m, loss_out);
}
extern "C" int wd_train_step_resident(WdModel* m, float* loss_out) { return wd_train_step_slot(m, 0, loss_out); }

extern "C" int wd_train_step(WdModel* m, const WdBatch* b, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = select_slot(m, 0))) return rc;
    timer_begin(m);
    if ((rc = upload_current(m, b))) return rc;
    if ((rc = use_slot(m, 0, "training"))) return rc;
    float dummy;
    return train_current(m, loss_out ? loss_out : &dummy);
}

extern "C" int wd_forward_resident(WdModel* m, float* logits_out, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = select_slot(m, 0))) return rc;
    timer_begin(m);
    if ((rc = forward_core(m, false))) return rc;
    return finish_step(m, loss_out, logits_out);
}

extern "C" int wd_forward(WdModel* m, const WdBatch* b, float* logits_out, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = select_slot(m, 0))) return rc;
    timer_begin(m);
    if ((rc = upload_current(m, b))) return rc;
    if ((rc = forward_core(m, false))) return rc;
    return finish_step(m, loss_out, logits_out);
}


// forward + backward of the current batch; `join` brings the side streams back into the main stream (needed to end a capture)
static int backward_eager(WdModel* m, bool join) {
    int rc;
    if ((rc = forward_core(m, true))) return rc;
    if ((rc = backward_core(m))) return rc;
    if (join)
        for (int w = 0; w < 2; ++w)
            if (m->side_active[w]) {
                WD_CUDA(cudaEventRecord(m->ev_done[w], m->sstream[w]));
                WD_CUDA(cudaStreamWaitEvent(m->stream, m->ev_done[w], 0));
            }
    return WD_OK;
}

// Data-parallel steps run forward + backward, then the exchange (NCCL, outside the library), then merge + apply.  The first part
// is ~65 launches on three streams, graphed per batch slot.  Inside the graph the streams overlap as in the eager schedule; after
// it the sparse lists continue on their side streams, which wait for the graph through ev_bwd_done.
// The split step applies the embedding rows with the unfused kernels, which update host records through their mapped pointers:
// with an HBM cache in front of those records the update would bypass it, and a deferred Adam table's records lag behind the step.
static int refuse_split_step_with_cache(WdModel* m) {
    if (m->hcache.slots == 0 && m->n_defer_tab == 0) return WD_OK;
    set_error("the split step (wd_step_backward / wd_step_apply) is not supported on a model with a host-table cache or with "
              "deferred Adam tables (WD_PLACE_DEFER_ADAM)");
    return WD_EUNSUPPORTED;
}

extern "C" int wd_step_backward_slot(WdModel* m, int slot, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = use_slot(m, slot, "training"))) return rc;
    if ((rc = refuse_split_step_with_cache(m))) return rc;
    timer_begin(m);
    BatchSlot& sl = m->slots[slot];
    GraphRun how;
    if ((rc = run_train_graphed(m, sl.bwd, m->dbatch, [&](bool capturing) { return backward_eager(m, capturing); }, &how))) return rc;
    if ((rc = after_graph(m, how, &sl))) return rc;
    if ((rc = mark_slot_used(m))) return rc;
    if (loss_out) return finish_step(m, loss_out, nullptr);
    return WD_OK;
}

// loss of the most recent forward / train step (synchronises the model stream)
extern "C" int wd_last_loss(WdModel* m, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (!loss_out) { set_error("wd_last_loss: null output"); return WD_EINVAL; }
    return finish_step(m, loss_out, nullptr);
}

extern "C" int wd_step_backward(WdModel* m, const WdBatch* b, float* loss_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = refuse_split_step_with_cache(m))) return rc;
    if (b && (rc = wd_batch_upload(m, b))) return rc;
    timer_begin(m);
    if (!m->dbatch.label) { set_error("training needs labels"); return WD_EINVAL; }
    if ((rc = forward_core(m, true))) return rc;
    if ((rc = backward_core(m))) return rc;
    if (loss_out) return finish_step(m, loss_out, nullptr);
    return WD_OK;
}

extern "C" int wd_step_apply(WdModel* m) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (!m->grads_pending) { set_error("wd_step_apply without wd_step_backward"); return WD_ESTATE; }
    return apply_core(m);
}

extern "C" int64_t wd_dense_grad_count(WdModel* m) { return m ? m->dense_count + m->gs_count : 0; }
extern "C" void* wd_dense_grad_ptr(WdModel* m) { return m ? m->d_G : nullptr; }

extern "C" int wd_sparse_grads(WdModel* m, int which, void** rows, void** grads, int64_t* n, int32_t* width, int64_t* capacity) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (which < 0 || which > 1 || !m->lists[which].urow) { set_error("no sparse gradient list %d", which); return WD_EINVAL; }
    const RowList& l = m->lists[which];
    if (n) {                                   // the count needs a sync; pass n = NULL for the asynchronous fixed-size exchange
        int32_t nu = 0;
        WD_CUDA(cudaStreamSynchronize(m->stream));
        WD_CUDA(cudaStreamSynchronize(m->sstream[which]));
        WD_CUDA(cudaMemcpy(&nu, l.nuniq, 4, cudaMemcpyDeviceToHost));
        *n = nu;
    }
    if (rows) *rows = l.urow;
    if (grads) *grads = l.ugrad;
    if (width) *width = l.width;
    if (capacity) *capacity = m->max_nnz;
    return WD_OK;
}

// n_lists = 0: general (unsorted) list of n rows; n_lists > 0: n_lists sorted, duplicate-free lists of list_len rows each
static int sparse_set_impl(WdModel* m, int which, const void* rows_dev, const void* grads_dev, int64_t n, int n_lists, int64_t list_len) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (which < 0 || which > 1 || !m->lists[which].urow) { set_error("no sparse gradient list %d", which); return WD_EINVAL; }
    const bool side = m->side_active[which];
    auto merge = [&]() -> int {
        return n_lists > 0 ? merge_sparse_sorted(m, which, rows_dev, grads_dev, n_lists, list_len) : merge_sparse(m, which, rows_dev, grads_dev, n);
    };
    auto run = [&](bool) -> int { return side ? on_side(m, which, merge) : merge(); };
    // The count-based exchange changes n, the number of exchanged rows, every step: its merge runs eagerly.  The fixed-size
    // exchange passes the same buffers and shape every step, so its merge (~25 small launches on one stream) is graphed: the
    // data-parallel tail is otherwise bound by the launching thread, not by the GPU.
    if (n_lists == 0) return run(false);
    GraphRun how;
    return run_graphed(m, m->merge_graph[which], MergeKey{rows_dev, grads_dev, n_lists, list_len, side}, side ? m->sstream[which] : m->stream, run, &how);
}

extern "C" int wd_sparse_set(WdModel* m, int which, const void* rows_dev, const void* grads_dev, int64_t n) {
    return sparse_set_impl(m, which, rows_dev, grads_dev, n, 0, 0);
}
extern "C" int wd_sparse_set_sorted(WdModel* m, int which, const void* rows_dev, const void* grads_dev, int32_t n_lists, int64_t list_len) {
    if (n_lists < 1 || list_len < 1) { set_error("wd_sparse_set_sorted: bad list shape"); return WD_EINVAL; }
    return sparse_set_impl(m, which, rows_dev, grads_dev, 0, n_lists, list_len);
}

// ------------------------------------------------------------------------------------- row-sharded tables
static int shard_ready(WdModel* m, int slot, const char* needs_labels) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (m->shard.world <= 1) { set_error("model has no row-sharded tables (shard_world <= 1)"); return WD_ESTATE; }
    if (!m->shard.connected) { set_error("row-sharded model is not connected to its peers (wd_shard_connect_ipc / wd_shard_connect_local)"); return WD_ESTATE; }
    return use_slot(m, slot, needs_labels);
}

// Segment `phase` of the rank-step (ranks driven by ONE process: the caller runs segment k on every rank, then wd_shard_local_sync).
extern "C" int wd_shard_phase(WdModel* m, int slot, int phase, int train) {
    int rc = shard_ready(m, slot, train ? "training" : nullptr);
    if (rc) return rc;
    if (m->shard.ipc) { set_error("wd_shard_phase is for ranks of one process; multi-process ranks call wd_shard_train_step_slot"); return WD_ESTATE; }
    if (phase < 0 || phase > 4) { set_error("wd_shard_phase: phase %d outside [0, 4]", phase); return WD_EINVAL; }
    if (phase == 0) timer_begin(m);
    if ((rc = shard_step(m, train != 0, phase))) return rc;
    return train && phase == 4 ? mark_slot_used(m) : WD_OK;
}

// Loss (and optionally logits) of the step / forward just issued; synchronises the model stream.
extern "C" int wd_shard_finish(WdModel* m, float* loss_out, float* logits_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    return finish_step(m, loss_out, logits_out);
}

// The whole step of one rank of a multi-process job: ids, routing, serve, combine, towers, owners' updates, dense all-reduce and
// optimizers, with flag barriers in peer memory between the segments.  Every rank must call it once per step (it is a collective).
// Graphed per batch slot, barrier kernels included.
extern "C" int wd_shard_train_step_slot(WdModel* m, int slot, float* loss_out) {
    int rc = shard_ready(m, slot, "training");
    if (rc) return rc;
    if (!m->shard.ipc) { set_error("wd_shard_train_step_slot needs wd_shard_connect_ipc (ranks of one process use wd_shard_phase)"); return WD_ESTATE; }
    timer_begin(m);
    GraphRun how;
    if ((rc = run_train_graphed(m, m->slots[slot].shard, m->dbatch, [&](bool) { return shard_step(m, true, kAllSegments); }, &how))) return rc;
    if ((rc = after_graph(m, how, nullptr))) return rc;
    if ((rc = mark_slot_used(m))) return rc;
    if (loss_out) return finish_step(m, loss_out, nullptr);
    return WD_OK;
}

// Forward only on a sharded model (collective, multi-process ranks): logits of this rank's batch shard.
extern "C" int wd_shard_forward_slot(WdModel* m, int slot, float* logits_out, float* loss_out) {
    int rc = shard_ready(m, slot, nullptr);
    if (rc) return rc;
    if (!m->shard.ipc) { set_error("wd_shard_forward_slot needs wd_shard_connect_ipc"); return WD_ESTATE; }
    if ((rc = shard_step(m, false, kAllSegments))) return rc;
    return finish_step(m, loss_out, logits_out);
}

// ---- evaluation of a row-sharded model: every rank adds the metrics of its own rows to its accumulator (wd_eval_reset /
// wd_eval_finish: this rank's alone), then one collective sums the accumulators of all ranks
namespace wd { int shard_metrics_reduce(WdModel* m); }

static int check_eval_rows(WdModel* m, int32_t n_valid) {
    if (n_valid < 0 || n_valid > m->dbatch.B) { set_error("n_valid %d outside [0, batch size %d]", n_valid, m->dbatch.B); return WD_EINVAL; }
    if (n_valid > 0 && !m->dbatch.label) { set_error("evaluation needs labels"); return WD_EINVAL; }
    return WD_OK;
}

// Collective (multi-process ranks): the sharded forward of the slot's batch, then the metrics of its first n_valid rows, all on the
// device.  A rank without rows left enters with any one-row batch and n_valid = 0: its forward still serves its peers.  Graphed per
// batch slot and n_valid.
extern "C" int wd_shard_eval_accumulate_slot(WdModel* m, int slot, int32_t n_valid) {
    int rc = shard_ready(m, slot, nullptr);
    if (rc) return rc;
    if (!m->shard.ipc) { set_error("wd_shard_eval_accumulate_slot needs wd_shard_connect_ipc (ranks of one process use wd_shard_phase + wd_shard_eval_accumulate_phase)"); return WD_ESTATE; }
    if ((rc = check_eval_rows(m, n_valid))) return rc;
    auto issue = [&](bool) { int r = shard_step(m, false, kAllSegments); return r ? r : metrics_accumulate(m, n_valid); };
    GraphRun how;
    if ((rc = run_graphed(m, m->slots[slot].shard_eval, ShardEvalKey{m->dbatch, n_valid}, m->stream, issue, &how))) return rc;
    if (how == GraphRun::replayed) m->eval_batches++;        // (a capture ran the issuing code, which advanced it)
    if ((rc = mark_slot_used(m))) return rc;
    return finish_step(m, nullptr, nullptr);
}

// Ranks of one process: after segments 0..2 of wd_shard_phase(train = 0) on every rank, the metrics of the first n_valid rows of
// this rank's logits.
extern "C" int wd_shard_eval_accumulate_phase(WdModel* m, int32_t n_valid) {
    int rc = shard_ready(m, m->cur_slot, nullptr);
    if (rc) return rc;
    if (m->shard.ipc) { set_error("wd_shard_eval_accumulate_phase is for ranks of one process; multi-process ranks call wd_shard_eval_accumulate_slot"); return WD_ESTATE; }
    if ((rc = check_eval_rows(m, n_valid))) return rc;
    return metrics_accumulate(m, n_valid);
}

// Collective: the ten metrics of every rank's rows, identical bytes on every rank.  Multi-process ranks meet at flag barriers
// inside; ranks of one process call wd_shard_local_sync after their last accumulate, then this on every rank.
extern "C" int wd_shard_eval_finish(WdModel* m, double* out10) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (!out10) { set_error("wd_shard_eval_finish: null output"); return WD_EINVAL; }
    if (m->shard.world <= 1) { set_error("model has no row-sharded tables (shard_world <= 1)"); return WD_ESTATE; }
    if (!m->shard.connected) { set_error("row-sharded model is not connected to its peers (wd_shard_connect_ipc / wd_shard_connect_local)"); return WD_ESTATE; }
    if ((rc = shard_metrics_reduce(m))) return rc;
    if ((rc = finish_step(m, nullptr, nullptr))) return rc;          // (a peer that never arrived shows in the flags)
    return metrics_finish(m, m->shard.d_msum, out10);
}

// ------------------------------------------------------------------------------------------------- eval
extern "C" int wd_eval_reset(WdModel* m) {
    int rc = check_ready(m);
    if (rc) return rc;
    WD_CUDA(cudaMemsetAsync(m->d_metrics, 0, kMetricsDoubles * sizeof(double), m->stream));
    m->eval_batches = 0;
    return WD_OK;
}
extern "C" int wd_eval_accumulate(WdModel* m, const WdBatch* b) {
    int rc = wd_batch_upload(m, b);
    if (rc) return rc;
    if (!m->dbatch.label) { set_error("evaluation needs labels"); return WD_EINVAL; }
    if ((rc = forward_core(m, false))) return rc;
    if ((rc = metrics_accumulate(m, m->dbatch.B))) return rc;
    return finish_step(m, nullptr, nullptr);
}
extern "C" int wd_eval_accumulate_slot(WdModel* m, int slot) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = use_slot(m, slot, "evaluation"))) return rc;
    if ((rc = forward_core(m, false))) return rc;
    if ((rc = metrics_accumulate(m, m->dbatch.B))) return rc;
    if ((rc = mark_slot_used(m))) return rc;
    return finish_step(m, nullptr, nullptr);
}
extern "C" int wd_eval_finish(WdModel* m, double* out10) {
    int rc = check_ready(m);
    if (rc) return rc;
    return metrics_finish(m, m->d_metrics, out10);
}

// ------------------------------------------------------------------------------------------ debug / misc
extern "C" int wd_debug_column_ids(WdModel* m, int32_t* offsets_out, int64_t offsets_cap, int64_t* ids_out, int64_t ids_cap, int64_t* nnz_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    int64_t no = (int64_t)m->dbatch.B * m->n_columns + 1;
    int32_t nnz = 0;
    WD_CUDA(cudaMemcpy(&nnz, m->d_nnz, 4, cudaMemcpyDeviceToHost));
    if (nnz_out) *nnz_out = nnz;
    if (offsets_out) {
        if (offsets_cap < no) { set_error("offsets buffer too small"); return WD_EINVAL; }
        WD_CUDA(cudaMemcpy(offsets_out, m->d_col_offs, no * 4, cudaMemcpyDeviceToHost));
    }
    if (ids_out) {
        if (ids_cap < nnz) { set_error("ids buffer too small"); return WD_EINVAL; }
        std::vector<int32_t> tmp(nnz);
        WD_CUDA(cudaMemcpy(tmp.data(), m->d_e_id, (int64_t)nnz * 4, cudaMemcpyDeviceToHost));
        for (int i = 0; i < nnz; ++i) ids_out[i] = tmp[i];
    }
    return WD_OK;
}
// The batch a slot holds, read back (after its pending upload or parse): *batch_out rows, *nnz_out keys, *parts_out bit 0 offsets,
// bit 1 label, bit 2 weight present.  Arrays that are not NULL receive offsets [B * F + 1], keys [nnz], dense [B * Nd], label [B],
// weight [B]; pass NULLs first to learn the sizes.
extern "C" int wd_debug_slot(WdModel* m, int slot, int32_t* batch_out, int64_t* nnz_out, int32_t* parts_out, int32_t* offsets_out,
                             uint64_t* keys_out, float* dense_out, float* label_out, float* weight_out) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (slot < 0 || slot >= (int)m->slots.size() || !m->slots[slot].filled) { set_error("batch slot %d was never uploaded", slot); return WD_ESTATE; }
    WD_CUDA(cudaStreamSynchronize(m->stream_up));
    WD_CUDA(cudaStreamSynchronize(m->stream));
    const BatchSlot& sl = m->slots[slot];
    const DevBatch& v = sl.view;
    const int64_t B = v.B, F = m->n_cat_fields, Nd = m->n_dense_fields;
    int32_t nnz32 = (int32_t)(B * F);
    if (v.cat_offsets) WD_CUDA(cudaMemcpy(&nnz32, v.cat_offsets + B * F, 4, cudaMemcpyDeviceToHost));
    if (batch_out) *batch_out = (int32_t)B;
    if (nnz_out) *nnz_out = nnz32;
    if (parts_out) *parts_out = (v.cat_offsets ? 1 : 0) | (v.label ? 2 : 0) | (v.weight ? 4 : 0);
    if (offsets_out && v.cat_offsets) WD_CUDA(cudaMemcpy(offsets_out, v.cat_offsets, (B * F + 1) * 4, cudaMemcpyDeviceToHost));
    if (keys_out && nnz32 > 0) WD_CUDA(cudaMemcpy(keys_out, v.cat_keys, (int64_t)nnz32 * 8, cudaMemcpyDeviceToHost));
    if (dense_out && Nd > 0) WD_CUDA(cudaMemcpy(dense_out, v.dense, B * Nd * 4, cudaMemcpyDeviceToHost));
    if (label_out && v.label) WD_CUDA(cudaMemcpy(label_out, v.label, B * 4, cudaMemcpyDeviceToHost));
    if (weight_out && v.weight) WD_CUDA(cudaMemcpy(weight_out, v.weight, B * 4, cudaMemcpyDeviceToHost));
    return WD_OK;
}
extern "C" int wd_debug_deep_input(WdModel* m, float* out, int64_t cap) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (!m->use_deep) { set_error("model has no deep part"); return WD_EINVAL; }
    int64_t n = (int64_t)m->dbatch.B * m->d0_phys;
    if (cap < n) { set_error("buffer too small"); return WD_EINVAL; }
    WD_CUDA(cudaStreamSynchronize(m->stream));
    WD_CUDA(cudaMemcpy(out, m->d_X0, n * 4, cudaMemcpyDeviceToHost));
    return WD_OK;
}
extern "C" int wd_debug_hidden(WdModel* m, int tower, int layer, float* out, int64_t cap) {
    int rc = check_ready(m);
    if (rc) return rc;
    if (tower < 0 || tower >= (int)m->towers.size() || layer < 0 || layer >= m->towers[tower].n_hidden) { set_error("no such hidden layer"); return WD_EINVAL; }
    Layer& L = m->towers[tower].layers[layer];
    int64_t n = (int64_t)m->dbatch.B * L.N_phys;
    if (cap < n) { set_error("buffer too small"); return WD_EINVAL; }
    WD_CUDA(cudaStreamSynchronize(m->stream));
    if (!L.H) {
        // no fp32 copy of this layer: hi + lo of its bf16 copies, the value the next layer's GEMM reads
        std::vector<__nv_bfloat16> hi(n), lo(n);
        WD_CUDA(cudaMemcpy(hi.data(), L.Hs[0], n * sizeof(__nv_bfloat16), cudaMemcpyDeviceToHost));
        WD_CUDA(cudaMemcpy(lo.data(), L.Hs[1], n * sizeof(__nv_bfloat16), cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < n; ++i) out[i] = __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
        return L.N_phys;
    }
    WD_CUDA(cudaMemcpy(out, L.H, n * 4, cudaMemcpyDeviceToHost));
    return L.N_phys;
}
extern "C" int64_t wd_launch_count(WdModel* m) { return m ? m->launches : 0; }

// ------------------------------------------------------------------------------------------ layer summaries (summary.cu)
extern "C" int wd_summary_segments(WdModel* m, int32_t* kind, int32_t* tower, int32_t* layer, int32_t cap) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = summary_prepare(m, m->x0_real))) return rc;
    const SummaryState* S = m->summ;
    const int n = (int)S->h.size();
    for (int i = 0; i < n && i < cap; ++i) {
        if (kind) kind[i] = S->kind[i];
        if (tower) tower[i] = S->tower[i];
        if (layer) layer[i] = S->layer[i];
    }
    return n;
}
extern "C" int wd_summary_arm(WdModel* m) {
    int rc = check_ready(m);
    if (rc) return rc;
    if ((rc = summary_prepare(m, m->x0_real))) return rc;
    m->summary_armed = true;
    return WD_OK;
}
extern "C" int64_t wd_gemm_fallback_count(WdModel* m) { return m ? m->gemm_fallbacks : 0; }
extern "C" int wd_graph_stats(WdModel* m, int64_t* out, int32_t n) {
    if (!m || !out || n < 2) { wd::set_error("wd_graph_stats: bad arguments"); return WD_EINVAL; }
    out[0] = m->graph_captures;
    out[1] = m->graph_replays;
    return WD_OK;
}
extern "C" int wd_last_timings(WdModel* m, float* ms_out, int cap) {
    if (!m) return WD_EINVAL;
    int n = m->timer.n_last;
    for (int i = 0; i < n && i < cap; ++i) ms_out[i] = m->timer.ms[i];
    return n;
}
extern "C" const char* wd_timing_name(WdModel* m, int i) {
    if (!m || i < 0 || i >= m->timer.n_last) return "";
    return i == 0 ? "total" : m->timer.name[i];
}
extern "C" int wd_set_profile(WdModel* m, int enable) {
    if (!m) return WD_EINVAL;
    m->timer.enabled = enable != 0;
    return WD_OK;
}
extern "C" void* wd_stream(WdModel* m) { return m ? (void*)m->stream : nullptr; }
extern "C" void* wd_stream_sparse(WdModel* m, int which) {
    if (!m) return nullptr;
    return (which >= 0 && which < 2 && m->side_active[which]) ? (void*)m->sstream[which] : (void*)m->stream;
}
extern "C" int wd_sync(WdModel* m) {
    int rc = check_ready(m);
    if (rc) return rc;
    WD_CUDA(cudaStreamSynchronize(m->stream));
    return WD_OK;
}

// debugging aid (not part of the public header): stamps of the last train step's timeline (ns, globaltimer), WD_STEP_TRACE=1:
// [start, ids, gather, head, towers' backward, main stream end, grouping 0 / 1 end, reduce 0 begin / end, reduce 1 begin / end,
// apply 0 / 1 end] (0 = embedding rows, 1 = wide rows; side streams)
extern "C" int wd_debug_step_trace(WdModel* m, unsigned long long* out) {
    if (!m || !m->d_step_trace) return -1;
    cudaDeviceSynchronize();
    return cudaMemcpy(out, m->d_step_trace, sizeof(unsigned long long) * 16, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}
