// Shared declarations of libwd_b200: host-side model object, device plan tables, launch helpers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/wd_b200.h"

namespace wd {

constexpr int kSortTile = 1024;          // keys per radix-sort tile (sort.cu); sizes the per-tile histogram scratch

void set_error(const char* fmt, ...);

#define WD_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            wd::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return WD_ECUDA;                                                                  \
        }                                                                                     \
    } while (0)

constexpr uint32_t kInvalidRow = 0xFFFFFFFFu;
constexpr int kMaxSegs = 8;      // sources concatenated into one MLP layer input
constexpr int kMaxTowers = 8;    // deep towers per model: the head kernel takes all of their logits layers as one parameter block
constexpr int kNumSms = 132;     // SMs of an H100 SXM: the grid caps of the grid-stride kernels are sized by it
constexpr int kMaxDims = 8;      // distinct embedding widths per model
// sparse row lists (RowList, WdModel::lists): 0 embedding rows and 1 wide rows of the replicated tables; row-sharded tables add
// 2 / 3 = rows this rank OWNS that were touched by any rank this step (embedding / wide) and 4 / 5 = this rank's own ids
// grouped by owner rank (routing; only the key / value ping-pong buffers exist)
constexpr int kLists = 6;
constexpr int kMaxRanks = 16;    // ranks of one box a row-sharded table can be split over
constexpr int kMetricsDoubles = 512;  // doubles of an eval metric accumulator (layout: misc.cu)

// ---- device image of the categorical-column plan (all pointers are device pointers)
struct DevPlan {
    int n_cat_fields, n_dense_fields, n_columns;
    const uint8_t* field_is_string;
    const int32_t* col_kind;
    const int32_t* col_field;
    const int64_t* col_buckets;
    const int32_t* col_aux_off;
    const int32_t* col_aux_n;
    const int32_t* col_norm_kind;
    const float* col_norm_a;
    const float* col_norm_b;
    const int64_t* col_wide_base;
    const int32_t* col_emb_table;
    const int32_t* col_ind_off;
    const uint64_t* vocab_fp;
    const float* boundaries;
    const int32_t* cross_key_type;
    const int32_t* cross_key_idx;
    const int64_t* table_row_base;   // global embedding row id of row 0 of each table
    int d0_phys;
    // row-sharded tables (shard_world > 1): per column the slot in the sharded embedding / wide space (-1: replicated), the first
    // local row of each slot's shard, and per entry the owner rank / local row arrays the id stage fills (null: nothing sharded)
    int sh_world;
    const int32_t *sh_col_emb, *sh_col_wide;
    const int64_t *sh_base_emb, *sh_base_wide;
    uint32_t *sh_own_emb, *sh_lrow_emb, *sh_own_wide, *sh_lrow_wide;
};

// ---- device view of one batch
struct DevBatch {
    int B;
    const int32_t* cat_offsets;      // may be null: one key per (row, field)
    const uint64_t* cat_keys;
    const float* dense;
    const float* label;              // may be null
    const float* weight;             // may be null
};

struct EmbTable {
    int64_t rows;
    int dim;                 // physical width (multiple of 4)
    int dim_logical;         // embedding_column dimension; columns [dim_logical, dim) are zero padding
    int x0_off;
    int col;                 // producing column
    int64_t row_base;        // global row id base
    int64_t gs_off;          // small (dense-exchanged) table: float offset of its gradients in the small-table block; else -1
    float* data;            // arows * stride floats; record = [w[dim] | slot1[dim] | slot2[dim]] (+ stamp: see defer)
    int stride;              // dim * (1 + nslots), + 4 with defer
    bool sharded;            // row-sharded over the ranks: this rank holds rows r with r mod G == rank at local index r / G
    int64_t arows;           // rows allocated on this rank (= rows unless sharded); row_base then counts in the shard's row space
    int place;               // requested placement WD_PLACE_*
    bool host;               // records live in mapped page-locked host memory (staged through HBM every step, host_tables.cu)
    // WD_PLACE_DEFER_ADAM with the Adam dnn optimizer: record [w | m | v | stamp float4], lane 0 of the stamp = the last Adam step
    // the record reflects; on the host (deferred()) the untouched pass skips the table and rows catch up when staged (host_tables.cu)
    bool defer;
};
inline bool deferred(const EmbTable& tb) { return tb.host && tb.defer; }

struct TabDesc {            // per-table descriptor grouped by width (one 32-byte load in the gather kernels)
    float* data;
    int64_t row_base;
    int stride, x0, col, dim;
};

// Where the [w | s1 | s2] records of a set of embedding tables are.  Tables t < ntab with first row row_base[t] (ascending in a
// row-ordered set), records of stride[t] floats at data[t].  A staged table (stage[t] != 0; stage null: none is) keeps the records
// of the step's rows in stage_base instead, unique row u at staging row uslot[u] (u without a cache) with stride stage[t].
struct RowRecords {
    int ntab;
    const int64_t* row_base;
    float* const* data;
    const int32_t* dim;
    const int32_t* stride;
    const int32_t* stage;
    float* stage_base;
    const int32_t* uslot;
};
// One record set's device descriptors (the sets and who reads them: table at the top of host_tables.cu); per-table arrays a set
// does not need are null.
struct RecordSet {
    RowRecords rec{};
    const int32_t* x0 = nullptr;      // [ntab] offset of the table's slice in the deep input
    const int64_t* rows = nullptr;    // [ntab] rows of the table this set holds on this rank
    const int64_t* gs_off = nullptr;  // [ntab] float offset inside the small-table gradient block (-1: large table)
};

// HBM cache of the host records of one record set (host_tables.cu): the single-GPU cache in front of the replicated set
// (WdModel::hcache, list 0, global rows) or an owner's cache of its host shards (ShardSpace::cache, list 2, shard rows).  The
// set's staging buffer is then [slots | overflow rows]; a model has at most one cache.
struct HostCache {
    int64_t slots = 0;                       // C = 8 x 2^set_bits; 0: no cache (every staged row is an overflow row)
    int set_bits = 0;
    uint32_t* d_tag = nullptr;               // [C] row held by the slot (the set's row space), kInvalidRow: empty
    uint32_t* d_stamp = nullptr;             // [C] stamp of the last call that used the slot (0: empty)
    uint8_t* d_dirty = nullptr;              // [C] 1: the slot is newer than its host record
    uint32_t* d_now = nullptr;               // device counter, bumped once per stage-in (the stamp of that call)
    unsigned long long* d_stats = nullptr;   // [4] hits, loads, overflow rows, dirty evictions
    int32_t* d_uslot = nullptr;              // [rows] staging row of unique row u; null without a cache (row u)
    uint32_t* d_uvict = nullptr;             // [rows] row the slot of u held before u was loaded into it
    uint8_t* d_uflag = nullptr;              // [rows] kLoad / kVictimDirty (host_tables.cu)
    uint32_t *d_ck[2] = {}, *d_cv[2] = {};   // (set, u) pairs and their sort ping-pong buffers
};

// The sort and unique-row scratch of one set of touched rows (kLists), allocated by list_alloc; a routing list's non-key pointers stay null
struct RowList {
    uint32_t *keys = nullptr, *vals = nullptr;     // [max_nnz + 8] (row, occurrence) pairs; sorted pairs end here
    uint32_t *keys2 = nullptr, *vals2 = nullptr;   // their ping-pong copies
    uint32_t* urow = nullptr;                      // unique rows, ascending
    int32_t* ustart = nullptr;                     // segment starts in the sorted list (+1 sentinel)
    int32_t* choff = nullptr;                      // chunk offsets of hot rows (exclusive scan)
    float* ugrad = nullptr;                        // [max_nnz + 8][width] summed gradient of each unique row
    float* cpart = nullptr;                        // [chunk_cap(max_nnz)][width] chunk partial sums
    // device scalars: unique rows, entries of a merged external list, hot-row chunks, and (lists 0 / 1) unique rows below
    // small_base (what stays in the list)
    int32_t *nuniq = nullptr, *nvalid = nullptr, *nchunks = nullptr, *nubig = nullptr;
    int bits = 0, width = 0;                       // key bits of the row space (the invalid key 1 << bits sorts last); floats per ugrad row
    bool fused = false;                            // this step's rows were updated by the list's gradient-sum / combine launches (sparse.cu)
};
// one stream's scan / sort scratch (on_stream): scan chunk sums, radix-sort histograms [sort_hist_cap], finished scan blocks
struct SortScratch { int32_t *scan = nullptr, *hist = nullptr, *counter = nullptr; };

struct DenseTensor {         // one trainable dense tensor inside the dense arena
    int64_t off;             // offset in arena (floats)
    int64_t count;           // physical element count
    int rows, cols;          // physical shape (rows = K_phys for kernels, 1 for vectors)
    // gradient partials: grad[i] = sum_p gpart[p * gstride + i]
    int64_t gpart_off;       // offset in the partial buffer
    int gparts;
    int g_rowtiles;          // 1: partials are per 128-row batch tile (only the tiles of the current batch are live)
    int64_t gstride;
    int64_t wt_off;          // offset in each GEMM weight copy (WdModel::d_Wt ... d_Wq_lo), -1 if none
    int mirror_u;            // crelu layers (kernel, bias): column n + mirror_u holds minus column n, n < mirror_u (0: plain tensor)
};

// Stored operand forms the MLP GEMMs read (table at the top of mlp.cu): fp32 and transposed fp32 copies for the ffma, tc1x and
// tc3x engines, bf16 hi / lo copies for bf16x3.  A model allocates and writes only its family's copies.
enum OperandFamily { kFp32Operands = 0, kBf16Operands = 1 };

struct Seg {                 // one source of a layer input
    int src;                 // -1: deep input x, >=0: hidden layer index of the same tower
    int width;               // logical width
    int width_phys;          // padded to 32
    int k_off;               // physical row offset inside the layer's kernel
};

struct Layer {
    int n_in_segs;
    Seg segs[kMaxSegs];
    int K, K_phys;           // logical / physical input width
    int N, N_phys;           // logical / physical output width (1 for logits)
    int N_param;             // logical columns of kernel / bias: N, or N / 2 for a crelu layer (the other half mirrors them)
    int t_kernel, t_bias, t_gamma, t_beta;   // indices into Model::dense (-1 if absent)
    int wgrad_splits;        // split-K factor of this layer's weight gradient (= gparts of its kernel tensor)
    // activations (hidden layers only), all [max_batch_pad, N_phys] unless noted; null where the model's operand family has no
    // such copy (table at the top of mlp.cu)
    float* A;                // post-activation (pre-BN); the same buffer as H when neither batch norm nor dropout sits between them
    float* H;                // layer output (bf16 family: only for layers the logits layer reads)
    float* HT;               // fp32 family: transposed output [N_phys, ldt]
    float* dH;               // gradient w.r.t. H (accumulated over consumers)
    float* dZ;               // fp32 family: gradient w.r.t. pre-activation
    float* dZT;              // fp32 family: transposed [N_phys, ldt]
    __nv_bfloat16 *Hs[2], *dZs[2];   // bf16 family: hi / lo copies of H and dZ
    float* colpart;          // [3][row_tiles][N_phys] partial column sums: dbias, dgamma, dbeta
};

struct Tower {
    int n_hidden;
    int mode;
    std::vector<Layer> layers;   // n_hidden hidden layers + 1 logits layer
    float* logit;                // [max_batch]
};

struct PhaseTimer {          // named CUDA-event marks on the model stream (wd_set_profile)
    static constexpr int kMax = 160;
    cudaEvent_t ev[kMax];
    const char* name[kMax];
    float ms[kMax];
    int n = 0, n_last = 0;
    bool enabled = false;
};

// A CUDA graph of step work (api.cu run_graphed), replayed only while the key it was captured with stays equal.
template <class Key>
struct StepGraph {
    cudaGraphExec_t exec = nullptr;
    Key key{};
    int64_t launches = 0;    // kernel launches the capture recorded (added to WdModel::launches on every replay)
    int eager = 0;           // eager runs so far
    void destroy() {
        if (exec) cudaGraphExecDestroy(exec);
        exec = nullptr;
    }
};
// key of a slot's step graphs: the batch view (a slot re-uploaded with the same B, labels and weights keeps its graphs)
inline bool operator==(const DevBatch& a, const DevBatch& b) {
    return a.B == b.B && a.cat_offsets == b.cat_offsets && a.cat_keys == b.cat_keys && a.dense == b.dense && a.label == b.label && a.weight == b.weight;
}
struct MergeKey {            // key of a list's merge graph (wd_sparse_set_sorted)
    const void* rows;
    const void* grads;
    int n_lists;
    int64_t list_len;
    bool on_side;
    bool operator==(const MergeKey& o) const {
        return rows == o.rows && grads == o.grads && n_lists == o.n_lists && list_len == o.list_len && on_side == o.on_side;
    }
};

struct ShardEvalKey {        // key of a slot's eval graph on a row-sharded model (wd_shard_eval_accumulate_slot)
    DevBatch b;
    int n_valid;
    bool operator==(const ShardEvalKey& o) const { return b == o.b && n_valid == o.n_valid; }
};

struct BatchSlot {           // one device-resident batch (ring used by benchmarks / prefetch)
    int32_t* off = nullptr;
    uint64_t* keys = nullptr;
    float *dense = nullptr, *label = nullptr, *weight = nullptr;
    DevBatch view{};
    bool filled = false;
    // asynchronous refill (wd_batch_prefetch_slot): copies run on the upload stream between these two events
    cudaEvent_t ev_up = nullptr;             // recorded on the upload stream after the slot's copies
    cudaEvent_t ev_used = nullptr;           // recorded on the model stream after the last step that read the slot
    bool up_pending = false, used_recorded = false;
    // step graphs on this slot, one per entry point
    StepGraph<DevBatch> train;               // whole train step (wd_train_step_slot)
    StepGraph<DevBatch> bwd;                 // forward + backward of the split step (wd_step_backward_slot), side streams joined at its end
    StepGraph<DevBatch> shard;               // whole rank-step of a row-sharded model (wd_shard_train_step_slot)
    StepGraph<ShardEvalKey> shard_eval;      // sharded forward + metrics of its first n_valid rows (wd_shard_eval_accumulate_slot)
    bool bwd_side_active[2] = {false, false};   // side_active as the captured backward left it
};


// ---- row-sharded tables (shard.cu) ------------------------------------------------------------------------------------
// Pointers into ONE rank's exchange segment (a single cudaMalloc block that peers map through CUDA IPC, or address directly when
// all ranks live in one process).  Every rank lays its segment out identically, so a peer pointer = peer base + own offset.
struct ShardPeer {
    uint2* inbox;             // [G][pair_cap] entries {local row, bag} written by requester ranks
    int32_t* inbox_cnt;       // [G] entries each requester sent this step
    float* recv;              // [G][nbags][width] pooled partial sums written by owner ranks
    const float* bagscale;    // [nbags] 1 / (ids in the bag)   (embedding space: combiner = mean)
    const float* gradbase;    // dX0 (embedding space) / dlogit (wide space) of that rank: owners pull gradients from here
};
struct ShardSpace {           // one sharded table space on this rank: 0 = embedding tables, 1 = wide columns
    bool on = false;
    int width = 0;            // floats per pooled vector: max width of the sharded embedding tables / 1
    int n_slots = 0;          // sharded tables (embedding) / sharded wide columns
    int bags_per_row = 0;     // embedding: n_slots (bag = example * n_slots + slot); wide: 1 (bag = example)
    int64_t nbags_cap = 0;    // max_batch * bags_per_row
    int64_t local_rows = 0;   // rows of this rank's shard of the space
    int64_t pair_cap = 0;     // entries one rank may send to one owner per step
    std::vector<int32_t> h_col_slot;   // host copies (tensor IO)
    std::vector<int64_t> h_slot_base;
    int32_t* d_col_slot = nullptr;     // [n_columns] slot fed by column c, -1
    // the slots' records in slot order, row bases in the shard's row space (the shard set, host_tables.cu); the wide space fills
    // only rec.row_base: the first local row of each column's shard
    RecordSet set;
    uint32_t* d_adam_touched = nullptr;   // Adam: [ceil(local_rows / 32)] bit r: local row r was updated this step (sparse_dev.cuh)
    // host-placed shards (embedding space): the owner stages the records of the step's unique owned host rows (list 2) in HBM,
    // record of unique row u at staging row u (set.rec.stage: 0 for an HBM slot), or at cache.d_uslot[u] with a cache
    int stage_stride = 0;              // widest stride of the space's host slots; 0: every shard in HBM (place_tables)
    float* d_stage = nullptr;          // [cache.slots + max_nnz + 1][stage_stride] owner staging buffer (place_tables)
    HostCache cache;                   // wd_shard_cache_enable: HBM cache of this rank's host shard records
    float4* d_wide = nullptr;          // wide space: {w, n, z, -} per local row
    uint32_t* d_own = nullptr;         // [max_nnz] owner rank of entry j or kInvalidRow (not a sharded column)
    uint32_t* d_lrow = nullptr;        // [max_nnz] local row at the owner
    int32_t* d_ostart = nullptr;       // [G + 1] start of each owner's run in the routed (owner-sorted) list
    int32_t* d_bagmask = nullptr;      // [nbags] bit o: owner o holds a partial sum of the bag
    uint32_t* d_rtag = nullptr;        // owner side, per received entry: (source rank << 27) | bag
    uint32_t* d_rrow = nullptr;        // owner side, per received entry: local row
    int32_t* d_nrecv = nullptr;        // device scalar
    ShardPeer* d_peers = nullptr;      // [G] device copy
    ShardPeer peers[kMaxRanks];        // host copy (pointers are device addresses)
    int64_t off_inbox = 0, off_cnt = 0, off_recv = 0, off_bagscale = 0, off_grad = 0;   // offsets in the segment
};
struct ShardState {
    int world = 1, rank = 0;
    bool connected = false, ipc = false;
    uint8_t* seg = nullptr;            // this rank's exchange segment
    int64_t seg_bytes = 0;
    uint8_t* peer_seg[kMaxRanks] = {};
    ShardSpace sp[2];
    // flag barriers: flags[k][r] = last epoch rank r signalled on barrier k (written by rank r, through peer memory)
    int64_t off_flags = 0, off_gred = 0, off_G = 0;
    int64_t off_metrics = 0;            // this rank's eval metric accumulator (WdModel::d_metrics points here)
    double* d_msum = nullptr;           // [kMetricsDoubles] every rank's accumulator summed in rank order (wd_shard_eval_finish)
    uint32_t** d_peer_flags = nullptr;  // [G] device array of peers' flag blocks
    uint32_t* d_epoch = nullptr;        // [kBarriers] local epoch counters
    unsigned long long* d_trace = nullptr;   // WD_SHARD_TRACE=1: [kBarriers][2] enter / leave stamps of the last step's barriers
    float** d_peer_G = nullptr;         // [G] peers' dense gradient arenas
    float** d_peer_gred = nullptr;      // [G] peers' reduced slices
    float* gred = nullptr;              // this rank's reduced slice buffer (whole-arena sized; only the own slice is written)
    int64_t ar_count = 0;               // floats all-reduced per step (dense gradients + small-table block)
    cudaEvent_t ev_a = nullptr;         // after barrier A on the main stream (owner-side grouping may start)
    cudaStream_t aux = nullptr;         // the wide space's routing / serving and the local gathers, beside the embedding space's chain
    cudaEvent_t ev_ids2 = nullptr, ev_routed1 = nullptr, ev_a2 = nullptr, ev_aux_done = nullptr;
};
constexpr int kBarriers = 8;
constexpr int kAllSegments = -1;             // shard_step (shard.cu): every segment of the rank-step

// ---- layer summaries (summary.cu)
constexpr int kSummaryThreads = 256;
constexpr int kSummaryZeroBucket = (WD_SUMMARY_BUCKETS + 1) / 2;   // bucket of 0.0: the first limit above it (1e-12)
struct SummarySeg {          // one segment of the statistics kernel: a [B, cols] tensor read in place
    int kind;                // WD_SEG_*
    const float* ptr; int ld, cols;
    const uint8_t* mask;     // [cols] 1 = a real column (the deep input's logical columns), null: every column
    const float *gamma, *beta; int bn;   // hidden layers: BN affine
    float drop_rate; int layer_id;       //   and dropout (DropArgs)
    unsigned int drop_row0;
    int blk0, nblk;          // the segment's blocks in the grid
};
struct SummaryState {
    std::vector<SummarySeg> h;              // segments in wd_summary_segments order
    std::vector<int32_t> kind, tower, layer;
    int blocks = 0;                         // grid of the statistics kernel
    SummarySeg* d_seg = nullptr;
    uint8_t* d_mask = nullptr;
    double* d_limits = nullptr;             // [WD_SUMMARY_BUCKETS]
    unsigned long long* d_counts = nullptr; // [segments][WD_SUMMARY_BUCKETS]
    double* d_part = nullptr;               // [blocks][4] sum, sum of squares, min, max
    long long* d_ipart = nullptr;           // [blocks][3] values, zeros, non-finite values
};

struct TsvDev;                                 // device TSV parser: spec copy and scratch (tsv.cu)

struct DevAlloc { void* p; int64_t bytes; };   // one cudaMalloc of the model (dev_alloc / dev_free)

}  // namespace wd

struct WdModel {
    // ---- host copy of the plan
    int device = 0;
    bool use_wide = false, use_deep = false;
    int n_cat_fields = 0, n_dense_fields = 0, n_columns = 0;
    std::vector<int32_t> col_kind, col_field, col_aux_off, col_aux_n, col_norm_kind, col_emb_table, col_ind_off;
    std::vector<int64_t> col_buckets, col_wide_base;
    std::vector<float> col_norm_a, col_norm_b;
    int n_numeric = 0;
    int d0_phys = 0;
    int64_t wide_rows = 0;
    int activation = 0, batch_norm = 0;
    WdOptimizer lin_opt{}, dnn_opt{};
    int max_batch = 0, max_batch_pad = 0;   // pad: multiple of 128 (leading dim of transposed buffers)
    int64_t max_nnz = 0;
    int gemm_engine = 0;
    wd::OperandFamily operands = wd::kFp32Operands;   // of gemm_engine, decided in wd_model_create

    cudaStream_t stream = nullptr;
    // side streams, one per sparse gradient list (0 = embedding rows, 1 = wide rows): the id-only grouping, the gradient sums,
    // the data-parallel merge and the row updates of a list all run there, overlapping the towers on the main stream
    cudaStream_t sstream[2] = {nullptr, nullptr};
    cudaStream_t stream_up = nullptr;        // host->device refills of batch slots (wd_batch_prefetch_slot), overlapping the running step
    cudaEvent_t ev_ids = nullptr, ev_head = nullptr, ev_dx0 = nullptr, ev_bwd_done = nullptr, ev_wide_fwd = nullptr, ev_wgrad_rest = nullptr;
    bool sort_smem_opt_in = false;               // rs_scatter_kernel<RS_BIG_TILE, true> was granted its dynamic shared memory on this device
    bool crelu = false;                          // dnn_activation_function crelu: relu on mirrored kernels (mlp.cu crelu_fold / crelu_mirror)
    bool record_wgrad_rest = false;           // mlp_backward: record ev_wgrad_rest before the first layer's weight gradient
    int dense_split_tensor = -1, dense_part = 0;   // dense_apply: see mlp.cu (single-GPU step, split dense optimizer)
    cudaEvent_t ev_grouped[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
    bool side_pending[2] = {false, false};   // the list's grouping of this step was issued on its side stream
    bool side_active[2] = {false, false};    // the list's sums live on its side stream (merge / apply follow there)
    bool record_dx0 = false, dx0_recorded = false;
    wd::StepGraph<wd::MergeKey> merge_graph[2];   // data-parallel merge of list w (fixed-size exchange: wd_sparse_set_sorted)
    // ---- dense exchange of small tables (WdPlanDesc::dense_exchange_max_rows)
    int64_t dense_exchange_max_rows = 0;
    int64_t small_base[2] = {0, 0};          // first global row of the small embedding tables / small wide columns
    int64_t gs_count = 0, gs_emb_floats = 0; // floats of the small-table gradient block behind d_G[dense_count]; its embedding part
    int64_t gs_touch_off[2] = {0, 0};        // offsets (floats, inside the block) of the per-row "touched" counts: small embedding rows / small wide rows
    int n_small_tab = 0;                     // replicated tables that are small (the last ones of rtabs)
    // Adam: bitmaps of the replicated record sets (0: embedding rows, emb_total_rows bits; 1: wide rows, wide_rows bits), bit r set
    // when row r was updated this step, cleared by the set's untouched pass (sparse_dev.cuh); null unless that optimizer is Adam
    uint32_t* d_adam_touched[2] = {nullptr, nullptr};
    wd::ShardState shard;                    // row-sharded tables (world == 1: unused)
    wd::DevPlan dplan{};
    // what the model owns on the device, released by wd_model_destroy: streams and events (new_stream / new_event), and
    // everything cudaMalloc'ed (dev_alloc; bytes_allocated is their sum)
    std::vector<cudaStream_t> streams;
    std::vector<cudaEvent_t> events;
    std::vector<wd::DevAlloc> allocs;
    int64_t bytes_allocated = 0;
    // ---- host-placed embedding tables (host_tables.cu)
    std::vector<void*> host_allocs;          // cudaHostAlloc'ed table records (freed in destroy)
    int64_t host_bytes = 0;
    int n_host_tab = 0;
    std::vector<int> rtab_order;             // replicated table ids in global row order (the tables of rtabs)
    float* d_stage = nullptr;                // [max_nnz][stage_stride] records of the step's unique host rows, row u at u * stage_stride
    int stage_stride = 0;                    // largest stride of the host tables
    uint32_t* d_g_emb = nullptr;             // [max_nnz] ids the gather reads: e_emb, host-table entries replaced by their unique index u
    // HBM cache of host records (wd_host_cache_enable): d_stage is then [hcache.slots slots | max_nnz overflow rows]
    wd::HostCache hcache;
    // Adam on deferred host tables (host_tables.cu): tables with deferred() (host shards included), lr_t[j] of steps j = 1 ..
    // lr_t_last (later steps: lr), counters [rows caught up, steps replayed, steps skipped, longest gap]
    int n_defer_tab = 0;
    float* d_lr_t = nullptr;
    int64_t lr_t_last = 0;
    unsigned long long* d_defer_stats = nullptr;
    bool stepped = false;                    // a forward or train step was issued (step graphs may exist)

    // numeric deep columns (device arrays)
    int32_t *d_num_field = nullptr, *d_num_norm_kind = nullptr, *d_num_x0_off = nullptr;
    float *d_num_a = nullptr, *d_num_b = nullptr;

    // ---- the batch of the current slot (slots, cur_slot)
    int64_t keys_cap = 0;
    wd::DevBatch dbatch{};

    // ---- column ids (CSR over (row, column)) and per-entry arrays
    int32_t* d_col_offs = nullptr;           // [max_batch * n_columns + 1]
    uint32_t* d_e_wide = nullptr;            // [max_nnz] global wide row or kInvalidRow
    uint32_t* d_e_emb = nullptr;             // [max_nnz] global embedding row or kInvalidRow
    int32_t* d_e_bc = nullptr;               // [max_nnz] row * n_columns + column
    int32_t* d_e_id = nullptr;               // [max_nnz] column-local id (debug / parity)
    int32_t* d_nnz = nullptr;                // device scalar: entries this step
    int32_t* d_flags = nullptr;              // device error flags [4]
    wd::SortScratch scratch[4];              // scan / sort scratch, one set per stream (0 main, 1 + list for the side streams, 3 aux)
    int scratch_sel = 0;
    int64_t sort_hist_cap = 0;

    // ---- wide part: record {w, n, z, 0} per row
    float4* d_wide = nullptr;
    float* d_wide_logit = nullptr;           // [max_batch]

    // ---- deep part
    std::vector<wd::EmbTable> tables;
    int64_t emb_total_rows = 0;
    int emb_max_dim = 0;
    int n_dims = 0;
    int dims[wd::kMaxDims];                  // distinct widths
    int dim_ntables[wd::kMaxDims];
    // the record sets of the embedding tables and the gather view (table at the top of host_tables.cu)
    wd::RecordSet tabs;                      // every table in plan order
    wd::RecordSet rtabs;                     // the replicated tables in global row order (rtab_order)
    wd::TabDesc* d_dim_desc[wd::kMaxDims] = {};   // [dim_ntables] gather view of the replicated tables of width dims[i]
    float *d_X0 = nullptr, *d_dX0 = nullptr;
    float* d_X0T = nullptr;                  // fp32 family: transposed X0 [d0_phys, ldt]
    __nv_bfloat16* d_X0s[2] = {nullptr, nullptr};   // bf16 family: hi / lo copies of X0
    int ldt = 0;                             // leading dim of transposed activations (= max_batch_pad)
    std::vector<wd::Tower> towers;

    // ---- dense parameter arena
    std::vector<wd::DenseTensor> dense;
    int64_t dense_count = 0, gpart_count = 0, wt_count = 0;
    float *d_P = nullptr, *d_S1 = nullptr, *d_S2 = nullptr, *d_G = nullptr, *d_gpart = nullptr;
    // GEMM operand copies of the hidden layers' kernels W [K, N], wt_count elements each (DenseTensor::wt_off), rewritten after
    // every optimizer step; only the operand family's exist
    float* d_Wt = nullptr;                                      // fp32 family: Wt [N, K]
    float *d_W_hi = nullptr, *d_W_lo = nullptr;                 // fp32 family: tf32 hi / lo splits of W (3xTF32)
    float *d_Wt_hi = nullptr, *d_Wt_lo = nullptr;               // fp32 family: tf32 hi / lo splits of Wt (3xTF32)
    __nv_bfloat16 *d_Wq_hi = nullptr, *d_Wq_lo = nullptr;       // bf16 family: bf16 hi / lo splits of W
    wd::DenseTensor* d_dense_desc = nullptr;
    int row_tiles = 0;                       // max_batch_pad / 128
    int wgrad_splits = 4;

    // ---- loss / logits
    float* d_logits = nullptr;               // [max_batch]
    float* d_dlogit = nullptr;               // [max_batch]
    float* d_loss_part = nullptr;            // per-block partials
    float* d_loss = nullptr;                 // scalar
    unsigned long long* d_step_trace = nullptr;   // WD_STEP_TRACE=1: globaltimer stamps of the last step (wd_debug_step_trace)
    int32_t* d_head_counter = nullptr;       // blocks of the head kernel that have finished (last one sums the loss)
    float* d_bpow = nullptr;                 // Adam: {linear beta1^t, linear beta2^t, dnn beta1^t, dnn beta2^t}, multiplied in fp32 after every step (AdamOptimizer._finish)
    uint32_t* d_adam_step = nullptr;         // Adam: steps completed (advances with d_bpow; the "now" of deferred tables' stamps)
    float* h_loss_pinned = nullptr;

    wd::RowList lists[wd::kLists];           // sparse backward scratch: the sparse row lists

    // ---- eval metrics
    double* d_metrics = nullptr;             // accumulators
    int64_t eval_batches = 0;

    int64_t launches = 0;
    int64_t graph_captures = 0, graph_replays = 0;   // step graphs captured / replayed (wd_graph_stats)
    float dropout_rate = 0.f;               // dnn_dropout: tf.layers.dropout after every hidden layer's activation, train steps only
    unsigned long long dropout_seed = 0;
    unsigned int* d_step = nullptr;         // device: train steps completed (dropout counter; advances at the end of every step)
    bool fuse_dense = false;                // whole local step (train_eager): dense gradient reduction fused into the optimizer kernel
    int64_t gemm_fallbacks = 0;            // tensor-core engine GEMMs that ran on the FFMA kernel instead (tests assert 0)
    int cur_slot = 0;
    bool graphs_enabled = true;              // WD_NO_GRAPH=1 disables step graphs
    int cur_layer = 0;                       // layer being launched (names the profiling marks)
    wd::PhaseTimer timer;
    std::vector<wd::BatchSlot> slots;        // batch slots, allocated up to the highest one used (slot 0 by wd_model_create)
    wd::TsvDev* tsv = nullptr;               // device TSV parser (wd_tsv_parse_slot), created on first use
    int64_t tsv_device_batches = 0, tsv_host_batches = 0;   // batches wd_tsv_parse_slot parsed on the device / on the host
    bool initialized = false;
    bool grads_pending = false;
    // layer summaries (summary.cu): the next train step takes the statistics (wd_summary_arm); they await wd_summary_read
    wd::SummaryState* summ = nullptr;
    bool summary_armed = false, summary_ready = false;

    // ---- host-only plan bookkeeping (tensor IO, initialisation, summaries)
    std::vector<uint8_t> x0_real;            // [d0_phys] 1 where a physical deep-input column is a real feature
    int d0_logical = 0;
    std::vector<std::vector<int>> dense_index;   // [tower-layer id][sub] -> index into dense, -1
    std::vector<int> did_tower, did_layer;
};

namespace wd {
// ---- kernels / stages implemented in the .cu files (all enqueue on m->stream)
int ids_prepare(WdModel* m);                                     // ids.cu
int sparse_forward(WdModel* m);                                  // sparse.cu: wide logit + embedding pooling + numerics
int sparse_forward_wide(WdModel* m);                             //   the wide half alone
int sparse_forward_emb(WdModel* m);                              //   the deep half alone
int sparse_reduce_emb(WdModel* m);                               // sparse.cu: per-row gradient sums (needs dX0)
int sparse_reduce_wide(WdModel* m);                              // sparse.cu: per-row gradient sums (needs dlogit only)
int sparse_apply_which(WdModel* m, int which);                   // sparse.cu: optimizer on the touched rows of list 0 (embedding rows) / 1 (wide rows)
int sparse_group_which(WdModel* m, int which);                   // sparse.cu: sort (row, occurrence) pairs of one list, unique rows, chunks
// sparse.cu: list L over a space of `rows` rows, ugrad / cpart rows of `width` floats; sort_only: keys / values alone (routing)
int list_alloc(WdModel* m, int L, int64_t rows, int width, bool sort_only);
int merge_sparse_sorted(WdModel* m, int which, const void* rows, const void* grads, int n_lists, int64_t list_len);   // sparse.cu
int small_scatter(WdModel* m, int which);                        // sparse.cu: small-table rows of list `which` -> dense block
int small_apply(WdModel* m);                                     // sparse.cu: optimizer over the dense block (after its all-reduce)
int adam_untouched_replicated(WdModel* m);                       // sparse.cu: Adam rows of the replicated tables no update touched this step
int mlp_forward(WdModel* m, bool want_transposes);               // mlp.cu: towers -> logits, loss
int mlp_backward(WdModel* m);                                    // mlp.cu: grads of dense params, dX0
int dense_reduce_grads(WdModel* m);                              // mlp.cu
int dense_apply(WdModel* m);                                     // mlp.cu
int loss_forward(WdModel* m, bool need_grad);                    // mlp.cu: logits = wide + deep, loss, dlogit
int model_init_params(WdModel* m, uint64_t seed);                // init.cu
int step_tick(WdModel* m);                                       // misc.cu: train-step counter on the device (dropout)
// first row of this rank's batch in the global batch the dropout mask is drawn over (DropArgs::row0): rank * max_batch
inline unsigned int drop_row0(const WdModel* m) { return m->shard.world > 1 ? (unsigned int)m->shard.rank * (unsigned int)m->max_batch : 0u; }
int adam_tick(WdModel* m);                                       // misc.cu: beta powers advance (after every optimizer of the step)
int shard_build(WdModel* m, const WdPlanDesc* d);                // shard.cu: sharded spaces, their lists and the exchange segment
int place_tables(WdModel* m, int64_t hbm_reserve);               // host_tables.cu: allocate the tables (HBM / host) and staging buffers
int build_record_sets(WdModel* m);                               // host_tables.cu: upload the record sets and the gather view
int host_tables_stage_in(WdModel* m, bool train);                // host_tables.cu: cache lookup, host rows -> staging buffer, gather ids
int host_tables_write_back(WdModel* m);                          // host_tables.cu: overflow rows of the staging buffer -> host rows
int host_cache_sync(WdModel* m, bool flush, bool invalidate);    // host_tables.cu: dirty cached records -> host; optionally empty the cache
// host_tables.cu: dirty cached records of host table tb's local rows row0 .. row0 + rows - 1 -> host; optionally empty their slots
int host_cache_sync_rows(WdModel* m, const EmbTable& tb, int64_t row0, int64_t rows, bool invalidate);
// host_tables.cu: host records row0 .. row0 + rows - 1 of deferred table tb caught up to the current Adam step in place (stamp_only:
// just stamped)
int deferred_adam_settle(WdModel* m, const EmbTable& tb, int64_t row0, int64_t rows, bool stamp_only);
// host_tables.cu, over any record set `rr` whose staged tables (found by row base) keep the records of the unique rows of list L
// (lists[L].urow[0 .. *lists[L].nuniq)) in rr.stage_base at stride S, behind cache `c` (c.slots = 0: none, staging row u):
//   stage_in_rows    cache keys -> sort -> assign (train: the used slots turn dirty), then dirty victims home and the records
//                    to load -> their staging rows
//   write_back_rows  overflow staging rows -> host records (every staged row without a cache)
// `marks` names the phases (wd_last_timings): sort, assign, transfer in (null: the caller marks), write-back.
struct CacheMarks { const char *sort, *assign, *in, *out; };
int stage_in_rows(WdModel* m, HostCache& c, int L, const RowRecords& rr, int S, bool train, const CacheMarks& marks);
int write_back_rows(WdModel* m, const HostCache& c, int L, const RowRecords& rr, int S, const CacheMarks& marks);
int64_t hbm_reserve_bytes(const WdModel* m);                     // api.cu: HBM the model keeps free for its later allocations
// tsv.cu: device parse of n lines into the batch buffers on stream st, waiting for it; *status != 0: the buffers do not hold the
// batch (parse it on the host)
int tsv_parse_device(WdModel* m, const WdTsvSpec* sp, const char* text, int64_t text_len, const int64_t* starts, int n, int32_t* off,
                     uint64_t* keys, float* dense, float* label, float* weight, cudaStream_t st, int* status);
int tsv_parse_host(const WdTsvSpec* sp, const char* text, const int64_t* starts, int n, WdBatch* out);   // tsv.cu
void tsv_dev_destroy(WdModel* m);                                // tsv.cu
int metrics_accumulate(WdModel* m, int rows);                    // misc.cu: metrics of the first `rows` logits of the batch
int metrics_finish(WdModel* m, const double* acc, double* out10); // misc.cu: the ten metrics of an accumulator (synchronises)
int summary_prepare(WdModel* m, const std::vector<uint8_t>& x0_real);   // summary.cu: segments and buffers (first use)
int summary_launch(WdModel* m);                                  // summary.cu: statistics of the armed train step

// sorts (*keys, *vals) of length *d_n by the low `bits` bits of the key, with (*keys2, *vals2) as ping-pong buffers; the
// pointers are swapped so that the sorted pairs end in (*keys, *vals)
int radix_sort_pairs(WdModel* m, uint32_t** keys, uint32_t** vals, uint32_t** keys2, uint32_t** vals2, int bits, const int32_t* d_n);   // sort.cu
int exclusive_scan_i32(WdModel* m, int32_t* data, int64_t n, int32_t* total_out);   // sort.cu (in place, n known on host)
int seg_heads(WdModel* m, const int32_t* d_n, const uint32_t* keys, uint32_t invalid, int32_t* pos, int64_t cap, int32_t* ustart, uint32_t* urow,
              int32_t* d_nuniq);                                                    // sort.cu: unique rows of sorted keys (2 launches)
int chunk_offsets(WdModel* m, const int32_t* d_nuniq, const int32_t* ustart, uint32_t* urow, int32_t* choff, int64_t cap, int chunk,
                  int32_t* d_nchunks);                                              // sort.cu: hot-row chunk layout (2 launches)

template <typename T>
int dev_alloc(WdModel* m, T** p, int64_t count, bool zero = true) {
    if (count <= 0) count = 1;
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, (size_t)count * sizeof(T));
    if (e != cudaSuccess) {
        set_error("cudaMalloc of %lld bytes failed: %s", (long long)(count * sizeof(T)), cudaGetErrorString(e));
        return WD_ENOMEM;
    }
    if (zero) {
        e = cudaMemsetAsync(q, 0, (size_t)count * sizeof(T), m->stream);
        if (e != cudaSuccess) { set_error("cudaMemset failed: %s", cudaGetErrorString(e)); return WD_ECUDA; }
    }
    m->allocs.push_back({q, count * (int64_t)sizeof(T)});
    m->bytes_allocated += count * (int64_t)sizeof(T);
    *p = (T*)q;
    return WD_OK;
}
// frees an allocation of dev_alloc before the model dies, and takes its bytes off bytes_allocated
inline int dev_free(WdModel* m, void* p) {
    for (size_t i = 0; i < m->allocs.size(); ++i) {
        if (m->allocs[i].p != p) continue;
        WD_CUDA(cudaFree(p));
        m->bytes_allocated -= m->allocs[i].bytes;
        m->allocs.erase(m->allocs.begin() + i);
        break;
    }
    return WD_OK;
}
// a stream / an event the model owns (wd_model_destroy synchronises and destroys it)
inline cudaError_t new_stream(WdModel* m, cudaStream_t* s) {
    const cudaError_t e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
    if (e == cudaSuccess) m->streams.push_back(*s);
    return e;
}
inline cudaError_t new_event(WdModel* m, cudaEvent_t* ev, unsigned flags) {
    const cudaError_t e = cudaEventCreateWithFlags(ev, flags);
    if (e == cudaSuccess) m->events.push_back(*ev);
    return e;
}
// copies src[0 .. n) to the device array *dst, allocated here while *dst is null; an existing array is overwritten in place (a
// second upload of the same descriptor allocates nothing)
template <typename T> struct same_type { using type = T; };   // (keeps `src` out of the deduction of T)
template <typename T>
int upload(WdModel* m, T** dst, const typename same_type<T>::type* src, int64_t n) {
    if (!*dst) {
        int rc = dev_alloc(m, dst, n, true);
        if (rc) return rc;
    }
    if (n > 0) WD_CUDA(cudaMemcpyAsync((void*)*dst, src, n * sizeof(T), cudaMemcpyHostToDevice, m->stream));
    return WD_OK;
}
template <typename T, typename A>
int upload(WdModel* m, T** dst, const std::vector<A>& h) { return upload(m, dst, h.data(), (int64_t)h.size()); }

// record a named mark on the model stream (no-op unless profiling is on)
inline void mark(WdModel* m, const char* name) {
    PhaseTimer& t = m->timer;
    if (!t.enabled || t.n >= PhaseTimer::kMax) return;
    t.name[t.n] = name;
    cudaEventRecord(t.ev[t.n], m->stream);
    t.n++;
}

// run `fn` with the model's launches going to `stream` and its scan / sort scratch set `scratch_sel` (WdModel::scratch)
template <typename F>
int on_stream(WdModel* m, cudaStream_t stream, int scratch_sel, F fn) {
    cudaStream_t main_stream = m->stream;
    m->stream = stream; m->scratch_sel = scratch_sel;
    int rc = fn();
    m->stream = main_stream; m->scratch_sel = 0;
    return rc;
}
// on the side stream of sparse list `which`
template <typename F>
int on_side(WdModel* m, int which, F fn) { return on_stream(m, m->sstream[which], 1 + which, fn); }
// on the auxiliary stream of a row-sharded step (ShardState::aux)
template <typename F>
int on_aux(WdModel* m, F fn) { return on_stream(m, m->shard.aux, 3, fn); }

inline int grid_for(int64_t n, int block, int cap = kNumSms * 16) {
    int64_t g = (n + block - 1) / block;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}
}  // namespace wd
