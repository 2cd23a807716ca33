/*
 * wd_b200.h — C-ABI of libwd_b200.so: the H100-native (sm_90a) Wide&Deep CTR train/eval step.
 *
 * The reference (Lapis-Hong/wide_deep) has no native plugin/FFI boundary: its seam is the Python-level
 * estimator object built by build_custom_estimator (reference python/lib/build_estimator.py:264-294) whose
 * .train/.evaluate/.predict run TensorFlow's model_fn (reference python/lib/joint.py:81-269).  This header
 * is the boundary a maintainer binds instead of TensorFlow; each entry point cites what it replaces.
 *
 * Conventions: plain C, plain pointers and sizes; every function returns 0 on success or a negative
 * WD_E* code (never throws; wd_last_error() holds the message); the caller owns host buffers, the
 * library owns all device memory; one host thread drives one WdModel; handles are not thread-safe.
 * All device work is enqueued on the model's stream; functions that return host data synchronise it.
 * There is NO CPU fallback: every compute entry point fails with WD_ENODEVICE without a CUDA device.
 */
#ifndef WD_B200_H_
#define WD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WD_API_VERSION 3

enum { WD_OK = 0, WD_EINVAL = -1, WD_ENODEVICE = -2, WD_ECUDA = -3, WD_ENOMEM = -4, WD_EUNSUPPORTED = -5, WD_ESTATE = -6 };

/* categorical column kinds (reference python/lib/build_estimator.py:83-158) */
enum { WD_COL_HASH = 0, WD_COL_VOCAB = 1, WD_COL_IDENTITY = 2, WD_COL_BUCKET = 3, WD_COL_CROSS = 4 };
/* continuous normalisers (reference python/lib/build_estimator.py:61-68) */
enum { WD_NORM_NONE = 0, WD_NORM_MINMAX = 1, WD_NORM_STANDARD = 2, WD_NORM_LOG = 3 };
/* cross key sources: raw string field (dense input incl. padding) or a categorical column (sparse input) */
enum { WD_KEY_FIELD = 0, WD_KEY_COLUMN = 1 };
/* optimizers (reference python/lib/utils/model_util.py:62-105) */
enum { WD_OPT_SGD = 0, WD_OPT_ADAGRAD = 1, WD_OPT_FTRL = 2,
       WD_OPT_ADAM = 3     /* tf.train.AdamOptimizer: slots m, v; sparse gradients decay m, v over the WHOLE table (TF semantics) */,
       WD_OPT_RMSPROP = 4  /* tf.train.RMSPropOptimizer (not centered): slots rms (init 1), momentum; touched rows only */ };
/* activations (reference python/lib/utils/model_util.py:28-59) */
enum { WD_ACT_RELU = 0, WD_ACT_RELU6, WD_ACT_SIGMOID, WD_ACT_TANH, WD_ACT_LEAKY_RELU, WD_ACT_ELU, WD_ACT_SELU,
       WD_ACT_SOFTPLUS, WD_ACT_SOFTSIGN,
       WD_ACT_CRELU   /* tf.nn.crelu = concat(relu(z), relu(-z)): a hidden layer of u units feeds 2u features to whatever follows it
                       * (dropout, batch norm, the next layers).  The parameters keep the reference's shapes — kernel [in, u], bias [u]
                       * (wd_tensor_io / wd_tensor_size), batch-norm gamma / beta [2u]. */ };
/* dnn_connected_mode (reference python/lib/dnn.py:92-193) */
enum { WD_MODE_SIMPLE = 0, WD_MODE_FIRST_DENSE, WD_MODE_LAST_DENSE, WD_MODE_DENSE, WD_MODE_RESNET };
/* GEMM engine for the MLP */
enum { WD_GEMM_AUTO = 0, WD_GEMM_FFMA = 1, WD_GEMM_TC3X = 2 /* wgmma tf32, 3-pass split */,
       WD_GEMM_TC1X = 3 /* wgmma tf32 single pass: fast, NOT within the 1e-4 parity bar */,
       WD_GEMM_BF16X3 = 4 /* wgmma on bf16 hi/lo copies written by the producing kernels, 3 passes */ };
/* where an embedding table's records live (WdPlanDesc::table_placement) */
enum { WD_PLACE_HBM = 0, WD_PLACE_HOST = 1 /* mapped, page-locked host memory */,
       WD_PLACE_AUTO = 2 /* HBM if it fits, else host memory (resolved once by wd_model_create) */,
       WD_PLACE_DEFER_ADAM = 4 /* flag OR'ed into WD_PLACE_HOST / WD_PLACE_AUTO: Adam's untouched rows catch up when next read */ };

typedef struct WdOptimizer {
    int32_t kind;        /* WD_OPT_* */
    float lr, l1, l2, lr_power, init_acc;
    float beta1, beta2, epsilon;   /* Adam (epsilon also RMSProp) */
    float rho, momentum;           /* RMSProp decay / momentum */
} WdOptimizer;

/* Immutable description of the model, produced by wide_deep_b200.plan.compile_plan() from conf/*.yaml.
 * Replaces the feature-column lists of _build_model_columns (reference build_estimator.py:49-169). */
typedef struct WdPlanDesc {
    int32_t api_version;
    int32_t model_type;             /* bit0: wide part, bit1: deep part */
    int32_t n_cat_fields;           /* key fields of a batch (string features as uint64 fingerprints, identity as ints) */
    int32_t n_dense_fields;         /* continuous fields */
    const uint8_t *cat_field_is_string; /* [n_cat_fields] 1: fingerprints (Fingerprint64("") marks ''), 0: int ids */

    int32_t n_columns;              /* categorical columns, in evaluation order */
    const int32_t *col_kind;        /* WD_COL_* */
    const int32_t *col_field;       /* cat field (HASH/VOCAB/IDENTITY) | dense field (BUCKET) | -1 */
    const int64_t *col_buckets;     /* id range of the column */
    const int32_t *col_aux_off;     /* VOCAB: into vocab_fp; BUCKET: into boundaries; CROSS: into cross_key_* */
    const int32_t *col_aux_n;
    const int32_t *col_norm_kind;   /* BUCKET: normaliser applied before bucketising (quirk Q3) */
    const float *col_norm_a, *col_norm_b;
    const int64_t *col_wide_base;   /* first row in the wide table, -1: not a wide column */
    const int32_t *col_emb_table;   /* embedding table fed by this column, -1: none */
    const int32_t *col_ind_off;     /* indicator (multi-hot count) offset in the deep input, -1: none */
    const uint64_t *vocab_fp;       int32_t n_vocab_fp;
    const float *boundaries;        int32_t n_boundaries;
    const int32_t *cross_key_type;  /* WD_KEY_*; keys of each cross are stored in OP order */
    const int32_t *cross_key_idx;   int32_t n_cross_keys;

    int32_t n_tables;               /* embedding tables (combiner = mean) */
    const int64_t *table_rows;
    const int32_t *table_dim;       /* physical width: logical width padded to a multiple of 4 (pad columns stay 0) */
    const int32_t *table_dim_logical; /* embedding_column dimension (reference build_estimator.py:57-59) */
    const int32_t *table_x0_off;    /* physical column offset in the deep input, multiple of 4 */
    int32_t n_numeric;              /* numeric deep columns */
    const int32_t *num_field, *num_norm_kind, *num_x0_off;
    const float *num_norm_a, *num_norm_b;
    int32_t d0_phys;                /* physical width of the deep input (multiple of 32; padding columns stay 0) */
    int64_t wide_rows;              /* total rows of the wide weight table */

    int32_t n_towers;               /* at most 8 (WD_EUNSUPPORTED otherwise) */
    const int32_t *tower_nlayers;  /* hidden layers per tower */
    const int32_t *tower_mode;      /* WD_MODE_* */
    const int32_t *hidden_units;    /* concatenated over towers */
    int32_t activation;             /* WD_ACT_* */
    int32_t batch_norm;             /* inference-mode affine gamma/sqrt(1+1e-3), beta (quirk Q4) */
    WdOptimizer lin_opt, dnn_opt;
    int32_t max_batch;              /* rows per step this handle must accept */
    int64_t max_nnz;                /* upper bound on categorical-column ids per step (0: derive) */
    int64_t max_keys;               /* upper bound on batch keys per step (0: derive) */
    int32_t gemm_engine;            /* WD_GEMM_* */
    /* Data-parallel exchange format.  Embedding tables / wide columns with at most this many rows ("small") are laid out after
     * the large ones in the global row space and their per-step gradient leaves as a DENSE block appended to the dense gradient
     * arena (wd_dense_grad_ptr / wd_dense_grad_count: one all-reduce covers it), not as (row, gradient) list entries; only the
     * large tables' touched rows go through wd_sparse_grads / wd_sparse_set.  0 = every table uses the list (default).
     * wide_small_base = first wide row of the small wide columns (= wide_rows when there is none); the plan orders the wide
     * columns large-first. */
    int64_t dense_exchange_max_rows;
    int64_t wide_small_base;
    /* Row-sharded tables (the reference partitions large variables over its parameter servers with
     * tf.min_max_variable_partitioner, reference python/lib/joint.py:141-143).  shard_world = G > 1: this handle is rank
     * shard_rank of G; every embedding table with table_sharded[t] = 1 and every wide column with col_wide_sharded[c] = 1 keeps
     * only the rows r with r mod G == shard_rank (local row r / G).  The plan marks exactly the tables larger than
     * dense_exchange_max_rows, so a sharded run has no (row, gradient) lists: small tables exchange the dense block, large ones
     * are reached through the peer-memory exchange of wd_shard_* below.  shard_capacity: upper bound on the ids one rank routes
     * per step and table space (0: max_nnz); shard_slack x that bound is what one rank can receive as an owner. */
    int32_t shard_world, shard_rank;
    const uint8_t *table_sharded;       /* [n_tables] */
    const uint8_t *col_wide_sharded;    /* [n_columns] */
    int64_t shard_capacity;
    float shard_slack;
    /* dnn_dropout (reference python/lib/dnn.py:111-112: tf.layers.dropout(rate, training=True) after every hidden layer's
     * activation, TRAIN mode only).  The keep mask is a counter-based function of (dropout_seed, step, layer, row, column) — see
     * csrc/gemm.cuh — so runs are reproducible and the oracle can apply the same mask; 0 = no dropout. */
    float dropout_rate;
    uint64_t dropout_seed;
    /* Embedding-table placement, [n_tables] WD_PLACE_* (NULL: every table in HBM).  The reference keeps its tables in host RAM:
     * it trains on the CPU or spreads them over parameter servers (reference python/lib/build_estimator.py:211-214,
     * python/lib/joint.py:141-143).  A host-placed table keeps its [w | slots] records in mapped, page-locked host memory; every
     * step copies the records of the rows it touches into an HBM staging buffer, runs the same kernels on them and writes them
     * back, so results are bit-identical to the table in HBM.  WD_PLACE_AUTO: wd_model_create allocates the auto tables largest
     * first and moves to host memory only a table whose HBM allocation fails (with room kept for the buffers allocated after
     * creation).  With shard_world > 1 only the row-sharded tables (table_sharded[t] = 1) may be placed on the host: each rank's
     * shard lives in its own host memory and its owner stages the rows it owns (results bit-identical to the shards in HBM); the
     * auto placement then also keeps room for the sharded exchange buffers.  Host placement is refused (WD_EUNSUPPORTED) for a
     * replicated table of a sharded model, with dense_exchange_max_rows > 0 and shard_world <= 1, or with Adam as the dnn
     * optimizer; auto tables stay in HBM in those cases.
     * Adam: sparse Adam moves every row of a table every step (decay of m and v, then a step of w), which would stream a host
     * table over PCIe twice per step.  WD_PLACE_DEFER_ADAM OR'ed into a WD_PLACE_HOST / WD_PLACE_AUTO entry lifts the Adam
     * refusal for that table: its records become [w | m | v | stamp] (the stamp: the last Adam step the record reflects, in a
     * trailing float4) and a row that no gradient touched is brought up to date when it is next staged, by replaying the
     * steps it missed in order with the same fp32 operations, so results stay bit-identical to the table in HBM.  The replay
     * costs up to one step per missed step and row, until the row's values stop changing.  Ignored for other optimizers. */
    const uint8_t *table_placement;
} WdPlanDesc;

/* One batch in HOST memory (pinned for async copies).  Replaces the feature dict produced by input_fn
 * (reference python/lib/dataset.py:293-310): CSR over (row, cat field), row-major. */
typedef struct WdBatch {
    int32_t batch_size;
    const int32_t *cat_offsets;     /* [batch_size*n_cat_fields+1], NULL: exactly one key per (row, field) */
    const uint64_t *cat_keys;       /* [nnz] fingerprints / ints */
    int64_t nnz;
    const float *dense;             /* [batch_size*n_dense_fields] */
    const float *label;             /* [batch_size] 0/1, NULL for predict */
    const float *weight;            /* [batch_size] example weights, NULL = 1 (weight_column, dataset.py:159-163) */
} WdBatch;

typedef struct WdModel WdModel;

/* tensor selectors for wd_tensor_io */
enum { WD_T_WIDE_COL = 0, WD_T_EMB_TABLE = 1, WD_T_DENSE = 2, WD_T_WIDE_BIAS = 3 };
/* dense tensor ids: tower t, layer l (l == nlayers: logits): see wd_dense_tensor_id */
enum { WD_D_KERNEL = 0, WD_D_BIAS = 1, WD_D_GAMMA = 2, WD_D_BETA = 3 };

const char *wd_last_error(void);
int wd_version(void);
int wd_device_count(void);

/* Model lifetime.  Replaces WideAndDeepClassifier.__init__ (reference python/lib/joint.py:326-432). */
int wd_model_create(const WdPlanDesc *plan, int device, WdModel **out);
int wd_model_destroy(WdModel *m);
/* Device-side initialisation with the TF initialisers (truncated normal / glorot uniform / zeros). */
int wd_model_init(WdModel *m, uint64_t seed);
/* Number of optimizer steps already taken (checkpoint resume): restores Adam's beta1^t / beta2^t (the non-slot variables of
 * tf.train.AdamOptimizer); a no-op for the other optimizers.  Rows of WD_PLACE_DEFER_ADAM tables keep their step stamps: the
 * call moves "now", so a row stamped s then owes steps s+1 .. steps (none when s >= steps).  Writing a table's tensor
 * (wd_tensor_io) stamps every row with the current step. */
int wd_set_opt_step(WdModel *m, int64_t steps);
/* Copy a parameter or optimizer slot to/from host.  slot 0 = value, 1.. = optimizer accumulators
 * (Adagrad: acc; FTRL: n, z).  Logical (unpadded) shapes; kernels are [in, out] like tf.layers.dense. */
int wd_tensor_io(WdModel *m, int kind, int index, int sub, int slot, void *host, int64_t count, int to_device);
int64_t wd_tensor_size(WdModel *m, int kind, int index, int sub);
/* Copy rows row0 .. row0 + nrows - 1 of an embedding table (WD_T_EMB_TABLE: nrows x dimension floats) or a wide column
 * (WD_T_WIDE_COL: nrows floats) to/from host, slot as in wd_tensor_io; rows of a row-sharded tensor are this rank's local rows.
 * WD_EINVAL for any other kind and for a range outside the tensor.  wd_tensor_io's guarantees hold for the range: dirty cached
 * records of its rows go home before either direction, a write leaves no cached copy of them, and a WD_PLACE_DEFER_ADAM table's
 * rows are caught up before a read and stamped with the current step after a write.  The cost is that of the range (plus one pass
 * over an HBM cache's slot tags), not of the table: checkpoints move a table in bounded chunks through this call. */
int wd_tensor_io_rows(WdModel *m, int kind, int index, int sub, int slot, int64_t row0, int64_t nrows, void *host, int to_device);
/* Memory the model holds: device_bytes = HBM it allocated, host_bytes = page-locked host memory of its host-placed embedding
 * tables (WdPlanDesc::table_placement; a rank of a row-sharded model counts its own shards).  Either pointer may be NULL.  (The reference's parameters sit in host RAM on the CPU
 * or on the parameter servers, reference python/lib/build_estimator.py:211-214.) */
int wd_memory_usage(WdModel *m, int64_t *device_bytes, int64_t *host_bytes);
/* HBM cache of host-placed table records: an 8-way set-associative, write-back cache of whole [w | slots] records, with LRU
 * replacement inside a set.  Rows a step touches that are cached are neither fetched nor written home; results stay
 * bit-identical to the uncached model.  Call after wd_model_create and before the first step or forward (WD_ESTATE after).
 * `bytes` is the HBM budget of the records: it is rounded down to 8 x 2^k slots of the widest host record; the slot metadata
 * (9 bytes per slot) comes on top.  A no-op (capacity 0) when no table is on the host.  WD_ENOMEM when the cache would leave less
 * free HBM than the model keeps in reserve for its later allocations (batch slots, step graphs).  The cache is opt-in:
 * wd_step_backward(_slot) is refused (WD_EUNSUPPORTED) on a model with a cache.  This cache sits in front of the host tables of a
 * single-GPU model: on a row-sharded model (shard_world > 1) with host-placed shards it returns WD_EUNSUPPORTED (the owner's cache
 * of its shards is wd_shard_cache_enable). */
int wd_host_cache_enable(WdModel *m, int64_t bytes);
/* The same cache on one rank of a row-sharded model (shard_world > 1): it holds the most recently used records of the rank's own
 * host-placed shards (the rows it owns, in its shard row space) in its HBM, in front of the owner's stage-in and write-back.  Call
 * per rank, after wd_model_create and before the first step or forward.  Results stay bit-identical to the uncached model and to
 * the model with every shard in HBM, on both drivers (wd_shard_train_step_slot and wd_shard_phase).  Rules as
 * wd_host_cache_enable: WD_ESTATE after the first step or forward or when a cache exists, WD_EINVAL for a negative budget or slots
 * beyond 31-bit staging rows, WD_ENOMEM below the HBM reserve, a no-op (capacity 0) when this rank has no host-placed shard or the
 * budget is below one set.  WD_EUNSUPPORTED when shard_world == 1 (use wd_host_cache_enable).  A model has at most one cache. */
int wd_shard_cache_enable(WdModel *m, int64_t bytes);
/* Cumulative counters of the model's cache (either kind): out[0] capacity in slots, [1] hits, [2] misses loaded into a slot,
 * [3] overflow rows (staged without a slot: more misses in a set than it has ways), [4] dirty evictions written home.  All 0
 * without a cache.  Copies the first min(n, 5); reset != 0 zeroes the counters [1..4] after the copy.  Synchronises the model
 * stream. */
int wd_host_cache_stats(WdModel *m, int64_t *out, int32_t n, int32_t reset);
/* Cumulative counters of the catch-up of WD_PLACE_DEFER_ADAM tables: out[0] rows caught up (staged or settled with at least one
 * missed step), [1] steps replayed, [2] steps skipped because a row's values had stopped changing (past the last step whose
 * lr_t differs from lr), [3] the longest gap (missed steps of one row) seen.  Same conventions as wd_host_cache_stats: copies the
 * first min(n, 4), reset != 0 zeroes them after the copy, synchronises the model stream; all 0 without deferred tables. */
int wd_deferred_adam_stats(WdModel *m, int64_t *out, int32_t n, int32_t reset);

/* One training step: H2D copy, ids, forward, loss, backward, optimizers.  Replaces one
 * sess.run(train_op) of Estimator.train (reference python/train.py:128-133; joint.py:224-262).
 * loss_out (nullable): sum-reduced sigmoid cross entropy of this batch (joint.py:404-406). */
int wd_train_step(WdModel *m, const WdBatch *batch, float *loss_out);
/* Forward only: logits[batch_size].  Replaces Estimator.predict / the forward half of evaluate. */
int wd_forward(WdModel *m, const WdBatch *batch, float *logits_out, float *loss_out);

/* Device-resident variants used by bench.py's `value` and by multi-GPU: upload once, then step on the
 * resident batch (the e2e number uses wd_train_step with host buffers). */
int wd_batch_upload(WdModel *m, const WdBatch *batch);
int wd_train_step_resident(WdModel *m, float *loss_out);
/* Ring of device-resident batches (slot in [0, 64); buffers are allocated on first use): lets a caller
 * prefetch batch i+1 while step i runs, and lets the benchmark step through distinct resident batches. */
int wd_batch_upload_slot(WdModel *m, int slot, const WdBatch *batch);
/* Asynchronous refill — the counterpart of `dataset.prefetch(2 * batch_size)` in the reference's input_fn (python/lib/dataset.py:
 * 181-184): the host->device copies run on the library's upload stream, after the last step that read the slot and concurrently
 * with the step running on another slot; the next step on this slot waits for them on the device.  The (pinned) host buffers must
 * stay untouched until that step has been issued and has returned. */
int wd_batch_prefetch_slot(WdModel *m, int slot, const WdBatch *batch);
int wd_train_step_slot(WdModel *m, int slot, float *loss_out);   /* loss_out NULL: enqueue only, no sync */
/* Loss of the most recent forward / train step (device->host read, synchronises the model stream). */
int wd_last_loss(WdModel *m, float *loss_out);
int wd_forward_resident(WdModel *m, float *logits_out, float *loss_out);

/* Split step for data-parallel training (multi-GPU): phase 1 computes gradients and leaves
 *   dense grads  : device float[wd_dense_grad_count]  (to be sum-allreduced, joint.py loss is a SUM)
 *   sparse grads : unique rows + summed grads for the embedding and the wide tables
 * phase 2 applies the optimizers.  wd_sparse_* expose the device buffers for the exchange. */
int wd_step_backward(WdModel *m, const WdBatch *batch_or_null, float *loss_out);
int wd_step_backward_slot(WdModel *m, int slot, float *loss_out);
int wd_step_apply(WdModel *m);
int64_t wd_dense_grad_count(WdModel *m);
void *wd_dense_grad_ptr(WdModel *m);          /* device pointer */
/* Sparse gradient lists after wd_step_backward.  which: 0 = embedding rows, 1 = wide rows.
 * rows: device uint32[n] global row ids (sorted unique), grads: device float[n*width] (width 1 for wide,
 * max table dim for embeddings, rows of narrower tables are zero padded).  Entries [n, capacity) of `rows` hold
 * 0xFFFFFFFF (skipped by wd_sparse_set), so a fixed-size exchange needs no count: pass n = NULL to skip the
 * host synchronisation that reading the count requires. */
int wd_sparse_grads(WdModel *m, int which, void **rows, void **grads, int64_t *n, int32_t *width, int64_t *capacity);
/* Replace the sparse gradient list by a merged one (rows need not be unique or sorted). */
int wd_sparse_set(WdModel *m, int which, const void *rows_dev, const void *grads_dev, int64_t n);
/* Same, for the concatenation of n_lists lists of list_len rows each that are individually sorted ascending, duplicate-free
 * and padded with 0xFFFFFFFF — exactly what a fixed-size all-gather of wd_sparse_grads' buffers yields.  Merged without a
 * sort (one binary search per list and element); duplicates across lists are summed in list order.  With the same buffers
 * every step the merge is replayed from a CUDA graph.  (Replaces the push of sparse updates to the parameter servers,
 * reference python/train.py:197-217.) */
int wd_sparse_set_sorted(WdModel *m, int which, const void *rows_dev, const void *grads_dev, int32_t n_lists, int64_t list_len);

/* ---- Row-sharded tables (WdPlanDesc::shard_world > 1).  Replaces the partitioned variables + parameter-server pulls / pushes of
 * the reference's distributed mode (reference python/lib/joint.py:141-143 min_max_variable_partitioner; python/train.py:197-217)
 * with a synchronous, exact exchange through PEER MEMORY over NVLink: ids go to their owners, owners return pooled partial sums,
 * gradients are pulled by the owners inside their segmented reduction, dense gradients are all-reduced by a two-shot kernel.  No
 * collective library is involved; the ranks only need each other's exchange segment mapped.
 *   one process per GPU : every rank calls wd_shard_ipc_handle, the 64-byte handles are all-gathered by the host (any transport),
 *                         wd_shard_connect_ipc maps the peers; then wd_shard_train_step_slot / wd_shard_forward_slot are
 *                         COLLECTIVE calls (every rank, once per step); ranks meet at flag barriers in peer memory.
 *   one process, G handles (tests, also on a single GPU): wd_shard_connect_local; then for k = 0..4: wd_shard_phase on every
 *                         rank, which runs segment k of the rank-step that wd_shard_train_step_slot runs whole, followed by
 *                         wd_shard_local_sync, which stands in for the flag barriers closing the segment (events); then
 *                         wd_shard_finish for the loss.
 * Parameters of sharded tables are addressed per rank: wd_tensor_io / wd_tensor_size see this rank's rows (global rows rank,
 * rank + G, rank + 2G, ...). */
int wd_shard_info(WdModel *m, int32_t *world, int32_t *rank, int64_t *segment_bytes);
int wd_shard_ipc_handle(WdModel *m, void *handle_out64);                                   /* 64 bytes (cudaIpcMemHandle_t) */
int wd_shard_connect_ipc(WdModel *m, const void *handles /* n_ranks x 64 bytes, rank order */, int32_t n_ranks);
int wd_shard_connect_local(WdModel **models /* rank order */, int32_t n_ranks);
int wd_shard_local_sync(WdModel **models, int32_t n_ranks);
int wd_shard_phase(WdModel *m, int slot, int phase, int train);
int wd_shard_finish(WdModel *m, float *loss_out /* nullable */, float *logits_out /* nullable, [batch] */);
int wd_shard_train_step_slot(WdModel *m, int slot, float *loss_out /* NULL: enqueue only */);
int wd_shard_forward_slot(WdModel *m, int slot, float *logits_out, float *loss_out);
/* Evaluation of a row-sharded model.  Each rank adds the metrics of its own rows to its accumulator (wd_eval_reset first), on the
 * device; wd_shard_eval_finish then sums the accumulators of all ranks in rank order and returns the ten values of wd_eval_finish,
 * the same bytes on every rank.  Every rank enters every forward: a rank whose shard of the data has run out uploads any one-row
 * batch and passes n_valid = 0 (rows are masked by n_valid, not by weights).  "loss" is the mean over steps of the step's sum over
 * the rows of all ranks.  wd_eval_reset / wd_eval_finish still see this rank's accumulator alone.
 *   one process per GPU : wd_shard_eval_accumulate_slot (collective, once per step) = sharded forward of the slot's batch + metrics
 *                         of its first n_valid rows; graphed per slot and n_valid.  wd_shard_eval_finish (collective).
 *   one process, G handles: wd_shard_phase(train = 0) for segments 0..2 as for a forward, then wd_shard_eval_accumulate_phase on every
 *                         rank; after the last step wd_shard_local_sync, then wd_shard_eval_finish on every rank. */
int wd_shard_eval_accumulate_slot(WdModel *m, int slot, int32_t n_valid);
int wd_shard_eval_accumulate_phase(WdModel *m, int32_t n_valid);
int wd_shard_eval_finish(WdModel *m, double *out10);

/* Streaming eval metrics (binary head, reference joint.py:402-406): accumulate per batch, then finish.
 * out[0..9] = accuracy, accuracy_baseline, auc, auc_precision_recall, average_loss, label/mean, loss,
 *             precision, prediction/mean, recall. */
int wd_eval_reset(WdModel *m);
int wd_eval_accumulate(WdModel *m, const WdBatch *batch);
int wd_eval_finish(WdModel *m, double *out10);
/* wd_eval_accumulate on the batch a slot already holds (wd_batch_prefetch_slot, wd_tsv_parse_slot). */
int wd_eval_accumulate_slot(WdModel *m, int slot);

/* Stand-alone integer kernels (device), exposed so parity tests can check them bit-exactly:
 * Fingerprint64 over byte strings; hash-bucket; SparseCross chain. */
int wd_fingerprint64_device(const uint8_t *bytes, const int64_t *offsets, int64_t n, uint64_t *out);
/* Host implementations used by the TSV loader (same source, compiled for the host). */
uint64_t wd_fingerprint64(const uint8_t *bytes, size_t n);
uint64_t wd_fingerprint_cat64(uint64_t a, uint64_t b);

/* Column ids of the last uploaded/stepped batch, for parity tests: CSR over (row, column). */
int wd_debug_column_ids(WdModel *m, int32_t *offsets_out, int64_t offsets_cap, int64_t *ids_out, int64_t ids_cap, int64_t *nnz_out);
/* The batch slot `slot` holds, read back after its pending refill: *batch_out rows, *nnz_out keys, *parts_out bit 0 / 1 / 2 =
 * offsets / label / weight present.  Non-NULL arrays receive offsets[B * n_cat_fields + 1], keys[nnz], dense[B * n_dense_fields],
 * label[B], weight[B] (call with NULL arrays first for the sizes). */
int wd_debug_slot(WdModel *m, int slot, int32_t *batch_out, int64_t *nnz_out, int32_t *parts_out, int32_t *offsets_out,
                  uint64_t *keys_out, float *dense_out, float *label_out, float *weight_out);
/* Deep input matrix of the last forward: [batch, d0_phys]. */
int wd_debug_deep_input(WdModel *m, float *out, int64_t cap);
/* Output of hidden layer `layer` of tower `tower` after the last forward: [batch, N_phys]; returns N_phys.  On the bf16x3 engine a
 * layer that only other hidden layers read has no fp32 copy: it comes back as hi + lo of its bf16 copies, the value those layers'
 * GEMMs read. */
int wd_debug_hidden(WdModel *m, int tower, int layer, float *out, int64_t cap);
/* Kernel launch counter (launches of this library's kernels since creation). */
int64_t wd_launch_count(WdModel *m);
/* How many MLP GEMMs of a tensor-core engine (tc3x / tc1x) were handed to the fp32 FFMA kernel because their shape is not
 * covered by the wgmma kernel.  0 for every plan the library builds itself (all widths are padded to whole k-blocks); the
 * tests assert 0 so a silent downgrade cannot hide. */
int64_t wd_gemm_fallback_count(WdModel *m);
/* Step graphs since creation: out[0] = captures, out[1] = replays (launches of a graph captured by an earlier call).  A capture
 * that fails leaves the model eager for good without an error, so tests that mean to run a graph read these. */
int wd_graph_stats(WdModel *m, int64_t *out, int32_t n);
/* Per-phase device timings of the last synchronised step in milliseconds (CUDA events recorded on the model
 * stream between the stages, enabled by wd_set_profile).  Returns the number of phases n and fills
 * ms_out[0..min(n,cap)): [0] = whole step, [i] = the phase ending at mark wd_timing_name(m, i). */
int wd_last_timings(WdModel *m, float *ms_out, int cap);
const char *wd_timing_name(WdModel *m, int i);
int wd_set_profile(WdModel *m, int enable);
void *wd_stream(WdModel *m);
/* Timeline probe of the 3xBF16 GEMM (set WD_GEMM_PROBE=1 before the first launch): globaltimer stamps of CTA 0 for the last 32
 * launches, 8 per launch — kernel start, first operands landed, main loop of the first / last tile done, epilogue of the first tile
 * start / end, epilogue of the last tile start / end; out: uint64[256].  tools/gemm_probe.py prints them per layer. */
int wd_debug_gemm_probe(unsigned long long *out);
/* Stream on which sparse gradient list `which` is produced and on which wd_sparse_set(_sorted) will merge it and
 * wd_step_apply will apply it: each list has its own side stream, so its exchange overlaps the other list's and the
 * dense all-reduce on wd_stream. */
void *wd_stream_sparse(WdModel *m, int which);
int wd_sync(WdModel *m);

/* Layer summaries (the reference's add_layer_summary, python/lib/utils/model_util.py:15-17): statistics of the tensors a train
 * step's towers produce, taken on the GPU in the step's forward, before its optimizer.  Segments, in this order: the deep input
 * (its logical columns), per tower its hidden layers (the layer output, dropout and batch normalization included) and its logits,
 * then the wide logit.  Per segment: counts over TensorFlow's 1551 default histogram limits (value v, as a double, counts in
 * bucket i = the first i with limit[i] > v), the number of values, of zeros (-0.0 included) and of non-finite values (counted in
 * no bucket), and min, max, sum and sum of squares of the finite values, in double. */
#define WD_SUMMARY_BUCKETS 1551
enum { WD_SEG_DEEP_INPUT = 0, WD_SEG_HIDDEN = 1, WD_SEG_TOWER_LOGITS = 2, WD_SEG_WIDE_LOGIT = 3 };
/* The 1551 ascending bucket limits into out[0 .. cap); returns 1551 (out NULL: only the count).  Needs no GPU. */
int wd_summary_limits(double *out, int32_t cap);
/* The model's segments: kind[i] (WD_SEG_*), tower[i] and layer[i] (-1 where they do not apply) for the first `cap`; returns how
 * many there are. */
int wd_summary_segments(WdModel *m, int32_t *kind, int32_t *tower, int32_t *layer, int32_t cap);
/* The next train step (wd_train_step*, wd_step_backward*, the row-sharded rank-step) takes the statistics.  It runs outside the
 * step graphs; every other step stays as it is. */
int wd_summary_arm(WdModel *m);
/* Statistics of the last armed step (synchronises the model stream): counts[n][WD_SUMMARY_BUCKETS], ints[n][3] = values, zeros,
 * non-finite values, reals[n][4] = min, max, sum, sum of squares; n_segments must be the wd_summary_segments count.  WD_ESTATE
 * when no armed step ran since the last read. */
int wd_summary_read(WdModel *m, int64_t *counts, int64_t *ints, double *reals, int32_t n_segments);

/* TSV loader (host, multi-threaded).  Replaces _CsvDataset._parse_csv (reference python/lib/dataset.py:107-165):
 * parses `n_lines` tab-separated records into the WdBatch CSR arrays. */
typedef struct WdTsvSpec {
    int32_t n_columns;              /* columns per record incl. label when has_label */
    const int32_t *col_role;        /* per file column: -1 skip, 0 label, 1 string cat field, 2 int cat field, 3 dense */
    const int32_t *col_target;      /* field index for roles 1,2,3 */
    int32_t n_cat_fields, n_dense_fields;
    int32_t multivalue;             /* split string fields on ',' and drop empty tokens */
    int32_t tf_compat_pad;          /* quirk Q2: pad string fields to the batch max length with Fingerprint64("") */
    float pos_weight, neg_weight;   /* used when use_weight */
    int32_t use_weight;
    int32_t has_label;
} WdTsvSpec;
/* Returns nnz, or negative error.  keys_cap == 0 (or keys_out NULL), or nnz > keys_cap: only counts (offsets, dense, label and
 * weight are filled, no key is copied) — call again with a buffer of nnz keys and the same arguments otherwise: the follow-up call
 * copies the keys of the parse the first call did (one parse per batch).  Without tf_compat_pad
 * n_lines * n_cat_fields + number of ',' in the text is an upper bound of nnz. */
int64_t wd_tsv_parse(const WdTsvSpec *spec, const char *text, int64_t text_len, int32_t n_lines,
                     int32_t *offsets_out, uint64_t *keys_out, int64_t keys_cap,
                     float *dense_out, float *label_out, float *weight_out, int32_t n_threads);
/* Line index of a file image, for shuffled / sharded passes without splitting or joining text (reference python/lib/dataset.py:
 * 167-184: TextLineDataset -> shard -> shuffle -> batch): start offsets and lengths of the non-empty lines ('\r' before the
 * newline excluded).  Returns the number of lines (the arrays receive the first `cap` of them; pass NULL / 0 to count). */
int64_t wd_tsv_index_lines(const char *text, int64_t text_len, int64_t *starts_out, int32_t *lens_out, int64_t cap);
/* wd_tsv_parse over lines picked through that index: line i of the batch is text[starts[idx[i]] .. + lens[idx[i]]) (idx NULL:
 * line i).  Same outputs and return value as wd_tsv_parse. */
int64_t wd_tsv_parse_lines(const WdTsvSpec *spec, const char *text, const int64_t *starts, const int32_t *lens, const int64_t *idx,
                           int32_t n_lines, int32_t *offsets_out, uint64_t *keys_out, int64_t keys_cap,
                           float *dense_out, float *label_out, float *weight_out, int32_t n_threads);

/* The lines idx[0 .. n) of a file image (starts / lens from wd_tsv_index_lines; idx NULL: lines 0 .. n) copied into `out`, each
 * followed by '\n', on the loader's worker threads; out_starts[i] = offset of line i, out_starts[n] = total bytes.  Returns the
 * total; when it exceeds out_cap (or out is NULL) only out_starts is written.  Needs no GPU. */
int64_t wd_tsv_gather_lines(const char *text, const int64_t *starts, const int32_t *lens, const int64_t *idx, int32_t n,
                            char *out, int64_t out_cap, int64_t *out_starts, int32_t n_threads);
/* Device TSV parser: the n_lines lines of `text` (line i = text[starts[i], starts[i + 1] - 1), a trailing '\r' excluded; the
 * layout wd_tsv_gather_lines writes) are copied to the GPU and parsed there straight into batch slot `slot`, on the upload stream
 * behind the last step that read the slot (as wd_batch_prefetch_slot).  The slot then holds exactly what wd_tsv_parse_lines +
 * wd_batch_prefetch_slot would put there (label only with spec->has_label, weight only with use_weight and has_label).  Returns
 * when this parse has finished; `text` and `starts` may then be reused.  Records outside the exact int / float fast paths, a
 * wrong field count or more keys than the slot holds are parsed on the host instead, so errors carry the host parser's messages. */
int wd_tsv_parse_slot(WdModel *m, int slot, const WdTsvSpec *spec, const char *text, int64_t text_len, const int64_t *starts,
                      int32_t n_lines);
/* out[0] batches wd_tsv_parse_slot parsed on the device, out[1] batches it handed to the host parser (first min(n, 2)). */
int wd_tsv_parse_stats(WdModel *m, int64_t *out, int32_t n, int32_t reset);

/* Page-locked host buffers for the input pipeline (the `dataset.prefetch` buffers of the reference's input_fn, python/lib/
 * dataset.py:181-184): parse into these, hand them to wd_batch_prefetch_slot.  WD_ENODEVICE without a CUDA device. */
int wd_host_alloc(size_t bytes, void **out);
int wd_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif /* WD_B200_H_ */
