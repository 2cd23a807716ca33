"""Feature plan compiler: conf/*.yaml -> one immutable ``Plan`` the CUDA library consumes.

Replaces ``_build_model_columns`` (reference python/lib/build_estimator.py:49-169): instead of a list of
``tf.feature_column`` objects evaluated op-by-op each step, the YAML is compiled ONCE into flat slot tables
(categorical columns, embedding tables, wide row ranges, deep-input offsets, MLP topology, optimizer
hyper-parameters) that are handed to ``wd_model_create`` through the C-ABI (include/wd_b200.h: WdPlanDesc).

Semantics kept from the reference / TensorFlow (SURVEY.md Appendix A):
  * hash_bucket -> wide column + mean-pooled embedding of dim 2**ceil(ln(n**0.25))    (build_estimator.py:57-59,83-99)
  * vocab / identity -> wide column + indicator (multi-hot counts)                     (:101-120)
  * continuous -> numeric deep column (normalised); boundaries add a wide bucketized column OF THE
    NORMALISED value (quirk Q3)                                                        (:121-136)
  * crosses: keys are raw string features, identity columns, or bucketized RAW continuous values; the
    hash chain runs over categorical-column keys first, then raw string keys (SparseCross op order, A.5);
    optional embedding                                                                 (:138-158)
  * deep input = columns concatenated in sorted column-name order                      (dnn.py:88-90)
Physical layout: every deep column starts on a 4-float boundary and the deep input is padded to a multiple
of 32 floats (padding stays zero), so rows are 128-byte aligned and tensor-core K tiles need no tail.
"""
from __future__ import annotations

import ast
import ctypes
import math
import re
from collections import OrderedDict

import numpy as np

COL_HASH, COL_VOCAB, COL_IDENTITY, COL_BUCKET, COL_CROSS = range(5)
NORM = {None: 0, "min_max": 1, "standard": 2, "log": 3}
KEY_FIELD, KEY_COLUMN = 0, 1
OPT = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 3, "rmsprop": 4}
ACTS = ["relu", "relu6", "sigmoid", "tanh", "leaky_relu", "elu", "selu", "softplus", "softsign", "crelu"]      # WD_ACT_*
MODES = ["simple", "first_dense", "last_dense", "dense", "resnet"]
T_WIDE_COL, T_EMB_TABLE, T_DENSE, T_WIDE_BIAS = range(4)
D_KERNEL, D_BIAS, D_GAMMA, D_BETA = range(4)
GEMM = {"auto": 0, "ffma": 1, "tc3x": 2, "tc1x": 3, "bf16x3": 4}
PLACE_HBM, PLACE_HOST, PLACE_AUTO = range(3)      # WD_PLACE_*
PLACE_DEFER_ADAM = 4                              # WD_PLACE_DEFER_ADAM, OR'ed into host / auto entries
PLACE_NAMES = {PLACE_HBM: "hbm", PLACE_HOST: "host", PLACE_AUTO: "auto",
               PLACE_HOST | PLACE_DEFER_ADAM: "host+defer", PLACE_AUTO | PLACE_DEFER_ADAM: "auto+defer"}
API_VERSION = 3                                   # WD_API_VERSION


def embedding_dim(n):
    """Empirical embedding width of the reference: natural log (build_estimator.py:57-59, quirk Q12)."""
    return int(np.power(2, np.ceil(np.log(n ** 0.25))))


def _pad(n, m):
    return (n + m - 1) // m * m


def parse_optimizer(spec, default_lr):
    """'Adagrad' | 'Adam' | 'Ftrl' | 'RMSProp' | 'SGD' with the conf learning rate — the five names of the reference's factory
    (reference model_util.py:84-90) — or a ``tf.train.XOptimizer(...)`` constructor string whose own arguments win (the
    reference eval()s it, model_util.py:95-101; here it is parsed, never evaluated).  TensorFlow's defaults: Adam beta1 0.9 /
    beta2 0.999 / epsilon 1e-8 / learning_rate 0.001; RMSProp decay 0.9 / momentum 0 / epsilon 1e-10."""
    simple = {"Adagrad": "adagrad", "Ftrl": "ftrl", "SGD": "sgd", "Adam": "adam", "RMSProp": "rmsprop"}
    base = dict(l1=0.0, l2=0.0, lr_power=-0.5, init_acc=0.1, beta1=0.9, beta2=0.999, epsilon=1e-8, rho=0.9, momentum=0.0)
    if spec in simple:
        o = dict(base, kind=simple[spec], lr=float(default_lr))
        if o["kind"] == "rmsprop":
            o["epsilon"] = 1e-10
        return o
    m = re.match(r"^\s*tf\.train\.(\w+)Optimizer\((.*)\)\s*$", str(spec))
    cls = {"Adagrad": "adagrad", "Ftrl": "ftrl", "GradientDescent": "sgd", "Adam": "adam", "RMSProp": "rmsprop"}.get(m.group(1)) if m else None
    if cls is None:
        raise ValueError("Unsupported optimizer option: `{}`. Supported names are: "
                         "('Adagrad', 'Adam', 'Ftrl', 'RMSProp', 'SGD') or a tf.train.{{Adagrad,Adam,Ftrl,RMSProp,GradientDescent}}"
                         "Optimizer(...) expression.".format(spec))
    call = ast.parse("f(" + m.group(2) + ")", mode="eval").body
    kw = {k.arg: ast.literal_eval(k.value) for k in call.keywords}
    if call.args:
        kw.setdefault("learning_rate", ast.literal_eval(call.args[0]))
    if "learning_rate" not in kw and cls != "adam":           # (tf.train.AdamOptimizer has a default learning rate, 0.001)
        raise ValueError("learning_rate must be specified in `{}`".format(spec))
    if cls == "rmsprop" and kw.get("centered"):
        raise ValueError("centered RMSProp is not supported: `{}`".format(spec))
    return dict(kind=cls, lr=float(kw.get("learning_rate", 0.001)),
                l1=float(kw.get("l1_regularization_strength", 0.0)),
                l2=float(kw.get("l2_regularization_strength", 0.0)),
                lr_power=float(kw.get("learning_rate_power", -0.5)),
                init_acc=float(kw.get("initial_accumulator_value", 0.1)),
                beta1=float(kw.get("beta1", 0.9)), beta2=float(kw.get("beta2", 0.999)),
                epsilon=float(kw.get("epsilon", 1e-8 if cls == "adam" else 1e-10)),
                rho=float(kw.get("decay", 0.9)), momentum=float(kw.get("momentum", 0.0)))


class _OptC(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("lr", ctypes.c_float), ("l1", ctypes.c_float), ("l2", ctypes.c_float),
                ("lr_power", ctypes.c_float), ("init_acc", ctypes.c_float), ("beta1", ctypes.c_float), ("beta2", ctypes.c_float),
                ("epsilon", ctypes.c_float), ("rho", ctypes.c_float), ("momentum", ctypes.c_float)]


class PlanDescC(ctypes.Structure):
    """ctypes image of WdPlanDesc (include/wd_b200.h) — field order must match."""
    _P = ctypes.c_void_p
    _fields_ = [
        ("api_version", ctypes.c_int32), ("model_type", ctypes.c_int32),
        ("n_cat_fields", ctypes.c_int32), ("n_dense_fields", ctypes.c_int32),
        ("cat_field_is_string", _P),
        ("n_columns", ctypes.c_int32),
        ("col_kind", _P), ("col_field", _P), ("col_buckets", _P), ("col_aux_off", _P), ("col_aux_n", _P),
        ("col_norm_kind", _P), ("col_norm_a", _P), ("col_norm_b", _P),
        ("col_wide_base", _P), ("col_emb_table", _P), ("col_ind_off", _P),
        ("vocab_fp", _P), ("n_vocab_fp", ctypes.c_int32),
        ("boundaries", _P), ("n_boundaries", ctypes.c_int32),
        ("cross_key_type", _P), ("cross_key_idx", _P), ("n_cross_keys", ctypes.c_int32),
        ("n_tables", ctypes.c_int32), ("table_rows", _P), ("table_dim", _P), ("table_dim_logical", _P),
        ("table_x0_off", _P),
        ("n_numeric", ctypes.c_int32), ("num_field", _P), ("num_norm_kind", _P), ("num_x0_off", _P),
        ("num_norm_a", _P), ("num_norm_b", _P),
        ("d0_phys", ctypes.c_int32), ("wide_rows", ctypes.c_int64),
        ("n_towers", ctypes.c_int32), ("tower_nlayers", _P), ("tower_mode", _P), ("hidden_units", _P),
        ("activation", ctypes.c_int32), ("batch_norm", ctypes.c_int32),
        ("lin_opt", _OptC), ("dnn_opt", _OptC),
        ("max_batch", ctypes.c_int32), ("max_nnz", ctypes.c_int64), ("max_keys", ctypes.c_int64),
        ("gemm_engine", ctypes.c_int32),
        ("dense_exchange_max_rows", ctypes.c_int64), ("wide_small_base", ctypes.c_int64),
        ("shard_world", ctypes.c_int32), ("shard_rank", ctypes.c_int32),
        ("table_sharded", _P), ("col_wide_sharded", _P),
        ("shard_capacity", ctypes.c_int64), ("shard_slack", ctypes.c_float),
        ("dropout_rate", ctypes.c_float), ("dropout_seed", ctypes.c_uint64),
        ("table_placement", _P),
    ]


class Column(object):
    """One categorical column (id producer)."""
    __slots__ = ("name", "kind", "field", "buckets", "aux", "norm", "wide_base", "emb_table", "ind_off", "keys")

    def __init__(self, name, kind, field=-1, buckets=0, aux=None, norm=(0, 0.0, 0.0), keys=None):
        self.name, self.kind, self.field, self.buckets = name, kind, field, int(buckets)
        self.aux, self.norm, self.keys = aux, norm, keys
        self.wide_base, self.emb_table, self.ind_off = -1, -1, -1


class Plan(object):
    """Compiled model description.  Attributes of interest:
      cat_fields / dense_fields : ordered input field names (batch layout)
      columns                   : list[Column] in evaluation order
      tables                    : list of dict(name, column, rows, dim, x0_off, sharded, placement = PLACE_*)
      numerics                  : list of dict(name, field, norm, x0_off)
      deep_layout               : OrderedDict column name -> (logical offset, physical offset, width)
      towers                    : list of dict(hidden, mode)
      tensor_names              : OrderedDict TF variable name -> (kind, index, sub, logical shape)
    """

    def __init__(self, feature_conf, cross_conf, model_conf, model_type="wide_deep", max_batch=8192,
                 embedding_dim_override=None, tf_compat_pad=False, gemm_engine="auto", max_nnz=0, max_keys=0,
                 dense_exchange_max_rows=0, shard_world=1, shard_rank=0, shard_capacity=0, shard_slack=2.0, host_tables=None,
                 host_cache_bytes=0, shard_cache_bytes=0, defer_adam=False):
        if model_type not in ("wide", "deep", "wide_deep"):
            raise ValueError("Invalid model type: {}, must be one of `wide`, `deep`, `wide_deep`".format(model_type))
        self.model_type, self.max_batch, self.tf_compat_pad = model_type, int(max_batch), bool(tf_compat_pad)
        self.use_wide, self.use_deep = model_type != "deep", model_type != "wide"
        self.gemm_engine, self.max_nnz, self.max_keys = gemm_engine, int(max_nnz), int(max_keys)
        # data-parallel exchange format: tables / wide columns with at most this many rows travel as a dense gradient block
        # (all-reduced with the dense gradients) instead of (row, gradient) list entries; 0 = lists for everything
        self.dense_exchange_max_rows = int(dense_exchange_max_rows)
        # Row-sharded tables (the reference partitions large variables over the parameter servers with
        # min_max_variable_partitioner, python/lib/joint.py:141-143): with shard_world = G > 1 every embedding table / wide
        # column LARGER than dense_exchange_max_rows is split by row over the G ranks (row id -> rank id mod G, local row id // G);
        # the smaller ones stay replicated and exchange a dense gradient block.  So in sharded runs every table is one or the other
        # and no (row, gradient) list ever travels.
        self.shard_world, self.shard_rank = int(shard_world), int(shard_rank)
        self.shard_capacity, self.shard_slack = int(shard_capacity), float(shard_slack)
        if self.shard_world > 1 and self.dense_exchange_max_rows <= 0:
            self.dense_exchange_max_rows = 16384
        if not (0 <= self.shard_rank < max(self.shard_world, 1)):
            raise ValueError("shard_rank {} outside [0, {})".format(self.shard_rank, self.shard_world))
        is_sharded = lambda rows: self.shard_world > 1 and rows > self.dense_exchange_max_rows
        edim = (lambda n: int(embedding_dim_override)) if embedding_dim_override else embedding_dim

        # ---- input fields
        self.cat_fields, self.cat_is_string, self.dense_fields = [], [], []
        for f, c in feature_conf.items():
            if c["type"] == "category":
                self.cat_fields.append(f)
                self.cat_is_string.append(0 if c["transform"] == "identity" else 1)
            else:
                self.dense_fields.append(f)
        cat_idx = {f: i for i, f in enumerate(self.cat_fields)}
        dense_idx = {f: i for i, f in enumerate(self.dense_fields)}

        # ---- columns
        cols, self._vocab_fp, self._bounds = [], [], []
        deep = []   # (sorted-name key, kind, payload)
        self.vocab_tokens = {}

        def add_bounds(b):
            off = len(self._bounds)
            self._bounds.extend(float(x) for x in b)
            return (off, len(b))

        from . import _hashing_host as HH  # host Fingerprint64 (product code; C library)
        for f, c in feature_conf.items():
            t, tr, p = c["type"], c["transform"], c["parameter"]
            if t == "category":
                if tr == "hash_bucket":
                    col = Column(f, COL_HASH, cat_idx[f], p)
                    cols.append(col)
                    deep.append((f + "_embedding", "emb", (col, edim(p))))
                elif tr == "vocab":
                    toks = [str(v) for v in p]          # build_estimator.py:103 map(str, ...)
                    off = len(self._vocab_fp)
                    self._vocab_fp.extend(HH.fingerprint64(s) for s in toks)
                    col = Column(f, COL_VOCAB, cat_idx[f], len(toks), aux=(off, len(toks)))
                    self.vocab_tokens[f] = toks
                    cols.append(col)
                    deep.append((f + "_indicator", "ind", col))
                else:
                    col = Column(f, COL_IDENTITY, cat_idx[f], p)
                    cols.append(col)
                    deep.append((f + "_indicator", "ind", col))
                col.wide_base = 0   # marks "wide column"; bases assigned below
            else:
                norm = (NORM[tr], 0.0, 0.0)
                if tr == "min_max":
                    a, b = p["normalization"]
                    norm = (1, float(a), float(b - a))          # (x-a)/(b-a): subtract, then divide by the host-computed span
                elif tr == "standard":
                    m, s = p["normalization"]
                    norm = (2, float(m), float(s))
                if p["boundaries"]:
                    col = Column(f + "_bucketized", COL_BUCKET, dense_idx[f], len(p["boundaries"]) + 1,
                                 aux=add_bounds(p["boundaries"]), norm=norm)
                    col.wide_base = 0
                    cols.append(col)
                deep.append((f, "num", (dense_idx[f], norm)))
        hidden_keys = {}
        for names, size, is_deep in cross_conf:
            keys, leaf = [], []
            for f in names:
                c = feature_conf[f]
                if c["type"] == "continuous":
                    kname = f + "_bucketized#raw"
                    if kname not in hidden_keys:      # bucketized RAW value, only ever a cross key (build_estimator.py:145)
                        hc = Column(kname, COL_BUCKET, dense_idx[f], len(c["parameter"]["boundaries"]) + 1,
                                    aux=add_bounds(c["parameter"]["boundaries"]))
                        hidden_keys[kname] = hc
                        cols.append(hc)
                    keys.append((KEY_COLUMN, hidden_keys[kname]))
                    leaf.append(f + "_bucketized")
                elif c["transform"] == "identity":
                    kname = f + "#key"
                    if kname not in hidden_keys:
                        hc = Column(kname, COL_IDENTITY, cat_idx[f], c["parameter"])
                        hidden_keys[kname] = hc
                        cols.append(hc)
                    keys.append((KEY_COLUMN, hidden_keys[kname]))
                    leaf.append(f)
                else:
                    keys.append((KEY_FIELD, cat_idx[f]))
                    leaf.append(f)
            # SparseCross op order: SparseTensor inputs (categorical-column keys) first, then dense string inputs (A.5)
            keys = [k for k in keys if k[0] == KEY_COLUMN] + [k for k in keys if k[0] == KEY_FIELD]
            col = Column("_X_".join(sorted(leaf)), COL_CROSS, -1, size, keys=keys)
            col.wide_base = 0
            cols.append(col)
            if is_deep:
                deep.append((col.name + "_embedding", "emb", (col, edim(size))))
        # cross columns must come after the columns they use as keys
        order = [c for c in cols if c.kind != COL_CROSS] + [c for c in cols if c.kind == COL_CROSS]
        self.columns = order
        col_index = {id(c): i for i, c in enumerate(order)}
        self._col_index = col_index

        # ---- wide table layout
        # (row space: large columns first, then the small ones that are exchanged densely — see dense_exchange_max_rows)
        base = 0
        self.wide_columns = []
        is_wide = [c.wide_base == 0 and self.use_wide for c in order]
        small = [w and 0 < self.dense_exchange_max_rows >= c.buckets for c, w in zip(order, is_wide)]
        self.wide_small_base = None
        self.wide_sharded = [bool(w and is_sharded(c.buckets)) for c, w in zip(order, is_wide)]
        for want_small in (False, True):
            if want_small:
                self.wide_small_base = base
            for c, w, sm, sh in zip(order, is_wide, small, self.wide_sharded):
                if w and sm == want_small and not sh:
                    c.wide_base = base
                    base += c.buckets
        for c, w, sh in zip(order, is_wide, self.wide_sharded):
            if w:
                self.wide_columns.append(c)
                if sh:
                    c.wide_base = -1                  # rows live in the sharded wide space, not in the replicated one
            else:
                c.wide_base = -1
        self.wide_rows = base

        # ---- deep input layout (sorted column-name order, A.7)
        self.tables, self.numerics, self.deep_layout = [], [], OrderedDict()
        lo = po = 0
        if self.use_deep:
            for name, kind, payload in sorted(deep, key=lambda d: d[0]):
                po = _pad(po, 4)
                if kind == "emb":
                    col, dim = payload
                    col.emb_table = len(self.tables)
                    self.tables.append(dict(name=name, column=col, rows=col.buckets, dim=dim, x0_off=po, sharded=bool(is_sharded(col.buckets))))
                    width = dim          # physical width is _pad(dim, 4); the next column re-aligns to 4 anyway
                elif kind == "ind":
                    payload.ind_off = po
                    width = payload.buckets
                else:
                    fld, norm = payload
                    self.numerics.append(dict(name=name, field=fld, norm=norm, x0_off=po))
                    width = 1
                self.deep_layout[name] = (lo, po, width)
                lo += width
                po += width
        self.d0, self.d0_phys = lo, max(32, _pad(po, 32)) if self.use_deep else 0

        # ---- table placement (WD_PLACE_*).  None: auto — the library keeps every table in HBM that fits there and moves only the
        # tables whose HBM allocation fails to page-locked host memory.  "all" / a list of table names: exactly those tables in host
        # memory, every other one in HBM.
        self.host_tables = host_tables
        names = [t["name"] for t in self.tables]
        if host_tables is None:
            want = None
        elif isinstance(host_tables, str):
            if host_tables != "all":
                raise ValueError("host_tables must be None, 'all' or a list of embedding table names, got {!r}".format(host_tables))
            want = set(names)
        else:
            want = set(host_tables)
            unknown = sorted(want - set(names))
            if unknown:
                raise ValueError("host_tables: no embedding table named {} (tables: {})".format(unknown, names))
        # defer_adam: host and auto tables may be trained with the Adam dnn optimizer.  Sparse Adam moves every row every step; a
        # deferred table instead replays the steps a row missed when the row is next read (results unchanged, each missed step
        # costs one replayed step of that row until its values stop changing).  The library ignores it for other optimizers.
        self.defer_adam = bool(defer_adam)
        for t in self.tables:
            t["placement"] = PLACE_AUTO if want is None else (PLACE_HOST if t["name"] in want else PLACE_HBM)
            if self.defer_adam and t["placement"] != PLACE_HBM:
                t["placement"] |= PLACE_DEFER_ADAM
        # HBM budget (bytes) of the write-back cache of host-table records (wd_host_cache_enable); 0 = no cache.  The model has
        # a cache only when some table ended up on the host.
        if isinstance(host_cache_bytes, bool) or not isinstance(host_cache_bytes, (int, np.integer)) or host_cache_bytes < 0:
            raise ValueError("host_cache_bytes must be an int >= 0, got {!r}".format(host_cache_bytes))
        self.host_cache_bytes = int(host_cache_bytes)
        # HBM budget (bytes, per rank) of the owner's write-back cache of its host-placed shard records (wd_shard_cache_enable);
        # 0 = no cache.  Row-sharded plans only: one GPU caches its host tables through host_cache_bytes.
        if isinstance(shard_cache_bytes, bool) or not isinstance(shard_cache_bytes, (int, np.integer)) or shard_cache_bytes < 0:
            raise ValueError("shard_cache_bytes must be an int >= 0, got {!r}".format(shard_cache_bytes))
        if shard_cache_bytes > 0 and self.shard_world <= 1:
            raise ValueError("shard_cache_bytes caches the host shards of a row-sharded model (shard_world > 1); "
                             "a single-GPU model caches its host tables through host_cache_bytes")
        self.shard_cache_bytes = int(shard_cache_bytes)

        # ---- MLP
        hu = model_conf.get("dnn_hidden_units") or []
        towers = [list(h) for h in hu] if hu and isinstance(hu[0], (list, tuple)) else [list(hu)]
        cm = model_conf.get("dnn_connected_mode") or "simple"
        modes = [cm] * len(towers) if isinstance(cm, str) else list(cm)
        for m in modes:
            if m not in MODES:
                raise AssertionError("Invalid connected_mode: {}".format(m))
        self.towers = [dict(hidden=h, mode=m) for h, m in zip(towers, modes)] if self.use_deep else []
        act = model_conf.get("dnn_activation_function") or "relu"
        if act not in ACTS:
            raise ValueError("Unsupported activation name: {}. Supported names are: {}".format(act, tuple(sorted(ACTS))))
        self.activation = act
        self.batch_norm = 1 if model_conf.get("dnn_batch_normalization") else 0
        # dnn_dropout: tf.layers.dropout(rate) after every hidden layer's activation in TRAIN mode (reference dnn.py:111-112)
        self.dropout = float(model_conf.get("dnn_dropout") or 0.0)
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError("dnn_dropout must be in [0, 1), found {}".format(self.dropout))
        self.dropout_seed = 0x5EED0006
        # constant learning rates (quirk Q1: the reference's decay never advances, joint.py:145 vs 227)
        self.lin_opt = parse_optimizer(model_conf.get("linear_optimizer") or "Ftrl",
                                       model_conf.get("linear_initial_learning_rate") or 0.005)
        self.dnn_opt = parse_optimizer(model_conf.get("dnn_optimizer") or "Adagrad",
                                       model_conf.get("dnn_initial_learning_rate") or 0.001)

        # ---- tensor names (TensorFlow variable names of the reference's checkpoint)
        T = self.tensor_names = OrderedDict()
        for c in self.wide_columns:
            T["linear/linear_model/%s/weights" % c.name] = (T_WIDE_COL, col_index[id(c)], 0, (c.buckets,))
        if self.use_wide:
            T["linear/linear_model/bias_weights"] = (T_WIDE_BIAS, 0, 0, (1,))
        for i, t in enumerate(self.tables):
            T["dnn/input_from_feature_columns/input_layer/%s/embedding_weights" % t["name"]] = \
                (T_EMB_TABLE, i, 0, (t["rows"], t["dim"]))
        for ti, tw in enumerate(self.towers):
            dims = self.layer_dims(ti)
            for l, (i, o) in enumerate(dims):
                scope = "dnn/dnn_%d/" % (ti + 1) + ("hiddenlayer_%d" % l if l < len(dims) - 1 else "logits")
                did = self.dense_tensor_id(ti, l)
                T[scope + "/kernel"] = (T_DENSE, did, D_KERNEL, (i, o))
                T[scope + "/bias"] = (T_DENSE, did, D_BIAS, (o,))
                if self.batch_norm and l < len(dims) - 1:
                    T[scope + "/batch_normalization/gamma"] = (T_DENSE, did, D_GAMMA, (self.out_width(o),))
                    T[scope + "/batch_normalization/beta"] = (T_DENSE, did, D_BETA, (self.out_width(o),))

    # ------------------------------------------------------------------ helpers
    def is_sharded_tensor(self, name):
        """True for parameters of row-sharded tables / wide columns: a rank then holds global rows rank, rank + G, ..."""
        kind, index, _, _ = self.tensor_names[name]
        if self.shard_world <= 1:
            return False
        if kind == T_EMB_TABLE:
            return bool(self.tables[index]["sharded"])
        if kind == T_WIDE_COL:
            return bool(self.wide_sharded[index])
        return False

    def local_shape(self, name):
        """Shape of the part of tensor `name` this rank holds (the global shape unless the tensor is row-sharded)."""
        shape = tuple(self.tensor_names[name][3])
        if not self.is_sharded_tensor(name):
            return shape
        rows = (shape[0] - self.shard_rank + self.shard_world - 1) // self.shard_world
        return (rows,) + shape[1:]

    def dense_tensor_id(self, tower, layer):
        return sum(len(t["hidden"]) + 1 for t in self.towers[:tower]) + layer

    @staticmethod
    def layer_sources(mode, L):
        """Concat order of each hidden layer's input and of the logits input ('x' or hidden index);
        mirrors the five branches of _dnn_logit_fn (reference dnn.py:92-193)."""
        hid = []
        for l in range(L):
            if l == 0:
                hid.append(["x"])
            elif mode in ("simple", "last_dense"):
                hid.append([l - 1])
            elif mode == "first_dense":
                hid.append([l - 1, "x"])
            elif mode == "dense":
                hid.append(["x"] + list(range(l)))
            else:
                hid.append(list(range(l - 1, -1, -1)) + ["x"])
        if L == 0:
            last = ["x"]
        elif mode == "simple":
            last = [L - 1]
        elif mode == "first_dense":
            last = [L - 1, "x"]
        elif mode in ("last_dense", "dense"):
            last = ["x"] + list(range(L))
        else:
            last = list(range(L - 1, -1, -1)) + ["x"]
        return hid + [last]

    def layer_dims(self, tower):
        hu, mode = self.towers[tower]["hidden"], self.towers[tower]["mode"]
        srcs = self.layer_sources(mode, len(hu))
        w = lambda s: self.d0 if s == "x" else self.out_width(hu[s])
        return [(sum(w(s) for s in srcs[l]), hu[l] if l < len(hu) else 1) for l in range(len(hu) + 1)]

    def out_width(self, units):
        """Features a hidden layer of `units` units hands on (tf.nn.crelu doubles them, reference model_util.py:45-50)."""
        return 2 * units if self.activation == "crelu" else units

    def summary_segments(self):
        """Segments of the layer statistics, keys (kind, tower, layer) in the library's order (wd_summary_segments): the deep
        input, per tower its hidden layers and its logits, then the wide logit."""
        from .summary import SEG_DEEP_INPUT, SEG_HIDDEN, SEG_TOWER_LOGITS, SEG_WIDE_LOGIT
        out = [(SEG_DEEP_INPUT, -1, -1)] if self.use_deep else []
        for t, tw in enumerate(self.towers):
            out += [(SEG_HIDDEN, t, l) for l in range(len(tw["hidden"]))] + [(SEG_TOWER_LOGITS, t, -1)]
        if self.use_wide:
            out.append((SEG_WIDE_LOGIT, -1, -1))
        return out

    def summary_layout(self):
        """[(tag, segments)] of the reference's add_layer_summary calls in TRAIN mode.  A hidden layer's tag summarises `net` after
        the layer: its output followed by its connected mode's concatenation (dnn.py:92-193; resnet: quirk Q7); x is the deep
        input."""
        from .summary import LINEAR_TAG, SEG_DEEP_INPUT, SEG_HIDDEN, SEG_TOWER_LOGITS, SEG_WIDE_LOGIT, tower_tag
        x = (SEG_DEEP_INPUT, -1, -1)
        out = []
        for t, tw in enumerate(self.towers):
            h = lambda j: (SEG_HIDDEN, t, j)
            for l in range(len(tw["hidden"])):
                mode = tw["mode"]
                if mode in ("simple", "last_dense"):
                    segs = [h(l)]
                elif mode == "first_dense":
                    segs = [h(l), x]
                elif mode == "dense":
                    segs = [x] + [h(j) for j in range(l + 1)]
                else:
                    segs = [h(j) for j in range(l, -1, -1)] + [x]
                out.append((tower_tag(t, l), segs))
            out.append((tower_tag(t), [(SEG_TOWER_LOGITS, t, -1)]))
        if self.use_wide:
            out.append((LINEAR_TAG, [(SEG_WIDE_LOGIT, -1, -1)]))
        return out

    def exchange_rows(self, rows_per_column):
        """Upper bounds (K_emb, K_wide) on the touched rows per step that stay in the (row, gradient) lists, given the maximum
        number of ids one column contributes per step (batch size for single-valued columns): columns whose table is exchanged
        densely (dense_exchange_max_rows) contribute nothing."""
        t = self.dense_exchange_max_rows
        big = lambda n: not (0 < t >= n) and self.shard_world <= 1
        k_emb = sum(rows_per_column for tb in self.tables if big(tb["rows"]))
        k_wide = sum(rows_per_column for c in self.wide_columns if big(c.buckets))
        return k_emb, k_wide

    def summary(self):
        return dict(model_type=self.model_type, cat_fields=len(self.cat_fields), dense_fields=len(self.dense_fields),
                    columns=len(self.columns), wide_columns=len(self.wide_columns), wide_rows=self.wide_rows,
                    tables=len(self.tables), table_rows=sum(t["rows"] for t in self.tables),
                    table_params=sum(t["rows"] * t["dim"] for t in self.tables),
                    deep_dim=self.d0, deep_dim_phys=self.d0_phys,
                    towers=[(t["hidden"], t["mode"]) for t in self.towers],
                    placement=OrderedDict((t["name"], PLACE_NAMES[t["placement"]]) for t in self.tables))

    # ------------------------------------------------------------------ C image
    def to_c(self):
        """-> (PlanDescC, keepalive list of numpy arrays)."""
        keep = []

        def arr(x, dt):
            a = np.ascontiguousarray(np.asarray(x, dtype=dt))
            if a.size == 0:
                a = np.zeros(1, dtype=dt)
            keep.append(a)
            return a.ctypes.data

        C = self.columns
        ci = self._col_index
        ck_type, ck_idx, aux_off, aux_n = [], [], [], []
        for c in C:
            if c.kind == COL_CROSS:
                aux_off.append(len(ck_type))
                aux_n.append(len(c.keys))
                for kt, kv in c.keys:
                    ck_type.append(kt)
                    ck_idx.append(kv if kt == KEY_FIELD else ci[id(kv)])
            elif c.aux is not None:
                aux_off.append(c.aux[0])
                aux_n.append(c.aux[1])
            else:
                aux_off.append(0)
                aux_n.append(0)
        d = PlanDescC()
        d.api_version = API_VERSION
        d.model_type = (1 if self.use_wide else 0) | (2 if self.use_deep else 0)
        d.n_cat_fields, d.n_dense_fields = len(self.cat_fields), len(self.dense_fields)
        d.cat_field_is_string = arr(self.cat_is_string, np.uint8)
        d.n_columns = len(C)
        d.col_kind = arr([c.kind for c in C], np.int32)
        d.col_field = arr([c.field for c in C], np.int32)
        d.col_buckets = arr([c.buckets for c in C], np.int64)
        d.col_aux_off, d.col_aux_n = arr(aux_off, np.int32), arr(aux_n, np.int32)
        d.col_norm_kind = arr([c.norm[0] for c in C], np.int32)
        d.col_norm_a = arr([c.norm[1] for c in C], np.float32)
        d.col_norm_b = arr([c.norm[2] for c in C], np.float32)
        d.col_wide_base = arr([c.wide_base for c in C], np.int64)
        d.col_emb_table = arr([c.emb_table for c in C], np.int32)
        d.col_ind_off = arr([c.ind_off for c in C], np.int32)
        d.vocab_fp, d.n_vocab_fp = arr(self._vocab_fp, np.uint64), len(self._vocab_fp)
        d.boundaries, d.n_boundaries = arr(self._bounds, np.float32), len(self._bounds)
        d.cross_key_type, d.cross_key_idx, d.n_cross_keys = arr(ck_type, np.int32), arr(ck_idx, np.int32), len(ck_type)
        d.n_tables = len(self.tables)
        d.table_rows = arr([t["rows"] for t in self.tables], np.int64)
        d.table_dim = arr([_pad(t["dim"], 4) for t in self.tables], np.int32)
        d.table_dim_logical = arr([t["dim"] for t in self.tables], np.int32)
        d.table_x0_off = arr([t["x0_off"] for t in self.tables], np.int32)
        d.n_numeric = len(self.numerics)
        d.num_field = arr([n["field"] for n in self.numerics], np.int32)
        d.num_norm_kind = arr([n["norm"][0] for n in self.numerics], np.int32)
        d.num_x0_off = arr([n["x0_off"] for n in self.numerics], np.int32)
        d.num_norm_a = arr([n["norm"][1] for n in self.numerics], np.float32)
        d.num_norm_b = arr([n["norm"][2] for n in self.numerics], np.float32)
        d.d0_phys, d.wide_rows = self.d0_phys, self.wide_rows
        d.n_towers = len(self.towers)
        d.tower_nlayers = arr([len(t["hidden"]) for t in self.towers], np.int32)
        d.tower_mode = arr([MODES.index(t["mode"]) for t in self.towers], np.int32)
        d.hidden_units = arr([h for t in self.towers for h in t["hidden"]], np.int32)
        d.activation, d.batch_norm = ACTS.index(self.activation), self.batch_norm
        for dst, o in ((d.lin_opt, self.lin_opt), (d.dnn_opt, self.dnn_opt)):
            dst.kind, dst.lr, dst.l1, dst.l2 = OPT[o["kind"]], o["lr"], o["l1"], o["l2"]
            dst.lr_power, dst.init_acc = o["lr_power"], o["init_acc"]
            dst.beta1, dst.beta2, dst.epsilon = o.get("beta1", 0.9), o.get("beta2", 0.999), o.get("epsilon", 1e-8)
            dst.rho, dst.momentum = o.get("rho", 0.9), o.get("momentum", 0.0)
        d.max_batch, d.max_nnz, d.max_keys, d.gemm_engine = self.max_batch, self.max_nnz, self.max_keys, GEMM[self.gemm_engine]
        d.dense_exchange_max_rows = self.dense_exchange_max_rows
        d.shard_world, d.shard_rank = self.shard_world, self.shard_rank
        d.table_sharded = arr([1 if t["sharded"] else 0 for t in self.tables], np.uint8)
        d.col_wide_sharded = arr([1 if x else 0 for x in self.wide_sharded], np.uint8)
        d.shard_capacity, d.shard_slack = self.shard_capacity, self.shard_slack
        d.dropout_rate, d.dropout_seed = self.dropout, self.dropout_seed
        d.wide_small_base = self.wide_small_base if self.wide_small_base is not None else self.wide_rows
        d.table_placement = arr([t["placement"] for t in self.tables], np.uint8)
        return d, keep


def compile_plan(config, model_type=None, max_batch=None, **kw):
    """Build a Plan from a ``wide_deep_b200.config.Config``."""
    mt = model_type or config.train["model_type"]
    mb = max_batch or config.train["batch_size"]
    return Plan(config.read_feature_conf(), config.read_cross_feature_conf(), config.model, mt, mb, **kw)
