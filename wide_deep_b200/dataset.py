"""Input pipeline: TSV files -> CSR batches in pinned host memory.

Host-side mirror of ``input_fn`` / ``_CsvDataset`` (reference python/lib/dataset.py:62-195, 293-310): same
arguments (``csv_data_file`` may be a file or a directory, ``mode`` in {'train','eval','pred'}, ``batch_size``),
same parsing rules (TAB-separated, no quoting, NA token ``-`` -> per-type default, multi-valued string fields
split on ','), but the parser is the multi-threaded C++ loader in libwd_b200 (``wd_tsv_parse``): strings leave
it as Fingerprint64 values, so what crosses PCIe is the compact CSR the CUDA stage consumes.

Differences kept explicit:
  * shuffle: the reference shuffles with tf.data (buffer = num_examples, seed 123, dataset.py:180); that RNG
    stream cannot be reproduced outside TensorFlow, so 'train' mode shuffles whole files' lines with
    numpy's Philox(seed 123) instead — same intent (one seeded pass), different permutation;
  * distributed sharding: every ``world``-th line starting at ``rank`` (dataset.shard, dataset.py:173-174); training drops the
    last ``n_lines % world`` lines, evaluation and prediction keep them (``keep_tail``, ``shard_steps``).
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _native
from ._native import TsvSpecC
from .model import Batch


def list_files(path):
    """File or directory -> sorted list of data files, hidden files skipped (reference lib/utils/util.py:36-45,
    dataset.py:31-33)."""
    if not os.path.exists(path):
        raise AssertionError("data file: {} not found. Please check input data path".format(path))
    if os.path.isdir(path):
        return sorted(os.path.join(path, f) for f in os.listdir(path) if not f.startswith("."))
    return [path]


def _host_buffer(lib, pinned, nbytes, raw):
    """uint8 array of at least ``nbytes``: page-locked (its pointer appended to ``raw``, for wd_host_free) or, without a CUDA
    device, ordinary memory."""
    if not pinned:
        return np.zeros(max(nbytes, 8), dtype=np.uint8)
    p = ctypes.c_void_p()
    _native.check(lib.wd_host_alloc(max(nbytes, 8), ctypes.byref(p)))
    raw.append(p)
    return np.ctypeslib.as_array((ctypes.c_uint8 * max(nbytes, 8)).from_address(p.value))


class PinnedRing(object):
    """A ring of page-locked host buffer sets (one set = the arrays of one batch), allocated ONCE through the library
    (cudaHostAlloc).  The parser writes straight into a set and ``wd_batch_prefetch_slot`` copies from it asynchronously — the
    counterpart of the buffers ``dataset.prefetch`` owns in the reference's input_fn (python/lib/dataset.py:181-184).  A set is
    reused ``depth`` batches later, by which time the step that read its device copy has long been issued.  Without a CUDA
    device (CPU tests) the sets are ordinary numpy arrays."""

    def __init__(self, n_rows, n_cat_fields, n_dense_fields, key_cap, depth=4):
        self._lib = _native.lib()
        self.depth, self._i, self._raw = depth, 0, []
        self.n_rows, self.F, self.Nd, self.key_cap = n_rows, n_cat_fields, n_dense_fields, int(key_cap)
        self.pinned = self._lib.wd_device_count() > 0
        self.sets = [self._make_set() for _ in range(depth)]

    def _buf(self, nbytes):
        return _host_buffer(self._lib, self.pinned, nbytes, self._raw)

    def _make_set(self):
        n, F, Nd = self.n_rows, self.F, self.Nd
        return dict(offsets=self._buf((n * F + 1) * 4).view(np.int32), keys=self._buf(self.key_cap * 8).view(np.uint64),
                    dense=self._buf(n * max(Nd, 1) * 4).view(np.float32), label=self._buf(n * 4).view(np.float32),
                    weight=self._buf(n * 4).view(np.float32))

    def grow_keys(self, key_cap):
        """A batch needs more key room than the ring was sized for (long multi-valued rows): re-allocate every set's key buffer."""
        self.key_cap = int(key_cap)
        for s in self.sets:
            s["keys"] = self._buf(self.key_cap * 8).view(np.uint64)

    def next(self):
        s = self.sets[self._i % self.depth]
        self._i += 1
        return s

    def close(self):
        for p in self._raw:
            self._lib.wd_host_free(p)
        self._raw, self.sets = [], []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TsvTextBatch(object):
    """The text of one batch for the device parser (``WideDeepModel.parse_slot``): ``n`` lines in ``text`` (uint8, page-locked when a
    CUDA device is present), line i = ``text[starts[i]:starts[i + 1] - 1]``, and the parse spec of the reader that picked them.
    ``text`` and ``starts`` alias a ring set and stay valid for the next ``depth - 1`` batches of that ring."""

    def __init__(self, reader, text, starts, n):
        self.reader, self.text, self.starts, self.n = reader, text, starts, int(n)

    @property
    def batch_size(self):
        return self.n

    @property
    def has_label(self):
        return not self.reader.is_pred


class TextRing(object):
    """A ring of ``depth`` page-locked text buffers (plus line starts) for ``TsvTextBatch``: gathered lines land here so the device
    parser's host->device copy reads pinned memory.  A buffer that is too small for a batch is replaced by a larger one (the old
    one stays allocated until ``close``: a batch still in flight may alias it).  Without a CUDA device: numpy arrays."""

    def __init__(self, n_rows, text_cap, depth=6):
        self._lib = _native.lib()
        self.depth, self._i, self._raw = depth, 0, []
        self.pinned = self._lib.wd_device_count() > 0
        self.sets = [dict(text=self._buf(text_cap), starts=self._buf((n_rows + 1) * 8).view(np.int64)) for _ in range(depth)]

    def _buf(self, nbytes):
        return _host_buffer(self._lib, self.pinned, nbytes, self._raw)

    def next(self, text_bytes):
        s = self.sets[self._i % self.depth]
        self._i += 1
        if s["text"].size < text_bytes:
            s["text"] = self._buf(text_bytes + text_bytes // 4)
        return s

    def close(self):
        for p in self._raw:
            self._lib.wd_host_free(p)
        self._raw, self.sets = [], []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TsvReader(object):
    """Parses TSV text into ``Batch`` objects for a given Plan."""

    def __init__(self, config, plan, is_pred=False, n_threads=None):
        self.plan = plan
        schema = config.read_schema()
        fconf = config.read_feature_conf()
        train = config.train
        names = [schema[k] for k in sorted(schema)]
        if is_pred:
            names = [n for n in names if n != "clk"]
        cat_idx = {f: i for i, f in enumerate(plan.cat_fields)}
        dense_idx = {f: i for i, f in enumerate(plan.dense_fields)}
        role, target = [], []
        for n in names:
            if n == "clk":
                role.append(0); target.append(0)
            elif n in cat_idx:
                role.append(1 if plan.cat_is_string[cat_idx[n]] else 2); target.append(cat_idx[n])
            elif n in dense_idx:
                role.append(3); target.append(dense_idx[n])
            else:
                role.append(-1); target.append(0)          # unused schema column: parsed and discarded
        self._role = np.asarray(role, dtype=np.int32)
        self._target = np.asarray(target, dtype=np.int32)
        pos, neg = train.get("pos_sample_loss_weight"), train.get("neg_sample_loss_weight")
        self.use_weight = pos is not None and neg is not None      # dataset.py:70-72 (both must be set)
        spec = TsvSpecC()
        spec.n_columns = len(names)
        spec.col_role, spec.col_target = self._role.ctypes.data, self._target.ctypes.data
        spec.n_cat_fields, spec.n_dense_fields = len(plan.cat_fields), len(plan.dense_fields)
        spec.multivalue = 1 if train.get("multivalue") else 0
        spec.tf_compat_pad = 1 if plan.tf_compat_pad else 0
        spec.pos_weight, spec.neg_weight = float(pos or 1), float(neg or 1)
        spec.use_weight = 1 if self.use_weight else 0
        spec.has_label = 0 if is_pred else 1
        self._spec = spec
        self.is_pred = is_pred
        self.n_threads = n_threads or min(os.cpu_count() or 1, 16)
        self._lib = _native.lib()
        self._key_guess = 0                                           # keys of the largest batch seen (+25 %): first-call capacity

    def parse(self, lines, ring=None):
        """list of text lines (str or bytes, no trailing newline needed) -> Batch.  ``ring``: a PinnedRing whose next buffer set
        receives the batch (the returned Batch then aliases it and is valid until the ring comes round again)."""
        if lines and isinstance(lines[0], bytes):
            text = b"\n".join(lines)                                  # input_fn's path: no decode / encode round trip
        else:
            text = ("\n".join(l.rstrip("\n") for l in lines)).encode("utf-8")
        n = len(lines)
        F, Nd = len(self.plan.cat_fields), len(self.plan.dense_fields)
        if ring is not None:
            return self._parse_into_ring(text, n, ring)
        offsets = np.zeros(n * F + 1, dtype=np.int32)
        dense = np.zeros((n, max(Nd, 1)), dtype=np.float32)
        label = np.zeros(n, dtype=np.float32)
        weight = np.ones(n, dtype=np.float32)
        if self.plan.tf_compat_pad:
            # padded string fields (quirk Q2) can exceed the token count: ask for the size first (keys_cap = 0), then fill
            nnz = self._lib.wd_tsv_parse(ctypes.byref(self._spec), text, len(text), n, offsets.ctypes.data, None, 0,
                                         dense.ctypes.data, label.ctypes.data, weight.ctypes.data, self.n_threads)
            if nnz < 0:
                raise ValueError(self._lib.wd_last_error().decode())
            cap = max(nnz, 1)
        else:
            cap = n * max(F, 1) + text.count(b",") + 1               # every field holds at most (commas + 1) tokens
        keys = np.empty(cap, dtype=np.uint64)
        nnz = self._lib.wd_tsv_parse(ctypes.byref(self._spec), text, len(text), n, offsets.ctypes.data, keys.ctypes.data,
                                     keys.size, dense.ctypes.data, label.ctypes.data, weight.ctypes.data, self.n_threads)
        if nnz < 0:
            raise ValueError(self._lib.wd_last_error().decode())
        return Batch(n, keys[:nnz], offsets, dense[:, :Nd] if Nd else None, None if self.is_pred else label,
                     weight if (self.use_weight and not self.is_pred) else None)


def _parse_into_ring(self, text, n, ring, index=None):
    """``index`` = (starts, lens, idx): the batch's lines are picked out of the file image ``text`` (wd_tsv_parse_lines)."""
    F, Nd = len(self.plan.cat_fields), len(self.plan.dense_fields)
    if n > ring.n_rows:
        raise ValueError("batch of %d lines, pinned ring sized for %d" % (n, ring.n_rows))
    s = ring.next()                                                  # the oldest set: nothing in flight reads it any more

    def call():
        if index is None:
            return self._lib.wd_tsv_parse(ctypes.byref(self._spec), text, len(text), n, s["offsets"].ctypes.data, s["keys"].ctypes.data,
                                          ring.key_cap, s["dense"].ctypes.data, s["label"].ctypes.data, s["weight"].ctypes.data, self.n_threads)
        starts, lens, idx = index
        return self._lib.wd_tsv_parse_lines(ctypes.byref(self._spec), text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, n,
                                            s["offsets"].ctypes.data, s["keys"].ctypes.data, ring.key_cap, s["dense"].ctypes.data,
                                            s["label"].ctypes.data, s["weight"].ctypes.data, self.n_threads)

    nnz = call()
    if nnz > ring.key_cap:                                           # nothing was copied; the library keeps the parse for the next call
        ring.grow_keys(max(nnz, 2 * ring.key_cap))                   # (old key buffers stay allocated: in-flight batches alias them)
        nnz = call()
    if nnz < 0:
        raise ValueError(self._lib.wd_last_error().decode())
    b = Batch.__new__(Batch)                                         # views of the pinned set: no copies (Batch() would copy)
    b._ring = ring                                                   # the ring outlives every batch it holds (a prefetch queue may
    b.batch_size = n                                                 # still hold batches when the generator that owns it is done)
    b.keys, b.offsets = s["keys"][:nnz], s["offsets"][:n * F + 1]
    b.dense = s["dense"][:n * Nd].reshape(n, Nd) if Nd else None
    b.label = None if self.is_pred else s["label"][:n]
    b.weight = s["weight"][:n] if (self.use_weight and not self.is_pred) else None
    return b


def _parse_indexed(self, text, starts, lens, idx, ring=None):
    """Batch of the lines ``idx`` of the file image ``text`` (``starts`` / ``lens`` from wd_tsv_index_lines): no line is split off,
    copied or joined on the way to the parser."""
    n = len(idx)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    if ring is not None:
        return self._parse_into_ring(text, n, ring, index=(starts, lens, idx))
    F, Nd = len(self.plan.cat_fields), len(self.plan.dense_fields)
    offsets = np.zeros(n * F + 1, dtype=np.int32)
    dense = np.zeros((n, max(Nd, 1)), dtype=np.float32)
    label = np.zeros(n, dtype=np.float32)
    weight = np.ones(n, dtype=np.float32)
    keys = np.empty(max(self._key_guess, n * max(F, 1)), dtype=np.uint64)
    for _ in range(2):                                               # second round only if the guess was too small (parse is reused)
        nnz = self._lib.wd_tsv_parse_lines(ctypes.byref(self._spec), text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, n,
                                           offsets.ctypes.data, keys.ctypes.data, keys.size, dense.ctypes.data, label.ctypes.data,
                                           weight.ctypes.data, self.n_threads)
        if nnz < 0:
            raise ValueError(self._lib.wd_last_error().decode())
        if nnz <= keys.size:
            break
        keys = np.empty(nnz, dtype=np.uint64)
    self._key_guess = max(self._key_guess, int(nnz * 1.25) + 16)
    return Batch(n, keys[:nnz], offsets, dense[:, :Nd] if Nd else None, None if self.is_pred else label,
                 weight if (self.use_weight and not self.is_pred) else None)


def _gather_text(self, text, starts, lens, idx, ring):
    """TsvTextBatch of the lines ``idx`` of the file image ``text``: one copy of the lines into the ring's next buffer."""
    n = len(idx)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    nbytes = int(lens[idx].sum()) + n
    s = ring.next(nbytes)
    out_starts = s["starts"][:n + 1]
    got = self._lib.wd_tsv_gather_lines(text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, n, s["text"].ctypes.data,
                                        s["text"].size, out_starts.ctypes.data, self.n_threads)
    if got < 0 or got != nbytes:
        raise ValueError(self._lib.wd_last_error().decode() if got < 0 else "wd_tsv_gather_lines: %d bytes, %d expected" % (got, nbytes))
    tb = TsvTextBatch(self, s["text"], out_starts, n)
    tb._ring = ring                                                  # (as in _parse_into_ring: the buffers live while the batch does)
    return tb


TsvReader._parse_into_ring = _parse_into_ring
TsvReader.gather_text = _gather_text
TsvReader.parse_indexed = _parse_indexed


class Prefetcher(object):
    """Runs a batch generator on a background thread, ``depth`` batches ahead of the consumer: parsing (C++ worker threads, GIL
    released) overlaps the consumer's Python and the GPU step — tf.data's prefetch thread in the reference's input_fn."""

    def __init__(self, gen, depth=2):
        import queue
        import threading
        self._q = queue.Queue(maxsize=depth)
        self._done = object()
        self._err = None

        def run():
            try:
                for item in gen:
                    self._q.put(item)
            except BaseException as e:          # surfaced on the consumer's thread
                self._err = e
            self._q.put(self._done)

        self._t = threading.Thread(target=run, daemon=True)
        self._t.start()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if item is self._done:
            if self._err is not None:
                raise self._err
            raise StopIteration
        return item


def shard_steps(n_lines, world, batch_size):
    """A file of ``n_lines`` lines split over ``world`` ranks with its tail kept (rank r: lines r, r + world, ...) and batched per
    rank -> (steps, n_valid): the number of collective steps every rank runs, and n_valid[r][s], the lines rank r holds in step
    s (0: the rank has run out and only serves its peers).  Every rank computes the same, without communicating."""
    per = np.array([len(range(r, n_lines, world)) for r in range(world)], dtype=np.int64)
    steps = -(-int(per[0]) // batch_size)                         # rank 0 holds the most lines
    n_valid = np.clip(per[:, None] - np.arange(steps, dtype=np.int64)[None, :] * batch_size, 0, batch_size)
    return steps, n_valid


def interleave_ranks(parts):
    """Inverse of the line split: ``parts[r]`` holds a value per line of rank r -> one array in file order (line i of the file is
    line i // G of rank i % G)."""
    G = len(parts)
    out = np.empty(sum(len(p) for p in parts), dtype=np.result_type(*parts))
    for r, p in enumerate(parts):
        out[r::G] = p
    return out


class ShardPass(object):
    """One rank's pass over its lines of a file split over ``world`` ranks with the tail kept (``input_fn(keep_tail=True)``): iterates
    the rank's batches; ``steps`` and ``n_valid`` (this rank's lines per step) come from ``shard_steps``."""

    def __init__(self, batches, n_lines, rank, world, batch_size):
        self._batches = batches
        self.n_lines = n_lines
        self.steps, n_valid = shard_steps(n_lines, world, batch_size)
        self.n_valid = [int(v) for v in n_valid[rank]]

    def __iter__(self):
        return self._batches


def input_fn(csv_data_file, img_data_file, mode, batch_size, config=None, plan=None, rank=0, world=1, seed=123, pinned=False,
             device_parse=False, keep_tail=False):
    """Iterator of ``Batch`` for one pass over the data (one epoch), mirroring the reference's
    ``input_fn(csv_data_file, img_data_file, mode, batch_size)`` (dataset.py:293-310).  ``img_data_file`` is
    accepted for signature compatibility and must be None (the CNN branch is out of scope).
    The files are read and the pinned ring is allocated HERE (on the caller's thread, whose CUDA device is the model's); only
    the per-batch parsing is lazy, so the returned iterator may be drained from a prefetch thread.
    ``device_parse=True``: the same lines, in the same batches, are yielded as ``TsvTextBatch`` (the batch's text gathered into a
    ring of page-locked buffers) for ``WideDeepModel.parse_slot``, which parses them on the GPU; ``pinned`` is then irrelevant.
    ``keep_tail=True`` (evaluation and prediction with ``world > 1``): rank r gets every line r, r + world, ... to the end of the
    file, and the result is a ``ShardPass``, which also tells how many steps every rank runs and how many lines rank r holds in
    each."""
    assert mode in ("train", "eval", "pred"), "mode must in `train`, `eval`, or `pred`, found {}".format(mode)
    if img_data_file:
        raise ValueError("image inputs are not supported by this library (cnn_use_flag: 0)")
    reader = TsvReader(config, plan, is_pred=(mode == "pred"))
    lib = _native.lib()
    # one image of all files + an index of its non-empty lines (wd_tsv_index_lines): sharding and shuffling permute INDICES, the
    # parser reads each batch's lines in place (wd_tsv_parse_lines) — no per-line Python objects, no per-batch join
    parts = []
    for f in list_files(csv_data_file):
        with open(f, "rb") as fh:
            parts.append(fh.read())
    text = parts[0] if len(parts) == 1 else b"\n".join(parts)
    del parts
    n_all = lib.wd_tsv_index_lines(text, len(text), None, None, 0)
    if n_all < 0:
        raise ValueError(lib.wd_last_error().decode())
    starts, lens = np.empty(max(n_all, 1), dtype=np.int64), np.empty(max(n_all, 1), dtype=np.int32)
    lib.wd_tsv_index_lines(text, len(text), starts.ctypes.data, lens.ctypes.data, n_all)
    order = np.arange(n_all, dtype=np.int64)
    if world > 1:
        # dataset.shard(num_workers, worker_index) (reference dataset.py:173-174): every world-th line.  Synchronous training
        # needs the same number of batches on every rank, so the few lines beyond a multiple of `world` are dropped; with the
        # tail kept, ranks that run out enter the remaining steps without rows (ShardPass.n_valid)
        order = order[rank::world]
        if not keep_tail:
            order = order[:n_all // world]
    if mode == "train":
        perm = np.random.Generator(np.random.Philox(seed)).permutation(len(order))
        order = order[perm]
    order = np.ascontiguousarray(order)
    if device_parse:
        mean_len = float(lens[:n_all].mean()) if n_all else 0.0
        tring = TextRing(batch_size, int(batch_size * (mean_len + 1) * 1.25) + 4096)

        def texts():
            for i in range(0, len(order), batch_size):
                yield reader.gather_text(text, starts, lens, order[i:i + batch_size], tring)

        return ShardPass(texts(), n_all, rank, world, batch_size) if keep_tail else texts()
    # pinned=True (estimator.train, which consumes batch by batch): parse into a ring of page-locked buffers so the host->device
    # refill of a batch slot is truly asynchronous; a yielded Batch stays valid for the next `depth - 1` batches
    ring = None
    if pinned:
        F, Nd = len(plan.cat_fields), len(plan.dense_fields)
        ring = PinnedRing(batch_size, F, Nd, key_cap=batch_size * max(F, 1) * 4, depth=6)

    def batches():
        for i in range(0, len(order), batch_size):
            yield reader.parse_indexed(text, starts, lens, order[i:i + batch_size], ring=ring)

    return ShardPass(batches(), n_all, rank, world, batch_size) if keep_tail else batches()
