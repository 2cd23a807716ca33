"""The sharded checkpoint layout: every rank writes the rows it holds, in bounded chunks, and any number of ranks restores them.

A checkpoint ``model.ckpt-<step>/`` is a directory of ``.npy`` files, one per (tensor, slot, writer rank), and ``manifest.json``:

  global_step   the step the checkpoint was taken at
  world         G, the number of ranks that wrote it
  tensors       TensorFlow variable name -> shape (global), slots (optimizer slots besides the value), sharded, files
                (files[slot] lists the slot's parts).  sharded: G parts, global row g in part g mod G at row g // G (the rows rank
                g mod G holds); else one part of the global shape, written by rank 0.

Rows of embedding tables and wide columns move through ``WideDeepModel.get_rows`` / ``set_rows`` in chunks of at most
``CHUNK_BYTES``; the dense tensors are small and move whole.  So a save holds one chunk of host memory at a time besides the dense
tensors, and a restore reads, chunk by chunk from memory-mapped parts, only the rows its rank holds: global rows g with
g mod G' = r' on rank r' of G' for a row-sharded tensor, every row for a replicated one.  The writer's and the reader's "whole or
sharded" may differ either way; they do whenever G changes, since whether a table is sharded depends on the GPU count.

Commit: every rank writes into ``model.ckpt-<step>.tmp/`` and fsyncs its files; after one barrier rank 0 writes the manifest and
renames the directory.  A directory without a manifest is never listed, so a crashed save leaves nothing a restore would pick.

This module also holds the flat layout, one ``model.ckpt-<step>.npz`` of every global tensor written by rank 0 (``save_npz`` /
``restore_npz``), and lists and rotates the checkpoints of a model directory in either layout: the newest step wins.
"""
from __future__ import annotations

import json
import math
import os
import shutil
from collections import OrderedDict

import numpy as np

from .plan import T_EMB_TABLE, T_WIDE_COL

PREFIX = "model.ckpt-"
MANIFEST = "manifest.json"
FORMAT = "wide_deep_b200.sharded/1"
CHUNK_BYTES = 64 << 20          # host bytes of rows one get_rows / set_rows call moves at most


# ------------------------------------------------------------------------------------------------------------ listing
def list_checkpoints(model_dir):
    """[(step, path)] of the complete checkpoints in model_dir, oldest first: ``model.ckpt-<step>.npz`` files and
    ``model.ckpt-<step>/`` directories that hold a manifest (``.tmp`` directories and directories without one are skipped)."""
    if not os.path.isdir(model_dir):
        return []
    found = []
    for f in os.listdir(model_dir):
        if not f.startswith(PREFIX):
            continue
        stem, p = f[len(PREFIX):], os.path.join(model_dir, f)
        if stem.endswith(".npz") and stem[:-4].isdigit() and os.path.isfile(p):
            found.append((int(stem[:-4]), 0, p))
        elif stem.isdigit() and os.path.isfile(os.path.join(p, MANIFEST)):
            found.append((int(stem), 1, p))
    return [(step, p) for step, _, p in sorted(found)]


def rotate(model_dir, keep):
    """Removes every checkpoint of model_dir but the newest `keep` (either layout)."""
    for _, p in list_checkpoints(model_dir)[:-keep]:
        if os.path.isdir(p):
            shutil.rmtree(p)
        else:
            os.remove(p)


# ------------------------------------------------------------------------------------------------------------ .npz layout
def save_npz(model_dir, m, get=None, write=True):
    """Flat ``model_dir/model.ckpt-<global step>.npz`` of model `m`: every tensor and optimizer slot, each the global tensor
    `get(name, slot)` returns (default m.get_tensor; a row-sharded model passes its collective gather, and every rank calls this
    while only the one with `write` writes).  Returns the file, or None where nothing was written."""
    get = get or m.get_tensor
    blob = {"global_step": np.asarray(m.global_step)}
    for name in m.tensor_names():
        blob[name] = get(name)
        for s in range(m.n_slots(name)):
            blob["%s/slot%d" % (name, s + 1)] = get(name, slot=s + 1)
    if not write:
        return None
    os.makedirs(model_dir, exist_ok=True)
    path = os.path.join(model_dir, "%s%d.npz" % (PREFIX, m.global_step))
    tmp = path + ".tmp.%d" % os.getpid()                 # written beside, then renamed: a crash never leaves a truncated
    with open(tmp, "wb") as fh:                          # checkpoint that list_checkpoints() would pick up
        np.savez(fh, **blob)
        fh.flush()
        os.fsync(fh.fileno())
    os.replace(tmp, path)
    return path


def restore_npz(path, m):
    """Every tensor of model `m` from the .npz file `path` (a row-sharded rank keeps its own rows of each global tensor)."""
    with np.load(path) as z:
        have = set(z.files)
        want = []
        for name in m.tensor_names():
            want.append((name, 0, tuple(m.plan.tensor_names[name][3])))
            for s in range(m.n_slots(name)):
                want.append(("%s/slot%d" % (name, s + 1), s + 1, tuple(m.plan.tensor_names[name][3])))
        missing = [k for k, _, _ in want if k not in have]
        if missing or "global_step" not in have:
            raise ValueError("checkpoint {} does not match this model (feature conf, model_type or optimizers changed?): "
                             "missing {} of {} tensors, e.g. {}".format(path, len(missing), len(want), missing[:3]))
        for key, slot, shape in want:
            if tuple(z[key].shape) != shape:
                raise ValueError("checkpoint {}: tensor {} has shape {}, the model expects {}".format(path, key, tuple(z[key].shape), shape))
        m.global_step = int(z["global_step"])
        m.set_opt_step(m.global_step)
        for key, slot, _ in want:
            m.set_tensor(key if slot == 0 else key[:key.rindex("/slot")], z[key], slot=slot)


# ------------------------------------------------------------------------------------------------------------ layout
def _is_rows(plan, name):
    return plan.tensor_names[name][0] in (T_EMB_TABLE, T_WIDE_COL)


def _chunk_rows(shape):
    return max(1, CHUNK_BYTES // (4 * int(np.prod(shape[1:], dtype=np.int64))))


def _part_name(i, name, slot, part=None, world=None):
    base = "%04d.%s.slot%d" % (i, name.replace("/", "."), slot)
    return base + (".npy" if part is None else ".part%d-of-%d.npy" % (part, world))


def _fsync(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _entries(m):
    """Manifest entries of the tensors of model `m` as its G = plan.shard_world ranks store them."""
    plan = m.plan
    G = plan.shard_world
    out = OrderedDict()
    for i, name in enumerate(plan.tensor_names):
        sharded = plan.is_sharded_tensor(name)
        slots = m.n_slots(name)
        files = [[_part_name(i, name, s, r, G) for r in range(G)] if sharded else [_part_name(i, name, s)] for s in range(1 + slots)]
        out[name] = {"shape": list(plan.tensor_names[name][3]), "slots": slots, "sharded": sharded, "files": files}
    return out


def _write_part(m, name, slot, path):
    shape = tuple(m.plan.local_shape(name))
    out = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=shape)
    if _is_rows(m.plan, name):
        step = _chunk_rows(shape)
        for r0 in range(0, shape[0], step):
            n = min(step, shape[0] - r0)
            out[r0:r0 + n] = m.get_rows(name, r0, n, slot)
    else:
        out[...] = m.get_tensor(name, slot)
    out.flush()
    del out
    _fsync(path)


# ------------------------------------------------------------------------------------------------------------ save
def save(model_dir, models, barrier=None):
    """Writes ``model_dir/model.ckpt-<global step>/`` from `models`, the ranks of one model this process drives: all G of them
    (LocalShardGroup; one GPU is G = 1), or one rank of a torchrun job with `barrier` the job's barrier.  A collective: every rank
    calls it at the same step.  Returns the directory in the process that holds rank 0, else None.  The other ranks return before
    rank 0 has committed: a second save at the same step could have a fast rank write into the .tmp directory rank 0 is still
    renaming, so a caller does not repeat a save while the step has not moved (WideAndDeepClassifier.save skips it)."""
    plan = models[0].plan
    step = int(models[0].global_step)
    final = os.path.join(model_dir, "%s%d" % (PREFIX, step))
    tmp = final + ".tmp"
    os.makedirs(tmp, exist_ok=True)
    entries = _entries(models[0])
    for m in models:
        r = m.plan.shard_rank
        for name, e in entries.items():
            for slot, files in enumerate(e["files"]):
                if e["sharded"]:
                    _write_part(m, name, slot, os.path.join(tmp, files[r]))
                elif r == 0:
                    _write_part(m, name, slot, os.path.join(tmp, files[0]))
    if barrier is not None:
        barrier()                                     # every rank's parts are on disk
    if all(m.plan.shard_rank != 0 for m in models):
        return None
    keep = {f for e in entries.values() for files in e["files"] for f in files}
    for f in os.listdir(tmp):                         # parts an earlier, crashed save of this step left behind
        if f not in keep:
            os.remove(os.path.join(tmp, f))
    manifest = {"format": FORMAT, "global_step": step, "world": plan.shard_world, "tensors": entries}
    with open(os.path.join(tmp, MANIFEST), "w") as fh:
        json.dump(manifest, fh, indent=1)
        fh.flush()
        os.fsync(fh.fileno())
    _fsync(tmp)
    if os.path.isdir(final):                          # the same step saved again
        shutil.rmtree(final)
    os.replace(tmp, final)
    _fsync(model_dir)
    return final


# ------------------------------------------------------------------------------------------------------------ restore
def read_manifest(path):
    """The manifest of sharded checkpoint `path`, checked for structure; ValueError when it is missing or malformed."""
    try:
        with open(os.path.join(path, MANIFEST)) as fh:
            man = json.load(fh)
    except (OSError, ValueError) as e:
        raise ValueError("checkpoint {}: no readable {} ({})".format(path, MANIFEST, e))
    try:
        if man["format"] != FORMAT:
            raise ValueError("format {!r}, expected {!r}".format(man["format"], FORMAT))
        G, step = man["world"], man["global_step"]
        if not (isinstance(G, int) and G >= 1 and isinstance(step, int) and step >= 0):
            raise ValueError("world {!r}, global_step {!r}".format(G, step))
        for name, e in man["tensors"].items():
            shape, slots, files = e["shape"], e["slots"], e["files"]
            if not (isinstance(shape, list) and shape and all(isinstance(d, int) and d >= 0 for d in shape)):
                raise ValueError("tensor {}: shape {!r}".format(name, shape))
            if not (isinstance(slots, int) and slots >= 0 and isinstance(files, list) and len(files) == 1 + slots):
                raise ValueError("tensor {}: {!r} slots, {!r} file lists".format(name, slots, files))
            for fs in files:
                if not (isinstance(fs, list) and len(fs) == (G if e["sharded"] else 1)
                        and all(isinstance(f, str) and os.path.basename(f) == f and f for f in fs)):
                    raise ValueError("tensor {}: parts {!r} (sharded {!r}, world {})".format(name, fs, e["sharded"], G))
    except (KeyError, TypeError, AttributeError) as e:
        raise ValueError("checkpoint {}: malformed {} ({!r})".format(path, MANIFEST, e))
    except ValueError as e:
        raise ValueError("checkpoint {}: malformed {}: {}".format(path, MANIFEST, e))
    return man


def _open_parts(path, name, e, slot, G):
    """Memory maps of the parts of one slot, each checked against the rows the manifest says it holds."""
    shape = tuple(e["shape"])
    parts = []
    for r, f in enumerate(e["files"][slot]):
        want = ((shape[0] - r + G - 1) // G,) + shape[1:] if e["sharded"] else shape
        try:
            a = np.load(os.path.join(path, f), mmap_mode="r")
        except (OSError, ValueError) as err:
            raise ValueError("checkpoint {}: part {} of tensor {} is unreadable ({})".format(path, f, name, err))
        if a.shape != want or a.dtype != np.float32:
            raise ValueError("checkpoint {}: part {} of tensor {} is {} {}, the manifest implies float32 {}".format(
                path, f, name, a.dtype, a.shape, want))
        parts.append(a)
    return parts


def _read_rows(m, name, slot, parts, S):
    """Rows of `name` this rank holds, from `parts` (S parts: global row g in part g mod S at row g // S), chunk by chunk.  Local
    row j of the target is global row o + T j; within a chunk, every P-th local row (P = S / gcd(S, T)) comes from the same part,
    at rows that step by T P / S there, so each part is read with one strided slice per chunk."""
    plan = m.plan
    R = plan.tensor_names[name][3][0]
    T, o = (plan.shard_world, plan.shard_rank) if plan.is_sharded_tensor(name) else (1, 0)
    n = len(range(o, R, T))
    P = S // math.gcd(S, T)
    d = T * P // S
    step = _chunk_rows(plan.tensor_names[name][3])
    for j0 in range(0, n, step):
        j1 = min(n, j0 + step)
        buf = np.empty((j1 - j0,) + parts[0].shape[1:], dtype=np.float32)
        for k in range(min(P, j1 - j0)):
            g0 = o + T * (j0 + k)
            cnt = len(range(j0 + k, j1, P))
            a = g0 // S
            buf[k::P] = parts[g0 % S][a:a + d * (cnt - 1) + 1:d]
        m.set_rows(name, j0, buf, slot)
        del buf                                       # before the next chunk's buffer: one chunk of host memory at a time


def restore(path, models):
    """Restores sharded checkpoint `path` into `models` (the ranks this process drives, as for `save`), whatever G wrote it.
    Checks everything before it writes anything; ValueError (restore's messages for the .npz layout) when the checkpoint does not
    match the model.  Returns the global step."""
    man = read_manifest(path)
    plan, G, have = models[0].plan, man["world"], man["tensors"]
    want = []
    for name in plan.tensor_names:
        want.append((name, 0))
        want.extend((name, s + 1) for s in range(models[0].n_slots(name)))
    missing = [name if s == 0 else "%s/slot%d" % (name, s) for name, s in want if name not in have or s > have[name]["slots"]]
    if missing:
        raise ValueError("checkpoint {} does not match this model (feature conf, model_type or optimizers changed?): "
                         "missing {} of {} tensors, e.g. {}".format(path, len(missing), len(want), missing[:3]))
    for name, s in want:
        key = name if s == 0 else "%s/slot%d" % (name, s)
        shape = tuple(plan.tensor_names[name][3])
        if tuple(have[name]["shape"]) != shape:
            raise ValueError("checkpoint {}: tensor {} has shape {}, the model expects {}".format(path, key, tuple(have[name]["shape"]), shape))
        if have[name]["sharded"] and not _is_rows(plan, name):
            raise ValueError("checkpoint {}: tensor {} is stored in row shards, the model holds it whole".format(path, key))
        _open_parts(path, name, have[name], s, G)
    step = int(man["global_step"])
    for m in models:
        m.global_step = step
        m.set_opt_step(step)                          # first: writes to deferred Adam tables stamp their rows with this step
        for name, s in want:
            e = have[name]
            parts = _open_parts(path, name, e, s, G)
            if _is_rows(plan, name):
                _read_rows(m, name, s, parts, G if e["sharded"] else 1)
            else:
                m.set_tensor(name, np.asarray(parts[0]), s)
            del parts
    return step
