"""Float64 reference of one train step of a row-sharded group of G ranks, from the ranks' own values, and an fp32 emulation of the
exchange for the CPU suite.

Reference (``GroupStepRef``): kernel_ref.StepRef on the concatenated batch.  Rank r's deep input, hidden outputs, column ids,
labels and weights are stacked at example offset B_0 + ... + B_(r-1); the parameters are the ones uploaded.  Every gradient then
follows StepRef's formulas, with two differences:

* A dense or replicated gradient is the sum of G per-rank partials, each a reduction over B_r rows, added in rank order by the
  two-shot all-reduce (csrc/shard.cu shard_ar_reduce_kernel).  Each add errs by at most u times the sum of |partials| <= M, so
  criterion 1's constant C * M grows by (G - 1) u M.  Criterion 2 is unchanged.
* A sharded embedding row's gradient is the sum over every occurrence on every rank of dX0[example, slice] * fl(1 / n_bag), the
  bag scale the requester stored; a sharded wide row sums dlogit the same way.  Rows no rank touched come back unchanged.

Dropout: rank r draws the keep mask of its row m at global row r * max_batch + m (csrc/gemm.cuh DropArgs::row0), so the reference
regenerates it there, at every batch size.  When every rank's batch is full, that is the mask one GPU draws on the concatenated
batch.

Emulation (``owner_sums``, ``all_reduce``, ``untouched_moves``): the owner's per-row sums in its order (occurrences sorted by
(row, tag), tag = source rank << 27 | bag; rows with at most kChunk = 16 occurrences summed directly, hotter rows in chunks of 16
combined in chunk order), the two-shot all-reduce with its ceil(n4 / G) float4 slices, and the Adam pass over each owner's
local rows.  ``DEFECTS`` plants one fault each; the CPU suite holds the checks to pass the healthy emulation and to fail every
defect.
"""
import numpy as np

from oracle.model import drop_keep
from tests import kernel_ref as KR

U = KR.U
K_CHUNK = 16
TAG_BAG_BITS = 27
DEFECTS = ("ar_drop_rank", "ar_drop_last_slice", "ar_shift_last_slice", "own_bag_scale", "pull_rank0", "local_row_mod",
           "drop_chunk", "untouched_none", "untouched_twice", "local_row_mask")


def f32_recip(n):
    """fl(1 / n) of the requester's bag scale (shard_send_kernel: 1.f / (float)count)."""
    return (np.float32(1) / np.asarray(n, dtype=np.float32)).astype(np.float64)


def group_keep(seed, step, layer_id, row0s, Bs, width, rate, local=False):
    """Keep mask [sum Bs, width] of one layer over the ranks' concatenated rows: rank r's row m at global row row0s[r] + m (local:
    at row m, the planted defect of a mask drawn from the local row)."""
    parts = []
    for r0, b in zip(row0s, Bs):
        r0 = 0 if local else r0
        parts.append(drop_keep(seed, step, layer_id, r0 + b, width, rate)[r0:])
    return np.concatenate(parts, axis=0)


# ------------------------------------------------------------------------------------------------ the float64 reference
def group_column_ids(models, Bs):
    """CSR (offsets [sum Bs * C + 1], ids) of the ranks' last batches, concatenated in rank order (the global batch's ids)."""
    offs, ids, base = [], [], 0
    for m, b in zip(models, Bs):
        m._rows_hint = b
        o, i = m.column_ids()
        assert o[0] == 0 and o[-1] == len(i), (o[0], o[-1], len(i))
        offs.append(o[:-1].astype(np.int64) + base)
        ids.append(i)
        base += len(i)
    return np.concatenate(offs + [np.array([base], dtype=np.int64)]), np.concatenate(ids)


class GroupStepRef(KR.StepRef):
    """StepRef of one step of G ranks: models[r] is rank r after the step, batches[r] its batch, params the global fp32
    parameters uploaded before it, step the dropout counter (train steps before it)."""

    def __init__(self, models, batches, params, engine, step=None):
        plan = models[0].plan
        self.plan, self.engine, self.params = plan, engine, {k: np.asarray(v, dtype=np.float64) for k, v in params.items()}
        self.G = len(models)
        self.Bs = [b.batch_size for b in batches]
        self.B = sum(self.Bs)
        self.row0s = [r * plan.max_batch for r in range(self.G)]
        if plan.use_deep:
            parts = [KR.gpu_forward_values(m, b) for m, b in zip(models, self.Bs)]
            self.X0p = np.concatenate([p[0] for p in parts], axis=0)
            self.H = [[np.concatenate([p[1][t][l] for p in parts], axis=0) for l in range(len(tw["hidden"]))]
                      for t, tw in enumerate(plan.towers)]
            self.X0 = KR.x0_logical(plan, self.X0p)
        else:
            self.X0p, self.H, self.X0 = None, [], None
        self.offs, self.ids = group_column_ids(models, self.Bs)
        self.label = np.concatenate([b.label for b in batches]).astype(np.float64)
        self.weight = np.concatenate([np.ones(b.batch_size) if b.weight is None else b.weight.astype(np.float64) for b in batches])
        self.act, self.bn = plan.activation, plan.batch_norm
        self.rate = plan.dropout if step is not None else 0.0
        self.step = step

    def _bag_scale(self, cnt):
        return f32_recip(np.maximum(cnt, 1))

    def _keep(self, t, l, width):
        if self.rate <= 0:
            return None
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(self.rate)))
        return group_keep(self.plan.dropout_seed, self.step, t * 64 + l, self.row0s, self.Bs, width, self.rate).astype(np.float64) * scale

    def gradients(self):
        ref, M, R, C = super(GroupStepRef, self).gradients()
        for name in C:
            if not self.plan.is_sharded_tensor(name):        # G partials added in rank order
                C[name] = C[name] + (self.G - 1) * U
        return ref, M, R, C


# ------------------------------------------------------------------------------------------------ fp32 emulation of the exchange
def owner_sums(rows, ranks, bags, grad, scale, G, n_rows, defect=None):
    """Per owner, the fp32 gradient sums of its local rows [ceil(n_rows / G), dim] (zero where untouched), and the float64
    reference and magnitude of the global rows [n_rows, dim].

    Occurrence k is global row rows[k] of example bags[k] on rank ranks[k], in the requester's order.  grad[r]: rank r's
    gradient rows [max_batch, dim] (dX0 slice / dlogit), scale[r]: its bag scales [max_batch] (fp32; 1 for wide rows)."""
    dim = grad[0].shape[1]
    rows, ranks, bags = (np.asarray(a, dtype=np.int64) for a in (rows, ranks, bags))
    local_n = (n_rows + G - 1) // G
    out = [np.zeros((local_n, dim), dtype=np.float32) for _ in range(G)]
    ref, mag = np.zeros((n_rows, dim)), np.zeros((n_rows, dim))
    for k in range(len(rows)):
        v = grad[ranks[k]][bags[k]].astype(np.float64) * float(scale[ranks[k]][bags[k]])
        ref[rows[k]] += v
        mag[rows[k]] += np.abs(v)
    order = np.lexsort((ranks << TAG_BAG_BITS | bags, rows))        # (row, tag): what the flatten + stable sort by row gives
    for o in range(G):
        mine = order[rows[order] % G == o]
        for row in np.unique(rows[mine]):
            occ = mine[rows[mine] == row]
            chunks = [occ] if len(occ) <= K_CHUNK else [occ[i:i + K_CHUNK] for i in range(0, len(occ), K_CHUNK)]
            if defect == "drop_chunk" and len(chunks) > 1:
                chunks = chunks[:-1]
            total = np.zeros(dim, dtype=np.float32)
            for ch in chunks:
                acc = np.zeros(dim, dtype=np.float32)
                for k in ch:
                    src = 0 if defect == "pull_rank0" else ranks[k]
                    sc = scale[o if defect == "own_bag_scale" else src][bags[k]]
                    acc = acc + grad[src][bags[k]] * np.float32(sc)
                total = total + acc
            out[o][row % G if defect == "local_row_mod" else row // G] = total
    return out, ref, mag


def interleave(shards, n_rows):
    """The global tensor from the owners' local rows: row r is rank r mod G's local row r // G (LocalShardGroup.get_tensor)."""
    G = len(shards)
    full = np.zeros((n_rows,) + shards[0].shape[1:], dtype=shards[0].dtype)
    for r in range(G):
        full[r::G] = shards[r][:len(range(r, n_rows, G))]
    return full


def all_reduce(arenas, defect=None):
    """Two-shot all-reduce of the ranks' fp32 arenas (length a multiple of 4): rank `me` sums float4s [me * slice4, (me + 1) *
    slice4) of every arena in rank order, slice4 = ceil(n4 / G), then every rank copies every slice.  -> every rank's result."""
    G = len(arenas)
    n4 = arenas[0].size // 4
    slice4 = (n4 + G - 1) // G
    last = max(o for o in range(G) if o * slice4 < n4) if n4 else 0
    red = [np.zeros_like(a) for a in arenas]
    for me in range(G):
        lo, hi = me * slice4, min(n4, (me + 1) * slice4)
        if defect == "ar_shift_last_slice" and me == last:
            lo += 1
        if lo >= hi:
            continue
        acc = arenas[0][4 * lo:4 * hi].copy()
        for r in range(1, G):
            if defect == "ar_drop_rank" and r == G - 1:
                continue
            acc = acc + arenas[r][4 * lo:4 * hi]
        red[me][4 * lo:4 * hi] = acc
    outs = []
    for me in range(G):
        out = arenas[me].copy()                      # the gather overwrites the rank's own partials
        for i in range(n4):
            owner = i // slice4
            if defect == "ar_drop_last_slice" and owner == last:
                continue
            out[4 * i:4 * i + 4] = red[owner][4 * i:4 * i + 4]
        outs.append(out)
    return outs


def untouched_moves(n_rows, G, touched, defect=None):
    """How many times the Adam untouched pass moves each global row: owner o walks its local rows j < ceil(n_rows / G), global
    row j * G + o, and moves the rows no gradient touched."""
    local_n = n_rows // G if defect == "untouched_none" else (n_rows + G - 1) // G
    count = np.zeros(n_rows, dtype=np.int64)
    for o in range(G):
        for j in range(local_n):
            cover = [j * G + o] + ([j * G] if defect == "untouched_twice" and o == G - 1 else [])
            for r in cover:
                if r < n_rows and not touched[r]:
                    count[r] += 1
    return count
