"""Host side of multi-GPU evaluation and prediction: the line split that keeps the file's tail (input_fn(keep_tail=True)), the step
count and per-rank valid rows every rank derives on its own (shard_steps), the interleave back to file order, and the C-ABI."""
import os

import numpy as np
import pytest

from wide_deep_b200.dataset import input_fn, interleave_ranks, shard_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _row_ids(batch, F):
    """One value per row that identifies the line: label, dense values and categorical keys hashed together."""
    out = []
    for i in range(batch.batch_size):
        lo, hi = (int(batch.offsets[i * F]), int(batch.offsets[(i + 1) * F])) if batch.offsets is not None else (i * F, (i + 1) * F)
        parts = (batch.keys[lo:hi].tobytes(), batch.label[i].tobytes(), b"" if batch.dense is None else batch.dense[i].tobytes())
        out.append(hash(parts))
    return np.asarray(out, dtype=np.int64)


@pytest.mark.parametrize("path,batch_size", [("data/eval/eval1", 64), ("data/test/test2", 3), ("data/test", 100)])
@pytest.mark.parametrize("world", [2, 3, 4, 16])
def test_keep_tail_puts_every_line_on_one_rank_in_file_order(native_lib, path, batch_size, world):
    from wide_deep_b200.config import Config
    from wide_deep_b200.plan import compile_plan
    cfg = Config()
    plan = compile_plan(cfg, "wide_deep", batch_size)
    F = len(plan.cat_fields)
    full = np.concatenate([_row_ids(b, F) for b in input_fn(os.path.join(ROOT, path), None, "eval", batch_size, config=cfg, plan=plan)])
    parts = []
    for r in range(world):
        p = input_fn(os.path.join(ROOT, path), None, "eval", batch_size, config=cfg, plan=plan, rank=r, world=world, keep_tail=True)
        assert p.n_lines == len(full)
        sizes, ids = [], []
        for b in p:
            sizes.append(b.batch_size)
            ids.append(_row_ids(b, F))
        assert sizes == [v for v in p.n_valid if v > 0], (r, sizes, p.n_valid)
        assert len(p.n_valid) == p.steps
        parts.append(np.concatenate(ids) if ids else np.zeros(0, dtype=np.int64))
    assert sum(len(x) for x in parts) == len(full)
    assert np.array_equal(interleave_ranks(parts), full)
    # the default split still drops the lines beyond a multiple of `world` (training relies on equal shards)
    short = input_fn(os.path.join(ROOT, path), None, "eval", batch_size, config=cfg, plan=plan, rank=world - 1, world=world)
    assert sum(b.batch_size for b in short) == len(full) // world


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("batch_size", [1, 2, 5, 64])
def test_shard_steps_around_multiples_of_a_global_batch(world, batch_size):
    gb = world * batch_size
    for k in range(4):
        for n in sorted({max(k * gb + d, 0) for d in range(-world - 1, world + 2)}):
            steps, nv = shard_steps(n, world, batch_size)
            assert nv.shape == (world, steps)
            assert int(nv.sum()) == n
            assert steps == max(-(-len(range(r, n, world)) // batch_size) for r in range(world))
            for r in range(world):
                lines = len(range(r, n, world))
                exp = [min(batch_size, max(lines - s * batch_size, 0)) for s in range(steps)]
                assert nv[r].tolist() == exp, (n, r)
            if steps:
                assert nv[0, -1] > 0                      # no step in which every rank only serves


def test_interleave_ranks():
    parts = [np.array([0, 3, 6]), np.array([1, 4]), np.array([2, 5])]
    assert interleave_ranks(parts).tolist() == list(range(7))
    assert interleave_ranks([np.array([0.5], dtype=np.float32), np.zeros(0, dtype=np.float32)]).tolist() == [0.5]


def test_sharded_eval_symbols_resolve_from_the_header(native_lib):
    from tests.test_abi import header_symbols
    from wide_deep_b200 import _native
    new = ["wd_shard_eval_accumulate_slot", "wd_shard_eval_accumulate_phase", "wd_shard_eval_finish"]
    syms = header_symbols()
    for s in new:
        assert s in syms and s in _native.SYMBOLS, s
        assert getattr(native_lib, s).argtypes == _native.SYMBOLS[s][1]
