"""A model owns every device resource it creates, the lazily created ones included (batch slots, their upload events, the device
TSV parser, the host-table cache, the layer-summary buffers, the profiling marks).  So a model built with the same plan after the
first one was destroyed allocates the same HBM and trains to the same bytes, and enabling the cache adds exactly its slots and
metadata to memory_usage()."""
import os

import numpy as np
import pytest

from tests.test_gpu_host_tables import _all_tensors, _assert_bytes_equal
from tests.test_gpu_tsv_device import _index

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 256
MAX_NNZ = B * 2048
WAYS, SET_BITS = 8, 4


def _stride(plan):
    """Floats per staged host record [w | Adagrad slot] of the widest table."""
    return max((t["dim"] + 3) // 4 * 4 * 2 for t in plan.tables)


def _cache_bytes(plan):
    """HBM a cache of WAYS << SET_BITS slots adds: the slots at the front of the staging buffer, per slot tag / stamp / dirty, the
    use counter and four statistics, per staged row uslot / uvict / uflag, and the two (set, row) sort ping-pong pairs."""
    C = WAYS << SET_BITS
    return C * _stride(plan) * 4 + C * 9 + 4 + 4 * 8 + MAX_NNZ * 9 + 4 * (MAX_NNZ + 8) * 4


def _run(cfg, plan):
    from wide_deep_b200 import _native
    from wide_deep_b200.dataset import TextRing, TsvReader
    from wide_deep_b200.model import WideDeepModel
    m = WideDeepModel(plan).init(7)
    lib = _native.lib()
    before = m.memory_usage()
    _native.check(lib.wd_host_cache_enable(m._h, WAYS * (1 << SET_BITS) * _stride(plan) * 4))
    cached = m.memory_usage()
    assert m.host_cache_stats()["capacity"] == WAYS << SET_BITS

    reader = TsvReader(cfg, plan)
    text = open(os.path.join(ROOT, "data", "train", "train1"), "rb").read()
    starts, lens = _index(lib, text)
    assert len(starts) >= 3 * B
    idx = [np.arange(k * B, (k + 1) * B, dtype=np.int64) for k in range(3)]
    ring = TextRing(B, 1 << 20)
    losses = []
    m.prefetch_slot(3, reader.parse_indexed(text, starts, lens, idx[0]))
    m.parse_slot(1, reader.gather_text(text, starts, lens, idx[1], ring))
    assert m.tsv_parse_stats()["device"] == 1
    losses.append(m.train_step_slot(3))
    m.arm_summary()
    losses.append(m.train_step_slot(1))
    stats = m.layer_statistics()
    m.set_profile(True)
    losses.append(m.train_step(reader.parse_indexed(text, starts, lens, idx[2])))
    assert "h2d" in m.last_timings()
    m.set_profile(False)
    losses.append(m.train_step_slot(3))
    out = dict(before=before, cached=cached, end=m.memory_usage(), losses=np.float32(losses), counts=stats.counts.copy(),
               tensors=_all_tensors(m))
    m.close()
    ring.close()
    return out


def test_second_model_after_destroy_matches_the_first():
    from wide_deep_b200.config import Config
    from wide_deep_b200.plan import compile_plan
    cfg = Config()
    plan = compile_plan(cfg, "wide_deep", B, max_nnz=MAX_NNZ, max_keys=B * 512, host_tables="all")
    a = _run(cfg, plan)
    b = _run(cfg, plan)
    assert a["cached"][0] == a["before"][0] + _cache_bytes(plan)
    assert a["cached"][1] == a["before"][1] > 0
    for k in ("before", "cached", "end"):
        assert a[k] == b[k], k
    assert a["losses"].tobytes() == b["losses"].tobytes()
    assert a["counts"].tobytes() == b["counts"].tobytes()
    _assert_bytes_equal(a["tensors"], b["tensors"])
