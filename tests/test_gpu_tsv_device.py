"""Device TSV parser (wd_tsv_parse_slot): a batch slot filled on the GPU from TSV text must hold, byte for byte, what the host
parser + wd_batch_prefetch_slot put there — on every bundled file and option, on a seeded corpus of edge cases, with the host
parser's error messages, and through whole training / evaluation runs."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = [("train", "train1"), ("train", "train2"), ("eval", "eval1"), ("test", "test1"), ("test", "test2"), ("pred", "pred1")]


def _config(multivalue, weights):
    from wide_deep_b200.config import Config
    cfg = Config()
    cfg.train["multivalue"] = 1 if multivalue else 0
    cfg.train["pos_sample_loss_weight"], cfg.train["neg_sample_loss_weight"] = (0.75, 0.25) if weights else (None, None)
    return cfg


def _model(cfg, pad, B, max_keys=None):
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import compile_plan
    plan = compile_plan(cfg, "wide_deep", B, tf_compat_pad=pad, max_nnz=B * 2048, max_keys=max_keys or B * 512)
    return WideDeepModel(plan)


def _index(lib, text):
    n = lib.wd_tsv_index_lines(text, len(text), None, None, 0)
    starts, lens = np.empty(max(n, 1), dtype=np.int64), np.empty(max(n, 1), dtype=np.int32)
    lib.wd_tsv_index_lines(text, len(text), starts.ctypes.data, lens.ctypes.data, n)
    return starts[:n], lens[:n]


def _assert_same(a, b, what):
    assert a.batch_size == b.batch_size, what
    for name in ("offsets", "keys", "dense", "label", "weight"):
        x, y = getattr(a, name), getattr(b, name)
        assert (x is None) == (y is None), (what, name)
        if x is not None:
            assert x.shape == y.shape and x.tobytes() == y.tobytes(), (what, name)


def _host_slot(m, slot, batch):
    m.prefetch_slot(slot, batch)
    return m.slot_batch(slot)


def _device_slot(m, slot, tb):
    m.parse_slot(slot, tb)
    return m.slot_batch(slot)


@pytest.mark.parametrize("pad", [0, 1])
@pytest.mark.parametrize("multivalue", [0, 1])
@pytest.mark.parametrize("weights", [0, 1])
def test_bundled_files_byte_equal_without_fallback(pad, multivalue, weights):
    from wide_deep_b200 import _native
    from wide_deep_b200.dataset import TextRing, TsvReader
    lib = _native.lib()
    cfg = _config(multivalue, weights)
    m = _model(cfg, bool(pad), 2048)
    m.tsv_parse_stats(reset=True)
    n_dev = 0
    for d, f in FILES:
        reader = TsvReader(cfg, m.plan, is_pred=(d == "pred"))
        text = open(os.path.join(ROOT, "data", d, f), "rb").read()
        starts, lens = _index(lib, text)
        ring = TextRing(2048, 1 << 20)
        for B, limit in ((1, 40), (64, None), (2048, None)):
            n = len(starts) if limit is None else min(limit, len(starts))
            for lo in range(0, n, B):                                  # the last batch is a ragged tail
                idx = np.arange(lo, min(lo + B, n), dtype=np.int64)
                host = _host_slot(m, 1, reader.parse_indexed(text, starts, lens, idx))
                dev = _device_slot(m, 0, reader.gather_text(text, starts, lens, idx, ring))
                _assert_same(dev, host, (f, B, lo))
                n_dev += 1
        ring.close()
    assert m.tsv_parse_stats() == dict(device=n_dev, host=0)


# ---- seeded edge corpus over the bundled schema
FAST_STR = ["-", "", "a", ",,", ",a", "a,", ",", ",,,", "a,,b", "x,y,z", "é,ü", "中文,日本", "ÿ" * 3, "k" * 65, "L" * 200 + ",s",
            "T1348648756099,T1356600029035", "-,-", " ", "a b"]
FAST_INT = ["-", "", "0", "-0", "007", "123456789012345678", "-123456789012345678", "42", "-5"]
SLOW_INT = ["1234567890123456789", " 1", "+1", "-0000000000000000001"]
FAST_FLOAT = ["-", "", "0", "-0", "0.0", "1.5", "-2.25", "123456789012345", "0.000000000000001", "1.23456789012345", "00012.5", "3.",
              ".5", "99999.999", "121.5958455249209", "23.36158434150282", "1.234567890123456", "1234567890123456", "1.00000005960464",
              "0.1000000014901161", "-9999999999999999999", "0.0000000000000000000001"]
# exponents, inf, spaces, '+', 20 digits, float midpoints (2^24 + 1) and decimals within a few double ulps of one
SLOW_FLOAT = ["1e5", "inf", "-inf", " 1", "+1", "12345678901234567890", "16777217", "33554434", "1.0000000596046448"]
FAST_LABEL = ["1", "01", "0", "-", "", "2", "-1"]
SLOW_LABEL = ["1.0", " 1", "+1"]


def _corpus(reader, rng, n, slow):
    role = reader._role
    ints, floats, labels = FAST_INT + (SLOW_INT if slow else []), FAST_FLOAT + (SLOW_FLOAT if slow else []), FAST_LABEL + (SLOW_LABEL if slow else [])
    lines = []
    for _ in range(n):
        cols = []
        for r in role:
            if r == 0:
                cols.append(labels[rng.integers(len(labels))])
            elif r == 1:
                cols.append(FAST_STR[rng.integers(len(FAST_STR))])
            elif r == 2:
                cols.append(ints[rng.integers(len(ints))])
            elif r == 3:
                cols.append(floats[rng.integers(len(floats))])
            else:
                cols.append(FAST_STR[rng.integers(len(FAST_STR))].replace(",", ""))
        lines.append("\t".join(cols).encode("utf-8"))
    return lines


def _text_batch(reader, lines, sep=b"\n"):
    """TsvTextBatch over hand-joined lines (sep b"\\r\\n": CRLF text, the '\\r' is not part of a line)."""
    from wide_deep_b200.dataset import TextRing, TsvTextBatch
    body = b"".join(l + sep for l in lines)
    ring = TextRing(len(lines), len(body) + 64, depth=1)
    s = ring.next(len(body))
    s["text"][:len(body)] = np.frombuffer(body, dtype=np.uint8)
    pos, starts = 0, [0]
    for l in lines:
        pos += len(l) + len(sep)
        starts.append(pos)
    s["starts"][:len(starts)] = starts
    tb = TsvTextBatch(reader, s["text"], s["starts"][:len(starts)], len(lines))
    tb._ring = ring
    return tb


@pytest.mark.parametrize("pad", [0, 1])
@pytest.mark.parametrize("multivalue", [0, 1])
def test_edge_corpus_byte_equal(pad, multivalue):
    from wide_deep_b200.dataset import TsvReader
    cfg = _config(multivalue, True)
    B = 256
    m = _model(cfg, bool(pad), B)
    reader = TsvReader(cfg, m.plan)
    rng = np.random.default_rng(1234 + 2 * pad + multivalue)
    for slow in (False, True):
        for step, sep in enumerate((b"\n", b"\r\n", b"\n", b"\r\n")):
            lines = _corpus(reader, rng, B - 37 * step, slow)
            m.tsv_parse_stats(reset=True)
            dev = _device_slot(m, 0, _text_batch(reader, lines, sep))
            host = _host_slot(m, 1, reader.parse(lines))
            _assert_same(dev, host, (slow, step))
            if not slow:
                assert m.tsv_parse_stats() == dict(device=1, host=0), step
    # every slow shape alone, in a batch of fast lines: byte-equal through the host fallback
    base = _corpus(reader, rng, 8, False)
    cols = [c.split(b"\t") for c in base]
    for r_want, shapes in ((2, SLOW_INT), (3, SLOW_FLOAT), (0, SLOW_LABEL)):
        c = int(np.nonzero(reader._role == r_want)[0][0])
        for v in shapes:
            lines = ["\t".join(x.decode() if j != c or i != 3 else v for j, x in enumerate(row)).encode() for i, row in enumerate(cols)]
            m.tsv_parse_stats(reset=True)
            dev = _device_slot(m, 0, _text_batch(reader, lines))
            host = _host_slot(m, 1, reader.parse(lines))
            _assert_same(dev, host, v)
            assert m.tsv_parse_stats() == dict(device=0, host=1), v


def test_errors_carry_host_messages():
    from wide_deep_b200._native import NativeError
    from wide_deep_b200.dataset import TsvReader
    cfg = _config(1, False)
    B = 64
    m = _model(cfg, True, B)
    reader = TsvReader(cfg, m.plan)
    rng = np.random.default_rng(7)
    good = _corpus(reader, rng, 20, False)
    cols = good[5].split(b"\t")
    ci = int(np.nonzero(reader._role == 2)[0][0])
    cf = int(np.nonzero(reader._role == 3)[0][0])
    bad_rows = [b"\t".join(cols[:-1]),                                                   # one field short
                good[5] + b"\textra",                                                    # one field too many
                b"\t".join(b"12x" if j == ci else x for j, x in enumerate(cols)),        # not an int
                b"\t".join(b"1.2.3" if j == cf else x for j, x in enumerate(cols))]      # not a float
    for bad in bad_rows:
        lines = good[:5] + [bad] + good[6:]
        with pytest.raises(ValueError) as host_err:
            reader.parse(lines)
        with pytest.raises(NativeError) as dev_err:
            m.parse_slot(0, _text_batch(reader, lines))
        assert str(host_err.value) in str(dev_err.value), (str(host_err.value), str(dev_err.value))
    # key overflow: a model whose slots hold fewer keys than the batch has
    small = _model(cfg, True, B, max_keys=B)
    lines = _corpus(reader, rng, B, False)
    with pytest.raises(NativeError) as host_err:
        small.prefetch_slot(1, reader.parse(lines))
    with pytest.raises(NativeError) as dev_err:
        small.parse_slot(0, _text_batch(reader, lines))
    assert "keys, capacity" in str(host_err.value) and str(host_err.value) == str(dev_err.value)


def _train_eval(tmp, device_parse, B):
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import input_fn
    from wide_deep_b200.estimator import build_custom_estimator
    cfg = Config()
    cfg.runconfig["save_checkpoints_steps"], cfg.runconfig["save_checkpoints_secs"] = None, 10 ** 9
    est = build_custom_estimator(os.path.join(tmp, "dp%d" % device_parse), "wide_deep", config=cfg, max_batch=B)
    m = est._ensure_model()
    losses, last = [], m.last_loss
    m.last_loss = lambda: losses.append(last()) or losses[-1]
    kw = dict(device_parse=True) if device_parse else {}
    est.train(input_fn=lambda: input_fn(os.path.join(ROOT, "data", "train"), None, "train", B, config=cfg, plan=est.plan,
                                        pinned=not device_parse, **kw))
    metrics = est.evaluate(input_fn=lambda: input_fn(os.path.join(ROOT, "data", "eval"), None, "eval", B, config=cfg, plan=est.plan, **kw))
    tensors = {}
    for name in m.tensor_names():
        for s in range(m.n_slots(name) + 1):
            tensors[(name, s)] = m.get_tensor(name, slot=s)
    return losses, metrics, tensors, m.tsv_parse_stats()


def test_training_and_evaluation_byte_equal(tmp_path):
    B = 512
    l0, m0, t0, s0 = _train_eval(str(tmp_path), False, B)
    l1, m1, t1, s1 = _train_eval(str(tmp_path), True, B)
    assert s0 == dict(device=0, host=0)
    assert s1["host"] == 0 and s1["device"] == len(l1) + (5000 + B - 1) // B
    assert np.array(l0, dtype=np.float32).tobytes() == np.array(l1, dtype=np.float32).tobytes()
    # the metric kernel sums in double with atomics (misc.cu), so two evaluations of byte-identical batches with byte-identical
    # parameters may differ in the last bits of a sum's order; anything beyond that would be a different input
    assert m0.keys() == m1.keys()
    for k in m0:
        assert m0[k] == m1[k] or abs(m0[k] - m1[k]) <= 1e-12 * abs(m0[k]), (k, m0[k], m1[k])
    for k in t0:
        assert t0[k].tobytes() == t1[k].tobytes(), k


def test_local_shard_group_byte_equal():
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import input_fn
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import compile_plan
    from wide_deep_b200.sharded import LocalShardGroup
    cfg = Config()
    G, per = 2, 256
    path = os.path.join(ROOT, "data", "train")

    def group():
        models = []
        for r in range(G):
            plan = compile_plan(cfg, "wide_deep", per, tf_compat_pad=True, shard_world=G, shard_rank=r, shard_slack=float(G),
                                max_nnz=per * 2048, max_keys=per * 512)
            models.append(WideDeepModel(plan).init(11))
        return LocalShardGroup(models)

    host, dev = group(), group()
    its_h = [input_fn(path, None, "train", per, config=cfg, plan=host.models[r].plan, rank=r, world=G) for r in range(G)]
    its_d = [input_fn(path, None, "train", per, config=cfg, plan=dev.models[r].plan, rank=r, world=G, device_parse=True) for r in range(G)]
    steps = 0
    for hb, tb in zip(zip(*its_h), zip(*its_d)):
        lh = host.train_step(list(hb))
        for m, t in zip(dev.models, tb):
            m.parse_slot(0, t)
        ld = dev.train_step(None)
        assert np.float32(lh).tobytes() == np.float32(ld).tobytes(), steps
        steps += 1
    assert steps > 10
    for m in dev.models:
        assert m.tsv_parse_stats() == dict(device=steps, host=0)
    for name in host.models[0].tensor_names():
        for s in range(host.models[0].n_slots(name) + 1):
            assert host.get_tensor(name, s).tobytes() == dev.get_tensor(name, s).tobytes(), (name, s)
