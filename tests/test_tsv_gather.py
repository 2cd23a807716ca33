"""wd_tsv_gather_lines (host only): the lines picked by index are copied out of a file image, newline-separated, with their starts;
and input_fn(device_parse=True) yields the same lines, in the same batches, as the host path parses."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _index(lib, text):
    n = lib.wd_tsv_index_lines(text, len(text), None, None, 0)
    starts, lens = np.empty(max(n, 1), dtype=np.int64), np.empty(max(n, 1), dtype=np.int32)
    assert lib.wd_tsv_index_lines(text, len(text), starts.ctypes.data, lens.ctypes.data, n) == n
    return starts[:n], lens[:n]


@pytest.mark.parametrize("n_threads", [1, 8])
def test_gather_lines_matches_index(n_threads):
    from wide_deep_b200 import _native
    lib = _native.lib()
    rng = np.random.default_rng(5)
    lines = [bytes(rng.integers(32, 127, size=int(rng.integers(0, 90))).astype(np.uint8)) for _ in range(3000)]
    text = b"\n".join(l + (b"\r" if i % 7 == 0 else b"") for i, l in enumerate(lines)) + b"\n\n"
    starts, lens = _index(lib, text)
    kept = [l for i, l in enumerate(lines) if l or i % 7 == 0]          # "\r" alone is a line, an empty line is not
    assert len(starts) == len(kept)
    idx = rng.permutation(len(starts))[:2100].astype(np.int64)
    want = [kept[i] for i in idx]
    out_starts = np.empty(len(idx) + 1, dtype=np.int64)
    need = lib.wd_tsv_gather_lines(text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, len(idx), None, 0, out_starts.ctypes.data,
                                   n_threads)
    assert need == sum(len(l) + 1 for l in want) == out_starts[-1]
    small = np.zeros(need - 1, dtype=np.uint8)                       # too small: sizing only, nothing copied
    assert lib.wd_tsv_gather_lines(text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, len(idx), small.ctypes.data, small.size,
                                   out_starts.ctypes.data, n_threads) == need
    assert not small.any()
    out = np.zeros(need, dtype=np.uint8)
    assert lib.wd_tsv_gather_lines(text, starts.ctypes.data, lens.ctypes.data, idx.ctypes.data, len(idx), out.ctypes.data, out.size,
                                   out_starts.ctypes.data, n_threads) == need
    assert out.tobytes() == b"".join(l + b"\n" for l in want)
    for i, l in enumerate(want):
        assert out[out_starts[i]:out_starts[i + 1] - 1].tobytes() == l
    # idx NULL: the first n lines in file order
    out2 = np.zeros(need, dtype=np.uint8)
    n2 = lib.wd_tsv_gather_lines(text, starts.ctypes.data, lens.ctypes.data, None, 10, out2.ctypes.data, out2.size, out_starts.ctypes.data,
                                 n_threads)
    assert out2[:n2].tobytes() == b"".join(l + b"\n" for l in kept[:10])


def test_gather_lines_rejects_bad_arguments():
    from wide_deep_b200 import _native
    lib = _native.lib()
    assert lib.wd_tsv_gather_lines(b"a", None, None, None, 1, None, 0, None, 1) < 0
    assert b"bad arguments" in lib.wd_last_error()


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_device_parse_input_fn_yields_the_host_batches_lines(mode):
    """Same file image, shard and shuffle: the text of every TsvTextBatch, parsed on the host, is the Batch the host path yields."""
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import TsvTextBatch, input_fn
    from wide_deep_b200.plan import compile_plan
    cfg = Config()
    B = 700
    plan = compile_plan(cfg, "wide_deep", B, tf_compat_pad=True, max_nnz=B * 2048, max_keys=B * 512)
    path = os.path.join(ROOT, "data", "train")
    for rank, world in ((0, 1), (1, 2)):
        host = list(input_fn(path, None, mode, B, config=cfg, plan=plan, rank=rank, world=world))
        dev = input_fn(path, None, mode, B, config=cfg, plan=plan, rank=rank, world=world, device_parse=True)
        n = 0
        for hb, tb in zip(host, dev):                                # (lazily: a ring set is reused a few batches later)
            n += 1
            assert isinstance(tb, TsvTextBatch) and tb.batch_size == hb.batch_size and tb.has_label
            lines = [tb.text[tb.starts[i]:tb.starts[i + 1] - 1].tobytes() for i in range(tb.n)]
            again = tb.reader.parse(lines)
            assert np.array_equal(again.keys, hb.keys) and np.array_equal(again.offsets, hb.offsets)
            assert np.array_equal(again.dense, hb.dense) and np.array_equal(again.label, hb.label)
        assert n == len(host) and next(dev, None) is None


def test_float_fast_path_equals_strtof_on_long_decimals():
    """The float fast path shared by the host and device parsers takes decimals of up to 19 significant digits: every one of them
    must decode to what libc's strtof returns (the host parser's reference)."""
    import ctypes
    from wide_deep_b200 import _native
    from wide_deep_b200._native import TsvSpecC
    lib = _native.lib()
    libc = ctypes.CDLL(None)
    libc.strtof.restype, libc.strtof.argtypes = ctypes.c_float, [ctypes.c_char_p, ctypes.c_void_p]
    rng = np.random.default_rng(99)
    vals = []
    for _ in range(60000):
        nd = int(rng.integers(14, 20))
        digits = "".join(str(d) for d in rng.integers(0, 10, size=nd)).lstrip("0") or "1"
        cut = int(rng.integers(0, len(digits) + 1))
        vals.append(("-" if rng.random() < 0.3 else "") + digits[:cut] + "." + digits[cut:])
    # decimals next to float midpoints: k + 0.5 ulp for floats in [1, 2) and [2^20, 2^21), printed to 16 and 19 digits
    for f in rng.random(3000).astype(np.float32) + np.float32(1):
        mid = float(f) + 2.0 ** -24
        vals += ["%.15f" % mid, "%.18f" % mid, "%.18f" % (mid + 2.0 ** -60)]
    role, target = np.array([3], dtype=np.int32), np.array([0], dtype=np.int32)
    spec = TsvSpecC()
    spec.n_columns, spec.col_role, spec.col_target = 1, role.ctypes.data, target.ctypes.data
    spec.n_cat_fields, spec.n_dense_fields = 0, 1
    text = "\n".join(vals).encode()
    dense = np.zeros(len(vals), dtype=np.float32)
    offs = np.zeros(1, dtype=np.int32)
    assert lib.wd_tsv_parse(ctypes.byref(spec), text, len(text), len(vals), offs.ctypes.data, None, 0, dense.ctypes.data, None, None, 4) == 0
    ref = np.array([libc.strtof(v.encode(), None) for v in vals], dtype=np.float32)
    bad = np.nonzero(ref.view(np.uint32) != dense.view(np.uint32))[0]
    assert bad.size == 0, [(vals[i], dense[i], ref[i]) for i in bad[:5]]
