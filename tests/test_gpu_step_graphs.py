"""Step graphs of the split data-parallel step on one GPU, without a process group: wd_step_backward_slot, a world-1 list
exchange on each list's side stream, the merge (wd_sparse_set_sorted or wd_sparse_set) and wd_step_apply.  Eight steps over two
alternating slots run each slot's forward + backward graph eager, eager, captured, replayed, and each list's sorted merge graph
eager twice, captured, then replayed five times.  The same steps with WD_NO_GRAPH=1 must give identical losses, tensors and launch
counts, and both must agree with plain wd_train_step on the same batches."""
import numpy as np
import pytest

from tests.helpers import copy_params_to_product, random_raw_batch, to_product_batch
from tests.test_gpu_parity import build_pair, small_conf
from wide_deep_b200.model import WideDeepModel

pytestmark = pytest.mark.gpu

B = 128
STEPS = 8
LISTS = (0, 1)          # embedding rows, wide rows (a wide_deep model has both)


def _split_steps(plan, om, batches, exchange):
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    losses = split_train(pm, batches, exchange)
    out = losses, {name: pm.get_tensor(name) for name in pm.tensor_names()}, pm.launch_count()
    pm.close()
    return out


def split_train(pm, batches, exchange):
    """The split step over two alternating slots with a world-1 exchange ("sorted" or "counted"); returns the losses."""
    import torch
    from wide_deep_b200.parallel import wrap_device
    dev = torch.device("cuda", pm.device)
    # the exchange's destination buffers are allocated once, so the sorted merge sees the same key every step; the merge cannot
    # read the library's own list in place (it writes the summed gradients there)
    bufs = {}
    for w in LISTS:
        _, _, _, width, cap = pm.sparse_grads(w, want_count=False)
        bufs[w] = (torch.empty(cap, dtype=torch.int32, device=dev), torch.empty((cap, width), dtype=torch.float32, device=dev))
    losses = []
    for i, batch in enumerate(batches):
        pm.upload_slot(i % 2, batch)
        pm.step_backward_slot(i % 2, want_loss=False)
        for w in LISTS:
            rows_ptr, grads_ptr, n, width, cap = pm.sparse_grads(w, want_count=exchange == "counted")
            k = cap if n is None else n
            r, g = bufs[w]
            with torch.cuda.stream(torch.cuda.ExternalStream(pm.stream_sparse(w), device=dev)):
                # the all-gather of a world-1 exchange
                r[:k].copy_(wrap_device(rows_ptr, (cap,), torch.int32, dev)[:k])
                g[:k].copy_(wrap_device(grads_ptr, (cap, width), torch.float32, dev)[:k])
                if exchange == "sorted":
                    pm.sparse_set_sorted(w, r.data_ptr(), g.data_ptr(), 1, cap)
                else:
                    pm.sparse_set(w, r.data_ptr(), g.data_ptr(), n)
        pm.step_apply()
        losses.append(pm.last_loss())
    pm.sync()
    return losses


@pytest.mark.parametrize("engine", ["ffma", "bf16x3"])
@pytest.mark.parametrize("exchange", ["sorted", "counted"])
def test_split_step_graphs_equal_eager(exchange, engine, monkeypatch):
    fc, cross, model = small_conf()
    om, plan, ref = build_pair(fc, cross, model, B=B, seed=11, engine=engine)
    rng = np.random.default_rng(13)
    batches = [to_product_batch(plan, random_raw_batch(fc, B, rng), (rng.random(B) < 0.3).astype(np.float32)) for _ in range(STEPS)]
    for batch in batches:
        ref.train_step(batch)
    expect = {name: ref.get_tensor(name) for name in ref.tensor_names()}
    ref.close()

    graph = _split_steps(plan, om, batches, exchange)
    monkeypatch.setenv("WD_NO_GRAPH", "1")          # read when the model is created
    eager = _split_steps(plan, om, batches, exchange)

    assert graph[0] == eager[0], (graph[0], eager[0])
    assert graph[2] == eager[2], (graph[2], eager[2])
    for name, exp in expect.items():
        np.testing.assert_array_equal(graph[1][name], eager[1][name], err_msg=name)
        scale = max(float(np.abs(exp).max()), 1e-3)
        err = float(np.max(np.abs(graph[1][name] - exp)))
        assert err <= 2e-5 * scale, "%s: max abs diff %g from wd_train_step (scale %g)" % (name, err, scale)
