"""Timeline of the nine 3xBF16 GEMM launches of one train step (CTA 0, globaltimer stamps via wd_debug_gemm_probe): when the first
operands land, when the main loop of the first / last tile ends, how long the tile epilogues take.  `python tools/gemm_probe.py`"""
import os, sys, ctypes, numpy as np
os.environ["WD_GEMM_PROBE"] = "1"; os.environ["WD_NO_GRAPH"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))   # repo root
from wide_deep_b200 import synthetic, _native
from wide_deep_b200.model import Batch, WideDeepModel
from wide_deep_b200.plan import Plan
B = 8192
fc, cross, model, emb = synthetic.criteo_conf()
n_cat = sum(1 for c in fc.values() if c["type"] == "category")
plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, max_nnz=B * (len(fc) + len(cross)), max_keys=B * n_cat, gemm_engine="bf16x3")
pm = WideDeepModel(plan); pm.init(1)
keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=0)
b = Batch(B, keys.reshape(-1), None, dense, label)
lib = _native.lib()
out = (ctypes.c_ulonglong * 256)()
for it in range(4):
    pm.train_step(b)
    lib.wd_debug_gemm_probe(out)
a = np.array(out[:], dtype=np.int64).reshape(32, 8)
names = ["fwd0", "fwd1", "fwd2", "dg2", "wg2", "dg1", "wg1", "dg0", "wg0"]
print("slot  first_data  mma_first_done  mma_last_done  epi_first_done  epi_last_done   (us from kernel start, CTA 0)")
for i in range(9):
    r = a[i]; t0 = r[0]
    print(names[i], " ".join("%8.1f" % ((x - t0) / 1e3) if x > 0 else "       -" for x in r[1:6]))
