"""The nine 3xBF16 GEMM launches of one Criteo-shaped train step (B = 8192).  `python tools/gemm_probe.py`

1. Timeline of CTA 0 (globaltimer stamps via wd_debug_gemm_probe, WD_GEMM_PROBE=1): when the first operands land, when the main
   loop of the first / last tile ends, when the epilogue of the first / last tile ends.
2. Per launch: the mean CUDA-event time over 20 profiled steps (set_profile / last_timings, phases gemm_*), set against the
   shape: 128 x 128 x 64 tile blocks, the tensor bound at 989 TFLOP/s (data sheet, 3 bf16 products), the operand bytes that pass
   from L2 into shared memory (64 KB per tile block), the achieved operand rate, the epilogue bytes, and the main-loop and
   epilogue time of CTA 0's first tile."""
import os, sys, ctypes, subprocess, numpy as np
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
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
except OSError:
    print("nvidia-smi not available")
print("slot  first_data  mma_first_done  mma_last_done  epi_first_done  epi_last_done   (us from kernel start, CTA 0)")
for i in range(9):
    r = a[i]; t0 = r[0]
    print(names[i], " ".join("%8.1f" % ((x - t0) / 1e3) if x > 0 else "       -" for x in r[1:6]))

# ---- per-launch event times
pm.set_profile(True)
acc, n = {}, 20
for it in range(n):
    pm.train_step(b)
    for k, v in pm.last_timings().items():
        if k.startswith("gemm_"):
            acc[k] = acc.get(k, 0.0) + v / n
pm.set_profile(False)

dims = [plan.d0_phys] + [int(u) for u in model["dnn_hidden_units"]]
def wgrad_splits(K, N):                    # the rule of api.cu (initial split 4, 132 SMs, each split >= 512 rows)
    tiles, sp = ((K + 127) // 128) * ((N + 127) // 128), 4
    while sp < 32 and tiles * sp * 2 <= 132 and B // (sp * 2) >= 512:
        sp *= 2
    return sp
rows = []
for l in range(3):                         # launch order: fwd0 fwd1 fwd2, then dg2 wg2 dg1 wg1 dg0 wg0
    K, N = dims[l], dims[l + 1]
    rows.append(("fwd%d" % l, "gemm_fwd_l%d" % l, B, N, K, 1, B * N * (12 if l == 2 else 8)))   # fp32 post-activation + bf16 hi/lo (+ fp32 output the logits read)
for l in (2, 1, 0):
    K, N = dims[l], dims[l + 1]
    rows.append(("dg%d" % l, "gemm_dgrad_l%d" % l, B, K, N, 1, B * K * 4))
    sp = wgrad_splits(K, N)
    rows.append(("wg%d" % l, "gemm_wgrad_l%d" % l, K, N, B, sp, K * N * 4 * sp))
order = {nm: i for i, nm in enumerate(names)}
print("\nlaunch  M x N x K            tiles(xsplits)  tile.kb  bound_us  operand_MB  epilogue_MB  measured_us  operand_TB/s  mainloop_us/tile  epilogue_us/tile")
tot = dict(tkb=0, bound=0.0, op=0.0, epi=0.0, meas=0.0)
for nm, phase, M, N, K, sp, epi_bytes in rows:
    tiles = ((M + 127) // 128) * ((N + 127) // 128)
    kb = (K + 63) // 64                    # k-blocks over the whole reduction, summed over the splits
    tkb = tiles * kb
    bound = 6.0 * M * N * K / 989e12 * 1e6
    op_mb = tkb * 65536 / 1e6
    meas = acc.get(phase, float("nan")) * 1e3
    r = a[order[nm]]
    ml = (r[2] - r[1]) / 1e3 if r[2] > 0 and r[1] > 0 else float("nan")
    ep = (r[4] - r[2]) / 1e3 if r[4] > 0 and r[2] > 0 else float("nan")
    print("%-6s  %5d x %4d x %4d  %4d%-9s  %6d  %8.1f  %10.0f  %11.0f  %11.1f  %12.2f  %16.1f  %16.1f" % (
        nm, M, N, K, tiles, (" x %d" % sp) if sp > 1 else "", tkb, bound, op_mb, epi_bytes / 1e6, meas, op_mb / meas, ml, ep))
    tot["tkb"] += tkb; tot["bound"] += bound; tot["op"] += op_mb; tot["epi"] += epi_bytes / 1e6; tot["meas"] += meas
print("sum     %37d  %8.1f  %10.0f  %11.0f  %11.1f  %12.2f" % (tot["tkb"], tot["bound"], tot["op"], tot["epi"], tot["meas"], tot["op"] / tot["meas"]))
