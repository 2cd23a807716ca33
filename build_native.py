"""Build libwd_b200.so (in-tree) with nvcc for sm_90a.  Used by __graft_entry__.build() and by hand:
    python build_native.py [--force]
The .so and the objects under build/ are git-ignored: history stays source-only and every checkout builds its own."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(ROOT, "wide_deep_b200", "csrc")
OUT = os.path.join(ROOT, "wide_deep_b200", "libwd_b200.so")
SOURCES = ["api.cu", "ids.cu", "sort.cu", "sparse.cu", "mlp.cu", "gemm_tc.cu", "gemm_bf16.cu", "misc.cu", "tsv.cu", "shard.cu", "host_tables.cu", "summary.cu"]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v" if os.environ.get("WD_PTXAS_V") else "-O3"]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(SRC, f) for f in os.listdir(SRC)] + [os.path.join(ROOT, "include", "wd_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    for s in SOURCES:
        o = os.path.join(ROOT, "build", s.replace(".cu", ".o"))
        src = os.path.join(SRC, s)
        objs.append(o)
        if not force and os.path.exists(o) and os.path.getmtime(o) > max(
                os.path.getmtime(src), *[os.path.getmtime(os.path.join(SRC, h)) for h in os.listdir(SRC) if h.endswith(".cuh")],
                os.path.getmtime(os.path.join(ROOT, "include", "wd_b200.h"))):
            continue
        cmd = ["nvcc"] + FLAGS + ["-c", src, "-o", o]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    fail = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or (verbose and out.strip()):
            print("---- %s\n%s" % (s, out))
        fail |= p.returncode != 0
    if fail:
        raise RuntimeError("nvcc failed")
    cmd = ["nvcc", "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print(OUT)
