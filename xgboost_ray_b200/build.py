"""Build libb2hist.so (sm_90a, H100) in-tree with nvcc.  Used by __graft_entry__.build().

    python -m xgboost_ray_b200.build [--force]

The .so and the object files are build products and stay out of git.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb2hist.so")
OBJ_DIR = os.path.join(CSRC, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
COMMON = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
          "-Xcompiler", "-fPIC,-ffp-contract=off", "-ccbin", "/usr/bin/g++"]
SOURCES = {
    "hist_kernel.cu": [],
    "hist_tma_kernel.cu": [],
    "split_kernel.cu": ["--fmad=false"],
    "partition_kernel.cu": ["--fmad=false"],
    "control_kernel.cu": ["--fmad=false"],
    "objective_kernel.cu": ["--fmad=false"],   # bit-exact gradients vs the oracle
    "sketch.cu": ["--fmad=false"],
    "auc_kernel.cu": ["--fmad=false"],
    "rank_kernel.cu": ["--fmad=false"],        # LambdaMART gradients and ranking metrics, bit-exact vs the reference
    "p2p_exchange.cu": [],                     # NVLink peer-memory histogram exchange
    "shap_kernel.cu": [],                      # TreeSHAP contributions / interactions, leaf indices
    "engine.cu": [],
}


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    headers = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "hist_common.cuh"), os.path.join(CSRC, "sampling.cuh"), os.path.join(CSRC, "p2p.cuh"), os.path.join(CSRC, "level_finalize.cuh"), os.path.join(CSRC, "decide.cuh"), os.path.join(CSRC, "objective_common.cuh"), os.path.join(HERE, "..", "include", "b2hist.h"), __file__]
    jobs = []
    objs = []
    for src, extra in SOURCES.items():
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        objs.append(op)
        if force or _stale(op, [sp] + headers):
            jobs.append([NVCC] + COMMON + extra + ["-c", sp, "-o", op])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n%s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r

    with ThreadPoolExecutor(max_workers=6) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _stale(OUT, objs):
        run([NVCC, "-shared", "-o", OUT] + objs + ["-ldl", "-ccbin", "/usr/bin/g++"])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
