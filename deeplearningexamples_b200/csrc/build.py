"""Build libdle_b200.so in-tree with nvcc for sm_90a (H100) only.

    python -m deeplearningexamples_b200.csrc.build [--force]

Each .cu is compiled to an object (in parallel) and linked into
deeplearningexamples_b200/libdle_b200.so (git-ignored; objects go to csrc/build/).
"""
import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT = os.path.join(PKG, "libdle_b200.so")
OBJ_DIR = os.path.join(HERE, "build")
SOURCES = ["gemm_sm90.cu", "attention_sm90.cu", "lamb.cu", "pointwise.cu", "loss.cu", "distill_sm90.cu"]
HEADERS = [os.path.join(HERE, "common.cuh"), os.path.join(os.path.dirname(PKG), "include", "dle_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src):
    obj = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
    if _stale(obj, [os.path.join(HERE, src)] + HEADERS):
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(HERE, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return obj, True
    return obj, False


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    with cf.ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(_compile, SOURCES))
    objs = [o for o, _ in results]
    if any(c for _, c in results) or _stale(OUT, objs):
        cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("built", OUT)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
