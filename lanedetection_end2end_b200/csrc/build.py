"""Build liblanefit_b200.so in-tree with nvcc for sm_90a (H100) (no torch headers involved).

    python -m lanedetection_end2end_b200.csrc.build [--force] [--verbose]
"""
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "liblanefit_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    srcs = sorted(glob.glob(os.path.join(HERE, "*.cu")))
    hdrs = glob.glob(os.path.join(HERE, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "..", "include", "*.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    newest_hdr = max([os.path.getmtime(h) for h in hdrs] + [0.0])

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), newest_hdr):
            return obj, False
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj, True

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(compile_one, srcs))
    objs = [o for o, _ in res]
    if force or any(c for _, c in res) or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
