"""Build libb2llava.so (sm_90a only) in-tree with nvcc. No torch dependency: the library is a plain
C-ABI shared object (include/b2llava.h) that the `llava` package binds with ctypes.

    python llava-plus-codebase_b200/build.py [--force] [--verbose]
"""
import argparse
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libb2llava.so")
SOURCES = ["gemm_wgmma.cu", "gemm_skinny.cu", "quant_fp8.cu", "gemv.cu", "decode_mega.cu", "attention.cu", "attention_wgmma.cu", "norms.cu", "vit_ops.cu", "misc_ops.cu", "sampling.cu", "beam.cu", "nf4.cu", "preprocess.cu", "model.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _newer(path, deps):
    if not os.path.exists(path):
        return False
    t = os.path.getmtime(path)
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(HERE, "..", "include", "b2llava.h"))
    objs, jobs = [], []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or not _newer(obj, [src] + headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for src, r in ex.map(compile_one, jobs):
            if r.returncode != 0:
                failed = True
                sys.stderr.write(f"[build] FAILED {src}\n{r.stdout}\n{r.stderr}\n")
            elif verbose:
                sys.stderr.write(f"[build] {os.path.basename(src)}\n{r.stderr}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if jobs or force or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
