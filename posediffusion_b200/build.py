"""Build libposediff_b200.so in-tree with nvcc for sm_90a (no torch headers, CUDA runtime only).

    python -m posediffusion_b200.build [--force]

The library is the product's only compute path; there is no fallback if it is missing.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(PKG, "libposediff_b200.so")
SOURCES = ["api_core.cu", "api_sampler.cu", "api_tc.cu", "api_vit.cu", "api_post.cu", "api_pre.cu", "api_train.cu", "api_vit_train.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v", f"-I{os.path.join(ROOT, 'include')}", f"-I{CSRC}"]


def nvcc_path() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libposediff_b200.so")
    return exe


def _deps() -> list:
    files = [os.path.join(ROOT, "include", "posediff_b200.h")]
    files += [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    return files


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    nvcc = nvcc_path()
    deps = _deps()
    objs, jobs = [], []
    for src in SOURCES:
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, deps):
            jobs.append([nvcc, *ARCH, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj])

    def run(cmd):
        res = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ, os.path.basename(cmd[cmd.index("-o") + 1]) + ".log")
        with open(log, "w") as fh:
            fh.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed: {' '.join(cmd)}\n{res.stdout}\n{res.stderr}")
        if verbose:
            print(res.stderr, file=sys.stderr)

    with ThreadPoolExecutor(max_workers=max(1, len(jobs))) as pool:
        list(pool.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run([nvcc, *ARCH, "-shared", "-o", LIB, *objs])
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
