"""Build the in-tree C-ABI shared library `vtp_b200/libvtp_b200.so` with nvcc for sm_90a.

No torch involvement: plain `nvcc -shared`, objects cached per source by mtime. Also builds oracle/ C checkers if
present.  Usage:  python -m vtp_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(HERE, "build")
LIB_PATH = os.path.join(HERE, "libvtp_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def sources() -> list[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers() -> list[str]:
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "vtp_b200.h"))
    return hs


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdrs = headers()
    objs, jobs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC, *NVCC_FLAGS, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, r in ex.map(compile_one, jobs):
                if verbose or r.returncode != 0:
                    sys.stderr.write(f"--- nvcc {os.path.basename(src)}\n{r.stdout}{r.stderr}\n")
                if r.returncode != 0:
                    raise RuntimeError(f"nvcc failed on {src}")
                with open(os.path.join(OBJ_DIR, os.path.basename(src) + ".ptxas.log"), "w") as f:
                    f.write(r.stderr)
    if force or jobs or _stale(LIB_PATH, objs):
        cmd = [NVCC, "-shared", "-o", LIB_PATH, *objs, "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
