"""In-tree build of libcozo_gpu.so (sm_90a, H100, only) with nvcc.

`python -m cozo_b200.build` or cozo_b200.build.build().  The library is placed at
cozo_b200/csrc/libcozo_gpu.so, next to the sources, so that the package runs from the repository tree.
Objects are rebuilt when a source, a header or this file (the flags) is newer than they are.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(CSRC, "libcozo_gpu.so")
SOURCES = ["common.cu", "hnsw.cu", "hnsw_f64.cu", "hnsw_build.cu", "graph.cu", "pagerank.cu", "merge.cu", "sharded.cu"]
HEADERS = ["common.cuh", "hnsw_codes.cuh", "hnsw_device.cuh", "hnsw_host.hpp", "graph_host.hpp", "pagerank_pb.cuh", "graph_kernels.cuh", "hnsw_build_kernels.cuh", os.path.join("..", "..", "include", "cozo_gpu.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = _nvcc()
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    jobs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs + [os.path.abspath(__file__)]):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), 8)) as ex:
            for log in ex.map(compile_one, jobs):
                if verbose and log:
                    print(log, file=sys.stderr)
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in srcs]
    if force or jobs or _stale(OUT, objs):
        cmd = [nvcc, "-shared", "-o", OUT] + objs + ARCH + ["-cudart", "static", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


def build_host(force: bool = False) -> str:
    """pybind11 harness over the C++ host layer (cozo_b200/host/*.hpp), linked against libcozo_gpu.so."""
    import sysconfig
    import pybind11
    host = os.path.join(HERE, "host")
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    out = os.path.join(host, "_cozo_host" + ext)
    deps = [os.path.join(host, f) for f in ("pymod.cpp", "data_value.hpp", "fixed_rule.hpp", "hnsw.hpp", "memcmp.hpp")]
    deps.append(os.path.join(CSRC, "..", "..", "include", "cozo_gpu.h"))
    if force or _stale(out, deps) or _stale(out, [OUT]):
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden",
               "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"],
               os.path.join(host, "pymod.cpp"), "-o", out,
               "-L", CSRC, "-lcozo_gpu", "-Wl,-rpath,$ORIGIN/../csrc"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"host module build failed:\n{r.stdout}\n{r.stderr}")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_host(force="--force" in sys.argv))
