"""In-tree build of ``ring_flash_attn_b200/_C*.so`` for sm_90a (H100).

nvcc cross-compiles without a GPU, so this runs on the CPU dev box; the resulting shared object lives
next to the sources (git-ignored) and travels with the tree.  Incremental: a translation unit is rebuilt
only when it or a header is newer than its object file.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-DRFA_BUILD"]
if os.environ.get("RFA_TRACE", "0") == "1":
    NVCC_FLAGS.append("-DRFA_TRACE")
CU_SOURCES = ["attn_fwd_sm90.cu", "attn_bwd_sm90.cu", "tensor_map.cu", "lse_layout.cu", "comm_sm90.cu"]
CPP_SOURCES = ["bindings.cpp", "peer_mem.cpp"]


def _so_path() -> str:
    return os.path.join(HERE, "_C" + sysconfig.get_config_var("EXT_SUFFIX"))


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build step failed:\n" + " ".join(cmd) + "\n" + r.stdout)
    return r.stdout


def build(verbose: bool = False, force: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension

    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    inc = []
    for p in cpp_extension.include_paths("cuda"):
        inc += ["-I", p]
    inc += ["-I", sysconfig.get_paths()["include"], "-I", CSRC]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    jobs = []
    objs = []
    for src in CU_SOURCES:
        s, o = os.path.join(CSRC, src), os.path.join(BUILD, src + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append([os.path.join(CUDA_HOME, "bin", "nvcc"), *NVCC_FLAGS, "-I", CSRC, "-c", s, "-o", o])
    for src in CPP_SOURCES:
        s, o = os.path.join(CSRC, src), os.path.join(BUILD, src + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append(["g++", "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                         "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H", *inc, "-c", s, "-o", o])
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for out in ex.map(_run, jobs):
            if verbose and out.strip():
                print(out)
    so = _so_path()
    if force or jobs or _stale(so, objs):
        libdirs = cpp_extension.library_paths("cuda")
        link = ["g++", "-shared", "-o", so, *objs]
        for d in libdirs:
            link += ["-L", d, f"-Wl,-rpath,{d}"]
        link += ["-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
        out = _run(link)
        if verbose and out.strip():
            print(out)
    return so


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
