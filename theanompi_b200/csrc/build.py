"""Ahead-of-time build of ``_tmpi_native.so`` for sm_90a (H100).

    python -m theanompi_b200.csrc.build [--force] [--verbose]

Every ``.cu`` is compiled with
``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3`` (``wgmma`` / ``setmaxnreg``
need the *a* feature target); ``.cpp`` files with g++; everything is linked into ONE shared
object placed inside the package so it travels with the source tree (git-ignored).  cudart is linked
statically and the driver API is reached through ``cudaGetDriverEntryPoint``, so the
module imports on a machine without a GPU driver.

A content hash of sources + flags is stored next to the ``.so``; ``build()`` is a
no-op when it matches.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
SO_PATH = os.path.join(PKG, "_tmpi_native.so")
OBJ_DIR = os.path.join(HERE, "_obj")
STAMP = os.path.join(PKG, "_tmpi_native.hash")

CU_SOURCES = ["gemm_wgmma.cu", "gemm_sgd.cu", "nn_kernels.cu", "bn_kernels.cu", "rnn_kernels.cu", "comm_kernels.cu"]
CPP_SOURCES = ["peer_arena.cpp", "binding.cpp"]
HEADERS = ["common.cuh", "gemm_wgmma.cuh", "api.h", "peer_arena.h"]

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "--use_fast_math", "-Xcompiler", "-fPIC",
                     "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function"]


def _includes():
    import pybind11
    return ["-I" + HERE, "-I" + os.path.join(CUDA_HOME, "include"), "-I" + pybind11.get_include(),
            "-I" + sysconfig.get_paths()["include"]]


def _hash():
    h = hashlib.sha256()
    for f in CU_SOURCES + CPP_SOURCES + HEADERS:
        with open(os.path.join(HERE, f), "rb") as fh:
            h.update(f.encode()); h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS + CXX_FLAGS).encode())
    h.update(sys.version.encode())
    return h.hexdigest()


def is_current():
    if not (os.path.exists(SO_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _hash()


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build step failed:\n%s\n%s" % (" ".join(cmd), r.stdout))
    if verbose and r.stdout.strip():
        print(r.stdout)
    return r.stdout


def build(force=False, verbose=False):
    if not force and is_current():
        if verbose:
            print("_tmpi_native.so is up to date")
        return SO_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    inc = _includes()
    jobs = []
    for f in CU_SOURCES:
        o = os.path.join(OBJ_DIR, f + ".o")
        jobs.append(([NVCC] + NVCC_FLAGS + inc + ["-c", os.path.join(HERE, f), "-o", o], o))
    for f in CPP_SOURCES:
        o = os.path.join(OBJ_DIR, f + ".o")
        jobs.append((["g++"] + CXX_FLAGS + inc + ["-c", os.path.join(HERE, f), "-o", o], o))
    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        list(ex.map(lambda j: _run(j[0], verbose), jobs))
    objs = [j[1] for j in jobs]
    link = [NVCC] + ARCH + ["-shared", "-o", SO_PATH] + objs + ["-cudart", "static", "-lpthread", "-ldl", "-lrt"]
    _run(link, verbose)
    with open(STAMP, "w") as f:
        f.write(_hash())
    return SO_PATH


def sass_summary(path=None):
    """Count the Hopper-specific SASS mnemonics in the built object (HGMMA = wgmma, UTMALDG = TMA loads, ...)."""
    import collections
    import re
    out = subprocess.run([os.path.join(CUDA_HOME, "bin", "cuobjdump"), "-sass", path or SO_PATH],
                         stdout=subprocess.PIPE, text=True).stdout
    pat = re.compile(r"\b(HGMMA|UTMALDG|UTMASTG|UBLKCP|UBLKRED|SYNCS|HMMA|MULTIMEM|RED|LDG\.E\.128)[A-Z0-9_.]*")
    cnt = collections.Counter(m.group(0).split(".")[0] for m in pat.finditer(out))
    return dict(cnt)


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv)
    print("built", p)
    if "--sass" in sys.argv:
        print(sass_summary())
