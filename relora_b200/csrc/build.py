"""Build the in-tree sm_90a extension ``relora_b200/_C.so``.

    python -m relora_b200.csrc.build [--force] [--verbose]

Kernel sources are plain CUDA (no torch headers) compiled with
``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo``; ``bindings.cpp`` (pybind11 over
``torch::Tensor``) is compiled with the host compiler and everything is linked into one shared
object next to the package.  nvcc cross-compiles without a GPU, so this runs on the CPU build box;
the resulting ``.so`` travels with the repository snapshot to the H100.  A content hash of the
sources + flags makes rebuilds incremental.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import hashlib
import json
import os
import shutil
import subprocess
import sys
import sysconfig
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
BUILD_DIR = os.path.join(HERE, "_build")
TARGET = os.path.join(PKG, "_C.so")

CUDA_SOURCES = ["gemm_wgmma.cu", "elementwise.cu", "norm_warp.cu", "rope.cu", "optim.cu", "loss.cu", "attention.cu", "fp8.cu", "comm.cu", "neox.cu", "gemm_mx.cu"]
CPP_SOURCES = ["bindings.cpp"]
HEADERS = ["common.cuh", "sm90.cuh", "gemm.h", "tensormap.h", "fp8out.h", "kernels.h", "attention.h", "comm.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
] + os.environ.get("RB_EXTRA_NVCC_FLAGS", "").split()  # e.g. -DRB_ATTN_GROUPS_FWD=3 for kernel experiments


def _cuda_home() -> str:
    for cand in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if cand and os.path.exists(os.path.join(cand, "bin", "nvcc")):
            return cand
    nvcc = shutil.which("nvcc")
    if nvcc:
        return os.path.dirname(os.path.dirname(nvcc))
    raise RuntimeError("nvcc not found; set CUDA_HOME")


def _torch_paths():
    import torch
    from torch.utils import cpp_extension

    inc = cpp_extension.include_paths()
    lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    return inc, lib, abi


def _existing(names: List[str]) -> List[str]:
    return [n for n in names if os.path.exists(os.path.join(HERE, n))]


def _digest(files: List[str], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for f in sorted(files):
        with open(os.path.join(HERE, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    return h.hexdigest()


def _run(cmd: List[str], verbose: bool, log_name: str) -> None:
    res = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(BUILD_DIR, log_name + ".log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(f"build step failed: {' '.join(cmd)}")


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD_DIR, exist_ok=True)
    cuda = _cuda_home()
    nvcc = os.path.join(cuda, "bin", "nvcc")
    inc, torch_lib, abi = _torch_paths()
    cu = _existing(CUDA_SOURCES)
    cpp = _existing(CPP_SOURCES)
    hdr = _existing(HEADERS)
    import torch

    stamp = _digest(cu + cpp + hdr, json.dumps([NVCC_FLAGS, torch.__version__, sys.version]))
    stamp_file = os.path.join(BUILD_DIR, "stamp.json")
    if not force and os.path.exists(TARGET) and os.path.exists(stamp_file):
        try:
            if json.load(open(stamp_file)).get("digest") == stamp:
                return TARGET
        except Exception:
            pass

    py_inc = sysconfig.get_paths()["include"]
    host_flags = ["-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=_C",
                  "-DTORCH_API_INCLUDE_EXTENSION_H", "-Wno-deprecated-declarations"]
    incs = [f"-I{p}" for p in inc] + [f"-I{py_inc}", f"-I{os.path.join(cuda, 'include')}", f"-I{HERE}"]

    jobs = []
    objs = []
    per_file_digest = {}
    old = {}
    if os.path.exists(stamp_file):
        try:
            old = json.load(open(stamp_file)).get("files", {})
        except Exception:
            old = {}
    hdr_digest = _digest(hdr, "")
    for src in cu:
        obj = os.path.join(BUILD_DIR, src + ".o")
        objs.append(obj)
        dg = _digest([src], hdr_digest + json.dumps(NVCC_FLAGS))
        per_file_digest[src] = dg
        if force or not os.path.exists(obj) or old.get(src) != dg:
            jobs.append(([nvcc, *NVCC_FLAGS, f"-I{HERE}", "-c", os.path.join(HERE, src), "-o", obj], src))
    for src in cpp:
        obj = os.path.join(BUILD_DIR, src + ".o")
        objs.append(obj)
        dg = _digest([src], hdr_digest + json.dumps(host_flags) + torch.__version__)
        per_file_digest[src] = dg
        if force or not os.path.exists(obj) or old.get(src) != dg:
            cxx = os.environ.get("CXX", "g++")
            jobs.append(([cxx, *host_flags, *incs, "-c", os.path.join(HERE, src), "-o", obj], src))

    with cf.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
        futs = [pool.submit(_run, cmd, verbose, name) for cmd, name in jobs]
        for f in futs:
            f.result()

    cxx = os.environ.get("CXX", "g++")
    link = [cxx, "-shared", "-o", TARGET + ".tmp", *objs, f"-L{torch_lib}", "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10",
            "-lc10_cuda", "-ltorch_python", f"-L{os.path.join(cuda, 'lib64')}", "-lcudart",
            f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}"]
    _run(link, verbose, "link")
    os.replace(TARGET + ".tmp", TARGET)
    with open(stamp_file, "w") as f:
        json.dump({"digest": stamp, "files": per_file_digest}, f)
    return TARGET


def ptxas_report() -> str:
    """Concatenate the ``-Xptxas -v`` output of the last build (registers / spills / smem per kernel)."""
    out = []
    for src in _existing(CUDA_SOURCES):
        p = os.path.join(BUILD_DIR, src + ".log")
        if os.path.exists(p):
            out.append(open(p).read())
    return "\n".join(out)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
