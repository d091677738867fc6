"""In-tree build of the native code (needs no GPU: nvcc cross-compiles for sm_90a):

    python -m bert_pytorch_b200.ops.build            # everything
    python -m bert_pytorch_b200.ops.build --host     # only the host helper

Produces ``ops/_C.so`` (CUDA kernels + torch bindings) and ``ops/_host.so`` (HDF5 chunk inflate +
dynamic masking, plain C++).  The kernels are compiled with plain nvcc (no torch headers -> seconds
per file) and only ``bindings.cpp`` sees torch; objects are cached by source hash under
``ops/_build``.  The ``.so`` files and ``ops/_build`` are build products (git-ignored).
"""
from __future__ import annotations

import argparse
import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")

CUDA_SOURCES = ["gemm_sm90.cu", "norm_embed.cu", "optim.cu", "loss.cu", "attention_sm90.cu", "comm.cu", "fp8.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
# erff/expf accuracy matters for GELU and softmax statistics -> no fast-math there
PRECISE = set(CUDA_SOURCES)


def _cuda_home() -> str:
    for c in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if c and os.path.exists(os.path.join(c, "bin", "nvcc")):
            return c
    raise RuntimeError("nvcc not found (set CUDA_HOME)")


def _digest(paths: List[str], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:16]


def _headers() -> List[str]:
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]


def _run(cmd: List[str], log: str) -> None:
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError(f"build step failed: {' '.join(cmd[:3])} ... (log: {log})")


def build_cuda(verbose: bool = True) -> str:
    import torch
    from torch.utils import cpp_extension
    os.makedirs(BUILD, exist_ok=True)
    cuda = _cuda_home()
    nvcc = os.path.join(cuda, "bin", "nvcc")
    objs = []
    jobs = []
    hdrs = _headers()
    for src in CUDA_SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        flags = [f for f in NVCC_FLAGS if not (f == "--use_fast_math" and src in PRECISE)]
        flags += os.environ.get("B200_NVCC_EXTRA", "").split()          # extra defines for A/B builds
        tag = _digest([path] + hdrs, " ".join(flags))
        obj = os.path.join(BUILD, f"{src}.{tag}.o")
        objs.append(obj)
        if not os.path.exists(obj):
            jobs.append(([nvcc] + flags + ["-I", CSRC, "-c", path, "-o", obj], os.path.join(BUILD, src + ".log")))
    bind_src = os.path.join(CSRC, "bindings.cpp")
    inc = cpp_extension.include_paths(device_type="cuda") if "device_type" in cpp_extension.include_paths.__code__.co_varnames \
        else cpp_extension.include_paths(cuda=True)
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=_C",
                 "-DTORCH_API_INCLUDE_EXTENSION_H", "-I", CSRC, "-I", sysconfig.get_paths()["include"],
                 "-I", os.path.join(cuda, "include")]
    for i in inc:
        cxx_flags += ["-isystem", i]
    tag = _digest([bind_src] + hdrs, " ".join(cxx_flags) + torch.__version__)
    bind_obj = os.path.join(BUILD, f"bindings.{tag}.o")
    if not os.path.exists(bind_obj):
        jobs.append((["g++"] + cxx_flags + ["-c", bind_src, "-o", bind_obj], os.path.join(BUILD, "bindings.log")))
    if verbose and jobs:
        print(f"[build] compiling {len(jobs)} translation unit(s) ...", flush=True)
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(lambda j: _run(*j), jobs))
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    out = os.path.join(HERE, "_C.so")
    link = ["g++", "-shared", "-o", out, bind_obj] + objs + [
        f"-L{torch_lib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
        f"-L{os.path.join(cuda, 'lib64')}", "-lcudart", f"-Wl,-rpath,{torch_lib}",
        f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}"]
    _run(link, os.path.join(BUILD, "link.log"))
    # objects of earlier source revisions are dead weight (hundreds of MB)
    keep = {os.path.basename(o) for o in objs} | {os.path.basename(bind_obj)}
    for f in os.listdir(BUILD):
        if f.endswith(".o") and f not in keep:
            os.remove(os.path.join(BUILD, f))
    if verbose:
        print(f"[build] {out}")
    return out


def build_host(verbose: bool = True) -> str:
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(CSRC, "host.cpp")
    out = os.path.join(HERE, "_host.so")
    tag = _digest([src], "host")
    stamp = os.path.join(BUILD, f"host.{tag}.stamp")
    if os.path.exists(out) and os.path.exists(stamp):
        return out
    _run(["g++", "-O3", "-march=x86-64-v2", "-std=c++17", "-fPIC", "-shared", "-pthread", src, "-o", out,
          "-l:libz.so.1"], os.path.join(BUILD, "host.log"))
    open(stamp, "w").close()
    if verbose:
        print(f"[build] {out}")
    return out


def build_all(verbose: bool = True) -> None:
    build_host(verbose)
    build_cuda(verbose)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--cuda", action="store_true")
    a = ap.parse_args()
    if a.host and not a.cuda:
        build_host()
    elif a.cuda and not a.host:
        build_cuda()
    else:
        build_all()
