"""In-tree build of the sm_90a (Hopper, H100) extension ``acco_b200/_C.so``.

Explicit ``nvcc`` / ``g++`` invocations (no JIT cache under ``~/.cache``: the built ``.so`` sits in the
tree, next to the package that loads it).  Every ``.cu`` is compiled with
``-gencode arch=compute_90a,code=sm_90a -lineinfo`` - sm_90a only, no fallback architectures.
Objects are cached in ``acco_b200/_build`` and rebuilt when a source or header is newer.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
import sysconfig
from typing import List

PKG = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "_build")
OUT = os.path.join(PKG, "_C.so")

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
              "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else (shutil.which("nvcc") or "nvcc")


def _newer(src_files: List[str], target: str) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_files)


def _run(cmd: List[str], log_path: str = None) -> None:
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log_path:
        with open(log_path, "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        raise RuntimeError(f"command failed ({p.returncode}): {' '.join(cmd)}\n{p.stdout[-4000:]}")


def cuda_sources() -> List[str]:
    return sorted(os.path.join(SRC, f) for f in os.listdir(SRC) if f.endswith(".cu"))


def build(verbose: bool = True, force: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(SRC, f) for f in os.listdir(SRC) if f.endswith((".cuh", ".h"))]
    cus = cuda_sources()
    cutlass_inc = []
    for root in sys.path:
        cand = os.path.join(root, "flashinfer", "data", "cutlass", "include")
        if os.path.isdir(cand):
            cutlass_inc = ["-I", cand]
            break
    jobs = []
    objs = []
    for cu in cus:
        o = os.path.join(OBJ, os.path.basename(cu)[:-3] + ".o")
        objs.append(o)
        if force or _newer([cu] + headers, o):
            jobs.append(([_nvcc()] + NVCC_ARCH + NVCC_FLAGS + ["-I", SRC] + cutlass_inc + ["-c", cu, "-o", o], o[:-2] + ".log"))
    inc = []
    cpp_jobs = []
    for name in sorted(f for f in os.listdir(SRC) if f.endswith(".cpp")):
        cpp = os.path.join(SRC, name)
        cpp_o = os.path.join(OBJ, name[:-4] + ".o")
        objs.append(cpp_o)
        if force or _newer([cpp] + headers, cpp_o):
            cpp_jobs.append((cpp, cpp_o))
    if cpp_jobs:
        for p in ce.include_paths(device_type="cuda") if "device_type" in ce.include_paths.__code__.co_varnames else ce.include_paths(cuda=True):
            inc += ["-I", p]
        inc += ["-I", sysconfig.get_paths()["include"]]
        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
        for cpp, cpp_o in cpp_jobs:
            jobs.append((["g++", "-O2", "-std=c++17", "-fPIC", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
                          f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-Wno-deprecated-declarations"] + inc + ["-c", cpp, "-o", cpp_o],
                         cpp_o[:-2] + ".log"))
    if jobs:
        if verbose:
            print(f"[acco_b200.build] compiling {len(jobs)} translation unit(s) for sm_90a ...", flush=True)
        with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(lambda j: _run(*j), jobs))
    if jobs or force or not os.path.exists(OUT):
        libs = []
        for p in ce.library_paths(device_type="cuda") if "device_type" in ce.library_paths.__code__.co_varnames else ce.library_paths(cuda=True):
            libs += ["-L", p, f"-Wl,-rpath,{p}"]
        cuda_lib = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "lib64")
        libs += ["-L", cuda_lib, f"-Wl,-rpath,{cuda_lib}"]
        tmp = OUT + ".tmp"
        _run(["g++", "-shared", "-o", tmp] + objs + libs + ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
                                                             "-ltorch_python", "-lcudart", "-lcuda"])
        os.replace(tmp, OUT)
        if verbose:
            print(f"[acco_b200.build] linked {OUT}", flush=True)
    return OUT


def ptxas_report() -> str:
    """Concatenated ``-Xptxas -v`` output of the last build (registers / spills / smem per kernel)."""
    out = []
    for f in sorted(os.listdir(OBJ)) if os.path.isdir(OBJ) else []:
        if f.endswith(".log"):
            out.append(f"==== {f}\n" + open(os.path.join(OBJ, f)).read())
    return "\n".join(out)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
