"""In-tree build of libcuipm.so (CUDA kernels for sm_90a + the C ABI of include/cuipm.h).

``python -m acados_b200.csrc.build [--force] [--verbose]``; also called by ``__graft_entry__.build()``.
nvcc cross-compiles without a GPU.  Objects are cached under csrc/build/ keyed by source mtime.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "libcuipm.so")
SOURCES = ["cuipm_kernel.cu", "cuipm_fast.cu", "cuipm_api.cu", "cuipm_reduce.cu", "cuipm_condense.cu", "cuipm_xcond.cu", "cuipm_assemble.cu", "cuipm_host.cpp"]
HEADERS = ["cuipm_device.h", "cuipm_internal.h", "cuipm_plan.h", "cuipm_fast_core.h", "cuipm_condense_core.h", "cuipm_condense_plan.h", "cuipm_assemble_core.h", os.path.join(ROOT, "include", "cuipm.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(ROOT, "include"), "-I" + HERE]
if os.environ.get("CUIPM_PROFILE"):
    FLAGS.append("-DCUIPM_PROFILE")   # per-pass cycle counters into the last row of the stat table (development)
# development variants: CUIPM_DEFS="-DX=1 -DY" adds defines, CUIPM_VARIANT=name builds csrc/variants/libcuipm_<name>.so
# (load it with CUIPM_LIB=<path>, see binding.py) next to the product library
FLAGS += os.environ.get("CUIPM_DEFS", "").split()
VARIANT = os.environ.get("CUIPM_VARIANT", "")
if VARIANT:
    OUT = os.path.join(HERE, "variants", f"libcuipm_{VARIANT}.so")


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    bdir = os.path.join(HERE, "build", VARIANT) if VARIANT else os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    hdrs = [h if os.path.isabs(h) else os.path.join(HERE, h) for h in HEADERS]
    objs = []
    procs = []
    for src in SOURCES:
        sp = os.path.join(HERE, src)
        obj = os.path.join(bdir, os.path.splitext(src)[0] + ".o")
        objs.append(obj)
        if force or _newer(obj, [sp] + hdrs):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(out)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _newer(OUT, objs):
        cmd = [NVCC, "-shared", "-cudart", "static", "-o", OUT] + objs
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout)
            raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
