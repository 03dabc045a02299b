"""Bytes the throughput kernel stages into shared memory (bulk and 16-byte asynchronous copies) per QP-iteration, counted on the
host emulation of its body on the benchmark's shape: chain-mass nx=21 nu=3 N=40, default options, eight lanes per QP,
iteration-sliced scheduling.  The sweeps of this kernel stream every stage input from global memory, so these bytes are what
its run time follows on the H100; the bound keeps a change from bringing a stream back unnoticed.  The forward sweeps used to
stage the Hessian of every stage for the stationarity rows of the residual of the linear system (2263 kB per QP-iteration);
the residual sweep, which holds the Hessian anyway, now forms those rows (1888 kB).

The count comes from a build of oracle/fast_emul.cpp, made in a temporary directory, that defines the kernel body's
FK_COUNT_STAGED hook (a no-op in every other build)."""
import ctypes as C
import os
import subprocess

import pytest

from acados_b200 import problems
from acados_b200.binding import default_opts
from oracle import oracle_binding as ob

KB_PER_QP_ITERATION_MAX = 1900.0

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTING_EMUL = r"""
static unsigned long long g_staged = 0;
#define FK_COUNT_STAGED(bytes) (g_staged += (bytes))
#include "fast_emul.cpp"
// bytes staged since the last call (and resets the count)
extern "C" unsigned long long fast_emul_take_staged_bytes()
{
    const unsigned long long b = g_staged;
    g_staged = 0;
    return b;
}
"""


@pytest.fixture(scope="module")
def counting_emul(tmp_path_factory):
    d = tmp_path_factory.mktemp("fast_emul_counting")
    src, lib = d / "fast_emul_counting.cpp", d / "libfast_emul_counting.so"
    src.write_text(COUNTING_EMUL)
    csrc = os.path.join(ROOT, "acados_b200", "csrc")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"), "-I" + csrc,
                    "-I" + os.path.join(ROOT, "oracle"), "-o", str(lib), str(src), os.path.join(csrc, "cuipm_host.cpp")], check=True)
    return str(lib)


def test_staged_bytes_per_qp_iteration(counting_emul, monkeypatch):
    monkeypatch.setattr(ob, "FAST_EMUL_LIB", counting_emul)
    lib = ob._load(counting_emul)
    lib.fast_emul_take_staged_bytes.restype = C.c_ulonglong
    b = problems.chain_mass(64, seed=1234)
    lib.fast_emul_take_staged_bytes()
    sol, info, redo = ob.fast_emul_solve(b, default_opts(), g=8, rr=True)
    staged = lib.fast_emul_take_staged_bytes()
    assert len(redo) == 0 and (info["status"] == 0).all()
    assert staged > 0          # the kernel body reports its copies
    kb = staged / float(info["iter"].sum()) / 1000.0
    assert kb <= KB_PER_QP_ITERATION_MAX, kb
