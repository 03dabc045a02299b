"""The throughput kernel stages the Hessian (residual sweep) and the state block Lxx of the next stage's factor (forward sweeps) as
packed lower triangles, n (n + 1) / 2 doubles, in place of full n x n blocks, for stage blocks of up to 32 rows (fast_packed in
acados_b200/csrc/cuipm_device.h); larger blocks keep the full ones.

The staged bytes per QP-iteration on the benchmark's shape (chain-mass nx=21 nu=3 N=40, default options, eight lanes per QP,
iteration-sliced scheduling) are counted on a build of the host emulation, made in a temporary directory, that defines the kernel
body's FK_COUNT_STAGED hook: 1888 kB with the full blocks, 1646 kB packed (residual sweep 508 -> 411 kB, forward sweeps
836 -> 702 kB).  The packed index maps differ by stage (stage 0: n = nu, interior: n = nx + nu, stage N: n = nx) and their
reads by lane mapping: the solutions of the iteration-sliced schedule are held to the oracle on packed shapes that run with
two, eight and 32 lanes per QP, with soft and masked constraints, and on the legged shape, which keeps the full blocks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from acados_b200 import problems
from acados_b200.binding import default_opts
from oracle import oracle_binding as ob

KB_PER_QP_ITERATION_MAX = 1700.0

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
    d = tmp_path_factory.mktemp("fast_emul_counting_packed")
    src, lib = d / "fast_emul_counting.cpp", d / "libfast_emul_counting.so"
    src.write_text(COUNTING_EMUL)
    csrc = os.path.join(ROOT, "acados_b200", "csrc")
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "include"), "-I" + csrc,
                    "-I" + os.path.join(ROOT, "oracle"), "-o", str(lib), str(src), os.path.join(csrc, "cuipm_host.cpp")], check=True)
    return str(lib)


def test_packed_blocks_staged_bytes(counting_emul, monkeypatch):
    monkeypatch.setattr(ob, "FAST_EMUL_LIB", counting_emul)
    lib = ob._load(counting_emul)
    lib.fast_emul_take_staged_bytes.restype = C.c_ulonglong
    b = problems.chain_mass(64, seed=1234)
    lib.fast_emul_take_staged_bytes()
    sol, info, redo = ob.fast_emul_solve(b, default_opts(), g=8, rr=True)
    staged = lib.fast_emul_take_staged_bytes()
    assert len(redo) == 0 and (info["status"] == 0).all()
    kb = staged / float(info["iter"].sum()) / 1000.0
    assert kb <= KB_PER_QP_ITERATION_MAX, kb


def _legged():
    return problems.random_qp(problems.random_shape(4, 48, 12, nbx=12, ns=12), 2, seed=3, umax=0.5, xmax=1.0, x0_scale=1.0)


def _soft_masked():
    return problems.random_qp(problems.random_shape(8, 8, 3, nbx=4, ns=2), 8, seed=5, mask_frac=0.3)


@pytest.mark.parametrize("shape,g,tol_u,max_redo", [
    ("pendulum_g2", 2, 1e-10, 0),         # nx=4 nu=1
    ("soft_masked_g8", 8, 1e-10, 3),      # nx=8 nu=3, soft and masked bounds
    ("chain_mass_g32", 32, 1e-10, 0),     # nx=21 nu=3, one QP per warp
    ("legged_g32", 32, 1e-9, 0),          # nx=48 nu=12: full blocks, tensor-core factorisation
])
def test_packed_blocks_iteration_sliced_against_oracle(shape, g, tol_u, max_redo):
    b = {"pendulum_g2": lambda: problems.named_config("c3", 16), "soft_masked_g8": _soft_masked,
         "chain_mass_g32": lambda: problems.chain_mass(3, N=12, seed=6), "legged_g32": _legged}[shape]()
    o = default_opts()
    sol, info, redo = ob.fast_emul_solve(b, o, g=g, rr=True)
    osol, oinfo = ob.oracle_solve(b, o)
    keep = np.setdiff1d(np.arange(b.nbatch), redo)
    assert len(redo) <= max_redo, redo
    assert (info["iter"][keep] == oinfo["iter"][keep]).all()
    assert (info["status"][keep] == oinfo["status"][keep]).all()
    lay = b.layout
    du = np.max(np.abs(lay.u_traj(sol) - lay.u_traj(osol))[keep])
    assert du <= tol_u, du
