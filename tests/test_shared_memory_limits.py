"""Shared-memory limits taken from the device (run on an H100 with -m gpu).

Whether a kernel's buffers fit in shared memory is decided against what the device lets a block request: its opt-in limit less the
kernel's own static shared memory.  And the dynamic shared-memory attribute belongs to a kernel, not to one solver object, so every
object sets it before each launch: objects of other shapes in the same process must not change what an earlier one can launch."""
import numpy as np
import pytest

from acados_b200 import problems as P
from acados_b200.binding import CuipmSolver, default_opts
from acados_b200.ocp_qp import OcpQpBatchSolver, OcpQpOptions, PackedBatch
from test_large_stage_blocks import _smem_kb
from test_ocp_qp_mirror import random_ocp_qp
from test_parity_gpu import _tol_default

pytestmark = pytest.mark.gpu


def test_buffers_just_below_the_dynamic_limit_run_from_global_scratch(built):
    """N = 3, nx = 4, nu = 36 with input boxes, 196 general constraints: the generic kernel's carve is 231 904 B, below the
    232 448 B an H100 block may have, but the kernel's static shared memory (1248 B at one warp per QP, 1312 B at two and four)
    comes on top of it.  The shape must run the global-scratch variant and match the oracle."""
    from oracle import oracle_binding as ob
    sh = P.random_shape(3, 4, 36, ng=196)
    assert _smem_kb(sh) * 1024 == 231904
    b = P.random_qp(sh, 8, seed=5)
    o = default_opts()
    s = CuipmSolver(b.shape, b.nbatch)
    sol, info = s.solve(b.qp, o)
    s.close()
    osol, oinfo = ob.oracle_solve(b, o)
    assert np.array_equal(info["status"], oinfo["status"]), (info["status"], oinfo["status"])
    assert np.array_equal(info["iter"], oinfo["iter"]), (info["iter"], oinfo["iter"])
    du = np.max(np.abs(b.layout.u_traj(sol) - b.layout.u_traj(osol)))
    assert du <= _tol_default("rand_general"), du


def _condenser_scratch_bytes(shape, cond_N):
    """scratch_doubles of the block condenser (cuipm_condense_core.h, cuipm_condense_plan.h) restated, in bytes."""
    N = shape.N
    n1, r1 = divmod(N, cond_N)
    k, n2max = 0, 0
    for blk in range(cond_N):
        m = n1 + 1 if blk < r1 else n1
        n2max = max(n2max, sum(shape.nu[k:k + m]) + shape.nx[k])
        k += m
    nxmax = max(max(shape.nx[j], shape.nu[j]) for j in range(N + 1))
    return 8 * (2 * nxmax * n2max + 4 * nxmax + 2 * n2max + 16)


def _legged_qps(n=4, seed=11):
    rng = np.random.default_rng(seed)
    return [random_ocp_qp(rng, soft=True, general=True, N=30, nx=48, nu=12) for _ in range(n)]


def _front_end_result(bs):
    return [np.copy(bs.get(k, f)) for k in range(bs.N + 1) for f in ("u", "x", "lam")] + [bs.info.copy(), bs.stat.copy()]


def test_condensed_front_end_solvers_of_two_shapes(built):
    """The legged shape at cond_N = 5 keeps 94 KB of condenser scratch on chip (above the 48 KB a launch gets without the
    attribute); at cond_N = 1 it needs 277 KB, in global memory.  Creating and using the second solver (a second cuipm_xcond
    chain) leaves the first one's solve bit-identical."""
    import torch
    qps = _legged_qps()
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    reduced = PackedBatch(qps).shape
    a = OcpQpBatchSolver(qps, OcpQpOptions(cond_N=5))
    scratch_a = _condenser_scratch_bytes(reduced, 5)
    # above the 48 KB a launch may have without the attribute, and on chip: the condenser compares its scratch with the opt-in
    # limit less its kernels' static shared memory, which is 0 B for condense_kernel and expand_kernel (-Xptxas -v); the 16 KB
    # margin only keeps the assertion independent of that figure
    assert 48 * 1024 < scratch_a < optin - 16 * 1024, scratch_a
    a.solve()
    ref = _front_end_result(a)
    b = OcpQpBatchSolver(qps, OcpQpOptions(qp_solver="FULL_CONDENSING_HPIPM"))
    assert _condenser_scratch_bytes(reduced, 1) > optin
    b.solve()
    a.solve()
    assert all(np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes() for x, y in zip(ref, _front_end_result(a)))
    a.close(); b.close()
