"""Stage blocks that do not fit in shared memory: the generic kernel's global-scratch variant (run on an H100 with -m gpu).

A shape whose stage-block buffers need more shared memory than a block may have -- a condensed QP of the chain-mass,
quadrotor or legged shape under full condensing or a coarse cond_N -- runs the generic kernel with those buffers in a per-QP slice
of a device scratch buffer, and the block condenser does the same with its scratch.  The tuning key "spill" = 1 forces the
variant on a shape that fits; there it must reproduce the on-chip kernel bit for bit, since it performs the same arithmetic in
the same order."""
import numpy as np
import pytest

from acados_b200 import problems as P
from acados_b200.binding import CuipmSolver, default_opts
from acados_b200.ocp_qp import OcpQpOptions, PackedBatch
from test_ocp_qp_mirror import random_ocp_qp
from test_oracle_vs_reference import CASES, LQ_CASES
from test_parity_gpu import _tol_default

pytestmark = pytest.mark.gpu


def _bits_equal(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def _assert_identical(r1, r2):
    (sol1, info1, stat1), (sol2, info2, stat2) = r1, r2
    for f in info1.dtype.names:
        assert _bits_equal(info1[f], info2[f]), f
    assert _bits_equal(sol1, sol2)
    assert _bits_equal(stat1, stat2)


def _solve(b, o, spill, warps=1, sol0=None):
    # fast = 0: every QP goes through the generic kernel, whichever throughput-kernel instance the shape has
    s = CuipmSolver(b.shape, b.nbatch)
    s.set_tuning("fast", 0)
    s.set_tuning("warps", warps)
    if spill:
        s.set_tuning("spill", 1)
    out = s.solve(b.qp, o, sol0=sol0, want_stat=True)
    return s, out


# ---- 1. the variant forced on shapes that fit: bit-identical to the on-chip kernel ----------------------------------------

FAMILIES = {
    **{n: (CASES[n], {}) for n in ("c1_mass_spring", "c2_chain_mass", "rand_box", "rand_general", "rand_soft", "rand_masked",
                                   "rand_x0_free", "unconstrained", "c5_sized", "rand_infeasible")},
    "lq_every_iteration": (CASES["rand_soft"], dict(lq_fact=2)),
    "lq_fallback": (LQ_CASES["infeasible_general"], dict(lq_fact=1)),
    "iterative_refinement": (CASES["rand_general"], dict(itref_corr_max=4, res_g_max=1e-12, res_b_max=1e-12, res_d_max=1e-12,
                                                         res_m_max=1e-12)),
    "iter_max_hit": (CASES["c2_chain_mass"], dict(iter_max=3)),
}


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("warps", [1, 2, 4])
def test_forced_variant_is_bit_identical(built, family, warps):
    make, kw = FAMILIES[family]
    b = make()
    o = default_opts(**kw)
    s0, r0 = _solve(b, o, spill=False, warps=warps)
    s1, r1 = _solve(b, o, spill=True, warps=warps)
    s0.close(); s1.close()
    _assert_identical(r0, r1)


@pytest.mark.parametrize("ws", [2, 3])
def test_forced_variant_warm_start(built, ws):
    b = CASES["rand_soft"]()
    s, (sol0, _, _) = _solve(b, default_opts(), spill=False)
    s.close()
    o = default_opts(warm_start=ws)
    s0, r0 = _solve(b, o, spill=False, sol0=sol0)
    s1, r1 = _solve(b, o, spill=True, sol0=sol0)
    s0.close(); s1.close()
    _assert_identical(r0, r1)


@pytest.mark.parametrize("name", ["c2_chain_mass", "rand_soft", "rand_masked", "rand_x0_free"])
@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("warps", [1, 4])
def test_forced_variant_sensitivities_and_getters(built, name, adjoint, warps):
    """cuipm_sens_* (forward and adjoint) and cuipm_get_ric after a solve with the variant forced: bit-identical."""
    b = CASES[name]()
    o = default_opts()
    seed = np.random.default_rng(17).standard_normal((b.nbatch, b.layout.sol_stride))
    out = []
    for spill in (False, True):
        s, _ = _solve(b, o, spill=spill, warps=warps)
        e = s.sens(seed, o, adjoint=adjoint)
        ric = []
        for q in (0, b.nbatch - 1):
            for k in range(b.shape.N + 1):
                nx, nu = b.shape.nx[k], b.shape.nu[k]
                ric += [s.get_ric(q, "Lr", k, (nu, nu)), s.get_ric(q, "P", k, (nx, nx)), s.get_ric(q, "p", k, (nx, 1)),
                        s.get_ric(q, "K", k, (nu, nx)), s.get_ric(q, "k", k, (nu, 1))]
        s.close()
        out.append((e, ric))
    assert _bits_equal(out[0][0], out[1][0])
    assert all(_bits_equal(x, y) for x, y in zip(out[0][1], out[1][1]))


def test_forced_variant_chunked_host_solve(built):
    """A host solve of 1024 QPs runs in 8 chunks on 8 streams at once: the scratch is indexed by QP, so the concurrent chunks
    never share a slice.  Bit-identical to the on-chip kernel and to one device-resident launch over the whole batch."""
    import torch
    b = P.chain_mass(1024, seed=4321)
    o = default_opts()
    s0, r0 = _solve(b, o, spill=False)
    s1, r1 = _solve(b, o, spill=True)
    s0.close()
    _assert_identical(r0, r1)
    d_qp = torch.from_numpy(b.qp).cuda()
    d_sol = torch.zeros((b.nbatch, b.layout.sol_stride), dtype=torch.float64, device="cuda")
    d_info = torch.zeros((b.nbatch, r1[1].dtype.itemsize // 8), dtype=torch.float64, device="cuda")
    s1.solve_device(b.nbatch, d_qp.data_ptr(), d_sol.data_ptr(), d_info.data_ptr(), o)
    assert _bits_equal(d_sol.cpu().numpy(), r1[0])
    assert d_info.cpu().numpy().tobytes() == r1[1].tobytes()
    s1.close()


# ---- 2. shapes the on-chip kernel cannot hold --------------------------------------------------------------------------

def _condensed(name, cond_N, nbatch, seed=7):
    from acados_b200.condensing import BlockCondenser
    from acados_b200.problems import Batch
    b = P.named_config(name, nbatch, seed=seed)
    bc = BlockCondenser(b.shape, cond_N)
    return b, bc, Batch(bc.cshape, bc.clay, bc.condense(b.qp), f"{name}_cond{cond_N}")


def _smem_kb(shape):
    """The planner's shared-memory formula (cuipm_plan.h) restated: kB the on-chip kernel would need."""
    e = lambda n: (n + 1) & ~1
    N = shape.N
    n = [shape.nx[k] + shape.nu[k] for k in range(N + 1)]
    nx1 = [shape.nx[k + 1] if k < N else 0 for k in range(N + 1)]
    nmax, ngmax, nsmax = max(n), max(shape.ng), max(shape.ns)
    nxmax = max(max(shape.nx[k], nx1[k]) for k in range(N + 1))
    nbgmax = max(shape.nb[k] + shape.ng[k] for k in range(N + 1))
    ncmax = max(2 * (shape.nb[k] + shape.ng[k] + shape.ns[k]) for k in range(N + 1))
    nvsmax = max(n[k] + 2 * shape.ns[k] for k in range(N + 1))
    M = e((nmax + 2) * nmax + 8)
    AL = e(max((nmax + 2) * (nxmax + ngmax), e(nmax) + e(nxmax) + 4 * e(ncmax)) + 8)
    Cb = 2 * e((nmax + 2) * ngmax) + 8 if ngmax > 0 else 0
    nvs, nxe, nc, nbg, nn, ns2 = e(nvsmax), e(nxmax), e(ncmax), e(nbgmax), e(nmax + 1), e(2 * nsmax)
    V = max(2 * nvs + 3 * nxe + 4 * nc + 2 * nbg, 2 * nvs + 5 * nxe + 4 * nc + 2 * ns2 + nbg, 2 * nc + 2 * nbg + 3 * nn + 2 * ns2 + 16,
            nvs + 2 * nc + 2 * nbg + 2 * ns2 + 3 * nxe, nvs + nc + e(ngmax)) + 8
    return 8 * (M + AL + Cb + V) / 1024


@pytest.mark.parametrize("name,cond_N", [("c2", 1), ("c2", 2), ("c4", 1), ("c4", 3), ("c5", 1), ("c5", 5)])
def test_refused_shapes_match_the_oracle(built, name, cond_N):
    from oracle import oracle_binding as ob
    import torch
    _, _, cb = _condensed(name, cond_N, 8)
    # the on-chip kernel cannot hold these blocks: more than the device's whole opt-in limit, before its static shared memory
    assert _smem_kb(cb.shape) * 1024 > torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    o = default_opts()
    s = CuipmSolver(cb.shape, cb.nbatch)
    sol, info = s.solve(cb.qp, o)
    s.close()
    osol, oinfo = ob.oracle_solve(cb, o)
    assert np.array_equal(info["status"], oinfo["status"]), (info["status"], oinfo["status"])
    assert np.array_equal(info["iter"], oinfo["iter"]), (info["iter"], oinfo["iter"])
    # the switch to the LQ refactorisation is triggered by round-off (see test_oracle_vs_reference): +-1 iteration
    assert np.max(np.abs(info["lq_count"] - oinfo["lq_count"])) <= 1
    du = np.max(np.abs(cb.layout.u_traj(sol) - cb.layout.u_traj(osol)))
    assert du <= _tol_default(name), du


def test_vector_area_beyond_shared_memory_is_refused(built):
    """What remains impossible: the vector area alone above the shared memory a block may have (here 4000 general constraints on
    one stage)."""
    sh = P.random_shape(1, 2, 2, ng=4000)
    with pytest.raises(RuntimeError, match="vectors alone"):
        CuipmSolver(sh, 1)


TIGHT = dict(tol_stat=1e-10, tol_eq=1e-10, tol_ineq=1e-10, tol_comp=1e-10)
SIZES = {"c2": dict(N=40, nx=21, nu=3), "c4": dict(N=50, nx=12, nu=4), "c5": dict(N=30, nx=48, nu=12)}


def _front_end_qps(name, n, seed=3):
    rng = np.random.default_rng(seed)
    return [random_ocp_qp(rng, soft=True, general=True, **SIZES[name]) for _ in range(n)]


@pytest.mark.parametrize("name,cond_N", [("c2", 1), ("c2", 2), ("c4", 1), ("c4", 3), ("c5", 1), ("c5", 5)])
def test_front_end_condensing_matches_uncondensed(built, name, cond_N):
    """OcpQpBatchSolver with FULL_CONDENSING_HPIPM (cond_N = 1) or a coarse cond_N: the solution of the uncondensed solve of the
    same QPs, both driven to 1e-10 (two different IPM trajectories: converged points are compared)."""
    from acados_b200.ocp_qp import OcpQpBatchSolver
    qps = _front_end_qps(name, 8)
    N = SIZES[name]["N"]
    opts = OcpQpOptions(qp_solver="FULL_CONDENSING_HPIPM", **TIGHT) if cond_N == 1 else OcpQpOptions(cond_N=cond_N, **TIGHT)
    a = OcpQpBatchSolver(qps, opts)
    b = OcpQpBatchSolver(qps, OcpQpOptions(**TIGHT))
    assert a.opts.cond_N == cond_N
    # a random instance may have no solution (the oracle stops it at the minimal step length, condensed or not): the
    # instances the uncondensed solve converges on are compared
    sa, sb = a.solve(), b.solve()
    ok = sb == 0
    assert ok.sum() >= 6 and (sa[ok] == 0).all(), (sa, sb)
    for k in range(N + 1):
        assert np.max(np.abs(a.get(k, "u") - b.get(k, "u"))[ok], initial=0.0) <= 1e-7
        assert np.max(np.abs(a.get(k, "x") - b.get(k, "x"))[ok]) <= 1e-7
    a.close(); b.close()


@pytest.mark.parametrize("name,cond_N", [("c2", 1), ("c4", 3), ("c5", 5)])
def test_xcond_chain_on_refused_shapes(built, name, cond_N):
    """cuipm_xcond_* (the object behind the front end's device path and the plugin's batched xcond entry) on shapes whose condensed
    stage blocks leave shared memory: condense_lhs then condense_rhs_and_solve on the same records reproduces the one pass bit for
    bit, solutions, summaries and statistics."""
    from acados_b200.binding import CuipmXcond
    qps = _front_end_qps(name, 6, seed=7)
    o = OcpQpOptions().to_cuipm()
    full = PackedBatch(qps, eliminate=False)
    xc = CuipmXcond(full.shape, [int(i) for i in qps[0].idxe[0]], cond_N, len(qps))
    sol, info, stat = xc.solve(full.qp, o, want_stat=True)
    assert (info["status"] == 0).sum() >= 4           # (a random instance may be infeasible)
    xc.condense_lhs(full.qp)
    sol2, info2, stat2 = xc.condense_rhs_and_solve(full.qp, o, want_stat=True)
    assert sol2.tobytes() == sol.tobytes() and info2.tobytes() == info.tobytes() and stat2.tobytes() == stat.tobytes()
    xc.close()


def test_device_condensing_of_the_legged_shape_matches_numpy(built):
    """c5 (nx=48, nu=12, N=30) fully condensed: 277 KB of condenser scratch per QP, in global memory.  cuipm_condense_device and
    cuipm_expand_device against acados_b200/condensing.py, and the lhs / rhs split against the one-pass condensing."""
    import torch
    from acados_b200.binding import CuipmCondenser
    b, bc, cb = _condensed("c5", 1, 8)
    dc = CuipmCondenser(b.shape, 1)
    q_np = cb.qp
    d_qp = torch.from_numpy(b.qp).cuda()
    d_out = torch.full((b.nbatch, bc.clay.qp_stride), 7.0, dtype=torch.float64, device="cuda")
    dc.condense(b.nbatch, d_qp.data_ptr(), d_out.data_ptr())
    torch.cuda.synchronize()
    assert np.max(np.abs(d_out.cpu().numpy() - q_np)) <= 1e-12 * max(1.0, np.max(np.abs(q_np)))
    d_split = torch.full_like(d_out, 7.0)
    dc.condense_lhs(b.nbatch, d_qp.data_ptr(), d_split.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(d_split, d_out)
    dc.condense_rhs(b.nbatch, d_qp.data_ptr(), d_split.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(d_split, d_out)
    s = CuipmSolver(cb.shape, cb.nbatch)
    s2, info = s.solve(np.ascontiguousarray(d_out.cpu().numpy()), default_opts())
    s.close()
    assert (info["status"] == 0).all()
    e_np = bc.expand(b.qp, s2)
    d_s2 = torch.from_numpy(s2).cuda()
    d_sol = torch.full((b.nbatch, b.layout.sol_stride), 7.0, dtype=torch.float64, device="cuda")
    dc.expand(b.nbatch, d_qp.data_ptr(), d_s2.data_ptr(), d_sol.data_ptr())
    torch.cuda.synchronize()
    assert np.max(np.abs(d_sol.cpu().numpy() - e_np)) <= 1e-11 * max(1.0, np.max(np.abs(e_np)))
    dc.close()
