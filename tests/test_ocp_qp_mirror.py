"""Host-side mirror of the reference's Python QP interface (acados_b200/ocp_qp.py): field handling, the stage-0
equality elimination / restore around the solve, record packing.

CPU part: the packed records are solved by the oracle (the checker) and the restored solution is checked (a) against
the reference's own golden multipliers for its two QP fixtures at the reference's own bar (atol 1e-5 on lam and pi,
examples/acados_python/tests/qp_test/test_ocpqp_solver.py:45-57), (b) through the KKT conditions of the ORIGINAL,
unreduced QP.  GPU part: the same through OcpQpSolver / OcpQpBatchSolver, i.e. the CUDA path."""
import json
import os

import numpy as np
import pytest

from acados_b200.binding import default_opts
from acados_b200.ocp_qp import OcpQp, OcpQpOptions, PackedBatch
from acados_b200.problems import Batch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["nonuniform_pendulum", "one_sided_test"]


def _load(name):
    g = json.load(open(os.path.join(GOLD, f"refqp_{name}.json")))
    return g, OcpQp.from_json(json_data=dict(g["qp"]))


def _unique_duals(lam, hard):
    lam = lam.copy()
    u = lam[hard:2 * hard] - lam[:hard]
    lam[:hard], lam[hard:2 * hard] = np.maximum(0.0, -u), np.maximum(0.0, u)
    return lam


def _check_golden(g, qp, res, iters, u_traj):
    for k in range(qp.N + 1):
        lam = res["lam"][k][0]
        if k == 0:
            lam = _unique_duals(lam, int(qp.dims.nb[0] + qp.dims.ng[0]))
        exp = np.asarray(g["exp_lam"][k], dtype=float)
        assert lam.shape == exp.shape and np.allclose(lam, exp, atol=1e-5), (k, lam, exp)
    for k in range(qp.N):
        assert np.allclose(res["pi"][k][0], np.asarray(g["exp_pi"][k]), atol=1e-5), k
    assert iters == g["ref_iter"]
    assert np.max(np.abs(u_traj - np.asarray(g["ref_u"]))) <= 1e-10          # parity with HPIPM itself on the inputs


def random_ocp_qp(rng, N=6, nx=4, nu=2, soft=True, general=True):
    """A QP in the user's form: x0 pinned through stage-0 state bounds marked as equalities."""
    qp = OcpQp(N)
    A = np.eye(nx) + 0.1 * rng.standard_normal((nx, nx)) / np.sqrt(nx)
    for k in range(N + 1):
        nuk = nu if k < N else 0
        W = rng.standard_normal((nx, nx))
        qp.set("Q", k, np.eye(nx) + 0.1 * W @ W.T / nx)
        qp.set("R", k, 0.5 * np.eye(nuk))
        qp.set("S", k, 0.01 * rng.standard_normal((nuk, nx)))
        qp.set("q", k, 0.1 * rng.standard_normal(nx))
        qp.set("r", k, 0.1 * rng.standard_normal(nuk))
        if k < N:
            qp.set("A", k, A)
            qp.set("B", k, rng.standard_normal((nx, nuk)) / np.sqrt(nx))
            qp.set("b", k, 0.05 * rng.standard_normal(nx))
        if k == 0:
            x0 = 0.3 * rng.standard_normal(nx)
            qp.set("idxb", 0, list(range(nuk + nx)))
            qp.set("lbu", 0, -0.4 * np.ones(nuk)); qp.set("ubu", 0, 0.4 * np.ones(nuk))
            qp.set("lbx", 0, x0); qp.set("ubx", 0, x0)
            qp.set("idxe", 0, list(range(nuk, nuk + nx)))
        else:
            nbx = 2
            qp.set("idxb", k, list(range(nuk)) + [nuk, nuk + 1])
            qp.set("lbu", k, -0.4 * np.ones(nuk)); qp.set("ubu", k, 0.4 * np.ones(nuk))
            xb = 0.25 if soft else 1.5
            qp.set("lbx", k, -xb * np.ones(nbx)); qp.set("ubx", k, xb * np.ones(nbx))
            if soft:
                qp.set("idxs_rev", k, [-1] * nuk + [0, 1] + ([-1] if general else []))
                for f, v in (("zl", 1.0), ("zu", 1.0), ("Zl", 10.0), ("Zu", 10.0), ("lls", 0.0), ("lus", 0.0)):
                    qp.set(f, k, v * np.ones(2))
        if general:
            qp.set("C", k, rng.standard_normal((1, nx)))
            qp.set("D", k, rng.standard_normal((1, nuk)))
            qp.set("lg", k, [-1.0]); qp.set("ug", k, [1.0])
    qp.make_consistent()
    return qp


def kkt_residuals(qp, res, q=0):
    """Inf-norms of (stationarity, dynamics, primal feasibility of hard bounds, complementarity) of the ORIGINAL QP."""
    N = qp.N
    stat = dyn = feas = comp = 0.0
    for k in range(N + 1):
        nu, nx, nb, ng, ns = (int(getattr(qp.dims, f)[k]) for f in ("nu", "nx", "nb", "ng", "ns"))
        u, x = res["u"][k][q], res["x"][k][q]
        v = np.concatenate([u, x])
        lam = res["lam"][k][q]
        H = qp.get_hessian_block(k)[:nu + nx, :nu + nx]
        g = np.concatenate([qp.r[k], qp.q[k]]) + H @ v
        if k < N:
            g += np.concatenate([qp.B[k].T, qp.A[k].T]) @ res["pi"][k][q]
            dyn = max(dyn, np.max(np.abs(qp.A[k] @ x + qp.B[k] @ u + qp.b[k] - res["x"][k + 1][q])))
        if k > 0:
            g[nu:] -= res["pi"][k - 1][q]
        dl = lam[nb + ng:2 * (nb + ng)] - lam[:nb + ng]
        np.add.at(g, np.asarray(qp.idxb[k], dtype=int), dl[:nb])
        if ng:
            g += np.concatenate([qp.D[k].T, qp.C[k].T]) @ dl[nb:]
        stat = max(stat, np.max(np.abs(g)))
        lb = np.concatenate([qp.lbu[k], qp.lbx[k]]); ub = np.concatenate([qp.ubu[k], qp.ubx[k]])
        val = np.concatenate([v[np.asarray(qp.idxb[k], dtype=int)], (qp.C[k] @ x + qp.D[k] @ u) if ng else np.zeros(0)])
        lo, hi = np.concatenate([lb, qp.lg[k]]), np.concatenate([ub, qp.ug[k]])
        sl = np.zeros(nb + ng); su = np.zeros(nb + ng)
        rev = np.asarray(qp.idxs_rev[k], dtype=int)
        if ns:
            sl[rev >= 0] = res["sl"][k][q][rev[rev >= 0]]
            su[rev >= 0] = res["su"][k][q][rev[rev >= 0]]
        feas = max(feas, np.max(np.maximum(lo - val - sl, 0.0), initial=0.0), np.max(np.maximum(val - su - hi, 0.0), initial=0.0))
        comp = max(comp, np.max(np.abs(lam[:nb + ng] * (val + sl - lo)), initial=0.0), np.max(np.abs(lam[nb + ng:2 * (nb + ng)] * (hi - val + su)), initial=0.0))
    return stat, dyn, feas, comp


def _oracle_solve(p, **kw):
    from oracle import oracle_binding as ob
    b = Batch(p.shape, p.layout, p.qp, "mirror")
    o = default_opts(**kw)
    sol, info = ob.oracle_solve(b, o)
    return sol, info, o


@pytest.mark.parametrize("name", NAMES)
def test_reference_fixture_through_the_mirror_cpu(built, name):
    g, qp = _load(name)
    assert qp.dims.nbxe[0] == qp.dims.nx[0]                      # x0 arrives as a stage-0 equality, as the user writes it
    p = PackedBatch([qp])
    assert p.shape.nx[0] == 0 and p.shape.nb[0] == qp.dims.nbu[0]
    sol, info, o = _oracle_solve(p, iter_max=500)
    assert info["status"][0] == 0
    res = p.unpack(sol, o.lam_min, o.t_min)
    _check_golden(g, qp, res, int(info["iter"][0]), p.layout.u_traj(sol)[0])


@pytest.mark.parametrize("soft,general", [(False, False), (True, False), (True, True)])
def test_elimination_and_restore_satisfy_the_original_kkt(built, soft, general):
    rng = np.random.default_rng(5)
    qps = [random_ocp_qp(rng, soft=soft, general=general) for _ in range(4)]
    p = PackedBatch(qps)
    sol, info, o = _oracle_solve(p, res_g_max=1e-10, res_b_max=1e-10, res_d_max=1e-10, res_m_max=1e-10)
    assert (info["status"] == 0).all()
    res = p.unpack(sol, o.lam_min, o.t_min)
    for i, qp in enumerate(qps):
        assert np.allclose(res["x"][0][i], qp.lbx[0])                                  # x0 restored
        stat, dyn, feas, comp = kkt_residuals(qp, res, i)
        assert stat <= 1e-8 and dyn <= 1e-9 and feas <= 1e-8 and comp <= 1e-7, (stat, dyn, feas, comp)
        lam0 = res["lam"][0][i]
        assert (lam0 >= 0).all()


def test_partial_elimination(built):
    """idxe marking only some stage-0 states: the others stay optimisation variables with their own bounds."""
    rng = np.random.default_rng(9)
    qp = random_ocp_qp(rng, soft=False, general=False)
    nu = int(qp.dims.nu[0])
    qp.set("idxe", 0, [nu, nu + 2])
    lbx, ubx = qp.lbx[0].copy(), qp.ubx[0].copy()
    lbx[[1, 3]] -= 0.3; ubx[[1, 3]] += 0.3
    qp.set("lbx", 0, lbx); qp.set("ubx", 0, ubx)
    p = PackedBatch([qp])
    assert p.shape.nx[0] == 2 and p.shape.nb[0] == nu + 2
    sol, info, o = _oracle_solve(p, res_g_max=1e-10, res_b_max=1e-10, res_d_max=1e-10, res_m_max=1e-10)
    res = p.unpack(sol, o.lam_min, o.t_min)
    stat, dyn, feas, comp = kkt_residuals(qp, res, 0)
    assert info["status"][0] == 0 and stat <= 1e-8 and dyn <= 1e-9 and feas <= 1e-8 and comp <= 1e-7


def test_field_handling_mirrors_the_reference():
    qp = OcpQp(3)
    with pytest.raises(ValueError):
        qp.set("A", 3, np.eye(2))            # no dynamics at the terminal stage
    with pytest.raises(ValueError):
        qp.set("Q", 4, np.eye(2))            # stage out of bounds
    with pytest.raises(ValueError):
        qp.set("nonsense", 0, np.eye(2))
    rng = np.random.default_rng(1)
    a = random_ocp_qp(rng)
    b = OcpQp.from_dict(json.loads(json.dumps(a.to_dict())))
    pa, pb = PackedBatch([a]), PackedBatch([b])
    assert np.array_equal(pa.qp, pb.qp) and pa.shape.idxb == pb.shape.idxb
    assert a.has_slacks() and not a.has_masks()
    with pytest.raises(ValueError):
        OcpQp.from_dict({"Q_0": np.eye(2), "Q_01": np.eye(2)})      # inconsistent zero padding
    with pytest.raises(ValueError):
        OcpQpOptions(qp_solver="FULL_CONDENSING_DAQP").make_consistent(3)
    c = random_ocp_qp(rng, nx=5)
    with pytest.raises(ValueError):
        PackedBatch([a, c])                  # a batch shares one structure


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_reference_fixture_through_the_mirror_gpu(built, name):
    """The reference's tests/qp_test/test_ocpqp_solver.py, run against this backend."""
    from acados_b200.ocp_qp import OcpQpSolver
    g, qp = _load(name)
    opts = OcpQpOptions()
    opts.iter_max = 500
    solver = OcpQpSolver(qp, opts=opts)
    status = solver.solve()
    assert status == 0
    it = solver.get_iterate()
    for k in range(qp.N + 1):
        exp = np.asarray(g["exp_lam"][k], dtype=float)
        assert np.allclose(it["lam"][k], exp, atol=1e-5), k
    for k in range(qp.N):
        assert np.allclose(it["pi"][k], np.asarray(g["exp_pi"][k]), atol=1e-5)
    assert solver.get_stats("iter") == g["ref_iter"]
    u = np.concatenate([it["u"][k] for k in range(qp.N + 1)])
    assert np.max(np.abs(u - np.asarray(g["ref_u"]))) <= 1e-10
    assert np.isfinite(solver.get_cost()) and solver.get_stats("statistics").shape == (g["ref_iter"] + 1, 20)
    solver.close()


@pytest.mark.gpu
def test_batch_solver_gpu(built):
    from acados_b200.ocp_qp import OcpQpBatchSolver
    rng = np.random.default_rng(5)
    qps = [random_ocp_qp(rng) for _ in range(16)]
    bs = OcpQpBatchSolver(qps)                     # elimination + restore on the device
    status = bs.solve()
    assert (status == 0).all()
    bh = OcpQpBatchSolver(qps, device_reduce=False)    # the same on the host: identical solve, identical restored solution
    assert (bh.solve() == 0).all() and np.array_equal(bh.get_stats("iter"), bs.get_stats("iter"))
    for k in range(bs.N + 1):
        # the reduced records differ in the last bit (summation order of the x0 terms); the IPM amplifies that to ~1e-11
        for f in ("u", "x", "sl", "su"):
            assert np.allclose(bs.get(k, f), bh.get(k, f), rtol=0, atol=1e-9), (k, f)
        for f in ("lam", "t"):
            assert np.allclose(bs.get(k, f), bh.get(k, f), rtol=1e-6, atol=1e-8), (k, f)
    bh.close()
    osol, oinfo, o = _oracle_solve(PackedBatch(qps))
    assert np.array_equal(bs.get_stats("iter"), oinfo["iter"])
    ores = PackedBatch(qps).unpack(osol, o.lam_min, o.t_min)
    for k in range(bs.N + 1):
        assert np.max(np.abs(bs.get(k, "u") - ores["u"][k]), initial=0.0) <= 1e-9
        assert np.max(np.abs(bs.get(k, "x") - ores["x"][k])) <= 1e-8
    for i, qp in enumerate(qps):
        stat, dyn, feas, comp = kkt_residuals(qp, bs.result, i)
        assert stat <= 1e-5 and dyn <= 1e-7 and feas <= 1e-7
    bs.close()


@pytest.mark.gpu
@pytest.mark.parametrize("warm_start,cond_N", [(2, None), (3, None), (2, 3), (3, 3)])
def test_warm_start_through_the_front_end_gpu(built, warm_start, cond_N):
    """warm_start >= 2: a solve starts from the previous solve's solution in the solver's (reduced or condensed) layout, as the
    reference's xcond solver does (ocp_qp_xcond_solver.c:554-569).  Solve, update with new vectors, solve again: the device route
    (cuipm_xcond) and the host route agree on iteration counts and solutions, and the second solve is not a cold one."""
    import copy
    from acados_b200.ocp_qp import OcpQpBatchSolver
    # the routes' first solutions differ in the last bits (see test_batch_solver_gpu); warm_start = 3 restarts from multipliers
    # clamped at lam0_min, which at the default tolerances leaves the routes ~1e-8 apart, so both run to 1e-10; a QP right at
    # the stopping threshold could still take one iteration more on one route: these instances have none
    tight = dict(tol_stat=1e-10, tol_eq=1e-10, tol_ineq=1e-10, tol_comp=1e-10)
    rng = np.random.default_rng(6)
    qps = [random_ocp_qp(rng) for _ in range(16)]
    new = copy.deepcopy(qps)
    for qp in new:
        x0 = qp.lbx[0] + 0.05 * rng.standard_normal(qp.lbx[0].shape)
        qp.set("lbx", 0, x0); qp.set("ubx", 0, x0)
        for k in range(qp.N + 1):
            qp.set("q", k, qp.q[k] + 0.05 * rng.standard_normal(qp.q[k].shape))
            if k < qp.N:
                qp.set("b", k, qp.b[k] + 0.01 * rng.standard_normal(qp.b[k].shape))
    routes = [OcpQpBatchSolver(qps, OcpQpOptions(warm_start=warm_start, cond_N=cond_N, **tight), device_reduce=d) for d in (True, False)]
    for bs in routes:
        # the first solve runs cold: from zeros, warm_start = 3 clamps the multipliers to lam0_min and stops at the minimal step
        bs.c_opts.warm_start = 0
        assert (bs.solve() == 0).all()
        bs.c_opts.warm_start = warm_start
        bs.update(new)
        bs.solve()
    bs, bh = routes
    assert np.array_equal(bs.info["status"], bh.info["status"]) and (bs.info["status"] == 0).sum() >= 12
    assert np.array_equal(bs.get_stats("iter"), bh.get_stats("iter"))
    ok = bs.info["status"] == 0
    for k in range(bs.N + 1):
        for f in ("u", "x", "sl", "su"):
            assert np.allclose(bs.get(k, f)[ok], bh.get(k, f)[ok], rtol=0, atol=1e-9), (k, f)
        for f in ("lam", "t"):
            assert np.allclose(bs.get(k, f)[ok], bh.get(k, f)[ok], rtol=1e-6, atol=1e-8), (k, f)
    cold = OcpQpBatchSolver(new, OcpQpOptions(cond_N=cond_N, **tight))
    cold.solve()
    assert any(not np.array_equal(bs.get(k, "u"), cold.get(k, "u")) for k in range(bs.N))
    bs.close(); bh.close(); cold.close()


@pytest.mark.gpu
@pytest.mark.parametrize("soft,general", [(False, False), (True, True)])
def test_device_elimination_matches_host(built, soft, general):
    """cuipm_reduce_device / cuipm_restore_device (the batched reduce_eq_dof / restore_eq_dof of row a15) against the
    host implementation above, which the CPU tests check against the reference's fixtures and the original KKT system."""
    import torch
    from acados_b200.binding import CuipmReducer, CuipmSolver
    rng = np.random.default_rng(11)
    qps = [random_ocp_qp(rng, soft=soft, general=general) for _ in range(32)]
    full = PackedBatch(qps, eliminate=False)              # records as posed: x0 = coinciding stage-0 bounds
    red = PackedBatch(qps)                                # host-side elimination
    r = CuipmReducer(full.shape, [int(i) for i in qps[0].idxe[0]])
    assert (r.reduced_shape.nx, r.reduced_shape.nb, r.reduced_shape.idxb, r.reduced_shape.idxs_rev) == \
           (red.shape.nx, red.shape.nb, red.shape.idxb, red.shape.idxs_rev)
    d_full = torch.from_numpy(full.qp).cuda()
    d_red = torch.zeros((len(qps), red.layout.qp_stride), dtype=torch.float64, device="cuda")
    r.reduce(len(qps), d_full.data_ptr(), d_red.data_ptr())
    torch.cuda.synchronize()
    got = d_red.cpu().numpy()
    assert np.max(np.abs(got - red.qp)) <= 1e-13 * max(1.0, np.max(np.abs(red.qp)))
    # solve the device-reduced records, restore on the device, compare with the host restore of the same solution
    o = default_opts()
    s = CuipmSolver(red.shape, len(qps))
    sol_red, info = s.solve(got, o)
    s.close()
    assert (info["status"] == 0).all()
    d_sol_red = torch.from_numpy(sol_red).cuda()
    d_sol_full = torch.zeros((len(qps), full.layout.sol_stride), dtype=torch.float64, device="cuda")
    r.restore(len(qps), d_full.data_ptr(), d_sol_red.data_ptr(), d_sol_full.data_ptr(), o.lam_min, o.t_min)
    torch.cuda.synchronize()
    sol_full = d_sol_full.cpu().numpy()
    r.close()
    ref = red.unpack(sol_red, o.lam_min, o.t_min)
    Lf = full.layout
    for k in range(full.N + 1):
        nu, nx, ns = full.shape.nu[k], full.shape.nx[k], full.shape.ns[k]
        ux = Lf.view(sol_full, "ux", k)
        assert np.array_equal(ux[:, :nu], ref["u"][k]) and np.allclose(ux[:, nu:nu + nx], ref["x"][k], rtol=0, atol=1e-15)
        assert np.array_equal(ux[:, nu + nx:nu + nx + ns], ref["sl"][k])
        assert np.allclose(Lf.view(sol_full, "lam", k), ref["lam"][k], rtol=1e-12, atol=1e-12)
        assert np.allclose(Lf.view(sol_full, "t", k), ref["t"][k], rtol=1e-12, atol=1e-14)
        if k < full.N:
            assert np.array_equal(Lf.view(sol_full, "pi", k), ref["pi"][k])
