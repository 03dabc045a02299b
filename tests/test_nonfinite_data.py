"""QPs with non-finite data, and acados-style infinite bounds, on every solver route.

A batch from an RL or MPC sweep routinely holds a QP whose linearisation diverged.  What a user needs from a batched solver then:
the bad QP gets the reference's status and iteration count (NAN_SOL, which the plugin reports as ACADOS_NAN_DETECTED), and every
other QP in the batch -- and every later solve on the same object -- gets the bits it would get without the bad QP.  The kernels
carry code that exists only for such data (the NaN-propagating norms rmax_nan / gmax_nan, the three NAN_SOL exits, the order of
the operands of every comparison a NaN reaches); these tests run it.

The poisoned batch: a clean seeded batch in which QPs 1, 3, ..., 13 carry exactly one defect each (DEFECTS), so that clean QPs sit
on both sides of each poisoned one and share its warps and chunks.  The masked-infinity family: clean QPs in which every other
state and input bound is masked out (dmask = 0) and holds +-1e10, the form in which acados passes one-sided bounds
(ocp_nlp_constraints_bgh.c sets dmask = 0 at or beyond +-ACADOS_INFTY and leaves the value in d).

CPU part: the oracle against the reference's answers, taken one QP per fresh reference object and stored in
tests/golden/reference/nonfinite.npz (tests/golden/make_reference_answers.py); the reference's carry-over of a NaN into later
solves on one object, recorded as observed behaviour; the throughput kernel's body on the warp emulation.
GPU part: every route against the oracle (poisoned QPs) and against its own clean run (clean QPs, bit for bit), no carry-over
across solves on one object, and the masked-infinity family within the bars of tests/test_parity_gpu.py."""
import copy
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from acados_b200 import problems as P  # noqa: E402
from acados_b200.binding import default_opts  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "reference", "nonfinite.npz")
TOL_U = 1e-10
NAN_SOL = 3
HANDED_BACK = 100
ACADOS_NAN_DETECTED = 1

DEFECTS = ("rq_nan", "b_nan", "hess_nan", "masked_bound_nan", "BAt_inf", "x0_nan", "unconstrained_rq_nan")
POISONED = {2 * i + 1: d for i, d in enumerate(DEFECTS)}       # QP index -> defect; the even QPs stay clean
NBATCH = 2 * len(DEFECTS) + 1
ITREF = (2, 0)                                                  # itref_corr_max: the acados default, and no refinement


# ---- batches --------------------------------------------------------------------------------------------------------------

def _clean(family, nbatch=NBATCH, seed=3):
    """The families: the throughput kernel's shapes (name, lanes per QP) and two shapes only the generic kernel takes."""
    if family == "chain_mass":
        return P.chain_mass(nbatch, N=10, seed=seed)
    if family == "pendulum":
        return P.random_qp(P.random_shape(20, 4, 1, nbx=0), nbatch, seed=seed, umax=0.5, x0_scale=1.0)
    if family == "legged":
        return P.random_qp(P.random_shape(3, 48, 12, nbx=12, ns=12), nbatch, seed=seed, umax=0.5, xmax=1.0, x0_scale=1.0)
    if family == "rand_soft":
        return P.random_qp(P.random_shape(8, 5, 2, nbx=3, ng=2, ns=3), nbatch, seed=seed, umax=0.3, xmax=3.0, x0_scale=1.0)
    if family == "rand_general":
        return P.random_qp(P.random_shape(8, 5, 2, nbx=2, ng=3), nbatch, seed=seed, umax=0.3, xmax=3.0, x0_scale=1.0)
    raise ValueError(family)


FAST_G = {"chain_mass": 8, "pendulum": 2, "legged": 32}       # lanes per QP of the throughput kernel's instance
FAMILIES = tuple(FAST_G) + ("rand_soft", "rand_general")


def poison(b, q, defect):
    """Gives QP q of batch b (records in place) the one defect named."""
    L, sh = b.layout, b.shape
    k = sh.N // 2                                               # an interior stage: nu, nx > 0 and constraints
    if defect == "rq_nan":
        L.view(b.qp, "rq", k)[q, sh.nu[k]] = np.nan             # a state gradient entry
    elif defect == "b_nan":
        L.view(b.qp, "b", k)[q, 1] = np.nan
    elif defect == "hess_nan":
        L.view(b.qp, "RSQ", k)[q, 0, 0] = np.nan                # R[0, 0]: the first pivot of the stage's factorisation
    elif defect == "masked_bound_nan":
        nb, ng = sh.nb[k], sh.ng[k]
        row = nb + ng                                           # the upper bound of the stage's first box constraint
        L.view(b.qp, "dmask", k)[q, row] = 0.0
        L.view(b.qp, "d", k)[q, row] = np.nan
    elif defect == "BAt_inf":
        L.view(b.qp, "BAt", k)[q, 0, 0] = np.inf
    elif defect == "x0_nan":
        L.view(b.qp, "b", 0)[q, :] = np.nan                     # x0 is eliminated: b_0 = b + A x0 is NaN in every entry
    elif defect == "unconstrained_rq_nan":
        for j in range(sh.N + 1):
            L.view(b.qp, "dmask", j)[q, :] = 0.0
        L.view(b.qp, "rq", k)[q, 0] = np.nan
    else:
        raise ValueError(defect)


def poisoned(family, nbatch=NBATCH, where=None):
    """(clean batch, poisoned batch): QP where[i] carries DEFECTS[i] (default: the odd QPs of a 15-QP batch)."""
    clean = _clean(family, nbatch)
    bad = P.Batch(clean.shape, clean.layout, clean.qp.copy(), clean.name + " poisoned")
    where = sorted(POISONED) if where is None else where
    for q, d in zip(where, DEFECTS):
        poison(bad, q, d)
    return clean, bad


def masked_infinity(family, nbatch=NBATCH):
    """Clean QPs in which every other box constraint is one-sided: the lower bound of even rows and the upper bound of odd rows
    are masked out and hold -1e10 / +1e10 (d stores lb and -ub)."""
    b = _clean(family, nbatch, seed=5)
    sh, L = b.shape, b.layout
    for k in range(sh.N + 1):
        nb, ng = sh.nb[k], sh.ng[k]
        d, m = L.view(b.qp, "d", k), L.view(b.qp, "dmask", k)
        for i in range(nb):
            row = i if i % 2 == 0 else nb + ng + i
            m[:, row] = 0.0
            d[:, row] = -1e10
    b.name += " masked-infinity"
    return b


def _sub(b, idx):
    return P.Batch(b.shape, b.layout, np.ascontiguousarray(b.qp[idx]), b.name)


# full-shape records (x0 a stage-0 equality) for the xcond chain and the tensor front end: defects 1 and 6 as a user poses them
FULL_N, FULL_COARSE = 10, 3
FULL_POISONED = {2: "q_nan", 5: "x0_nan"}


def full_qps(masked=False, nbatch=8):
    from test_ocp_qp_mirror import random_ocp_qp
    rng = np.random.default_rng(13)
    qps = [random_ocp_qp(rng, N=FULL_N, nx=4, nu=2, soft=True, general=True) for _ in range(nbatch)]
    if masked:
        for qp in qps:
            for k in range(1, FULL_N + 1):
                if qp.lbu[k].size:
                    qp.set("lbu", k, np.array([-1e10, qp.lbu[k][1]])); qp.set("lbu_mask", k, np.array([0.0, 1.0]))
                    qp.set("ubu", k, np.array([qp.ubu[k][0], 1e10])); qp.set("ubu_mask", k, np.array([1.0, 0.0]))
                qp.set("lbx", k, np.array([-1e10, qp.lbx[k][1]])); qp.set("lbx_mask", k, np.array([0.0, 1.0]))
                qp.set("ubx", k, np.array([qp.ubx[k][0], 1e10])); qp.set("ubx_mask", k, np.array([1.0, 0.0]))
    return qps


def poison_full(qps):
    bad = [q for q in qps]
    for i, d in FULL_POISONED.items():
        q = _copy_qp(qps[i])
        if d == "q_nan":
            v = q.q[FULL_N // 2].copy(); v[1] = np.nan
            q.set("q", FULL_N // 2, v)
        else:
            v = np.full(q.lbx[0].shape, np.nan)
            q.set("lbx", 0, v); q.set("ubx", 0, v.copy())
        bad[i] = q
    return bad


def _copy_qp(qp):
    return copy.deepcopy(qp)


def _full_oracle(qps, cond_N, o):
    """The host chain on the QPs as posed: x0 elimination (PackedBatch), block condensing to cond_N stages, the oracle's IPM.
    Returns (sol, info) of the reduced (cond_N = N) or condensed records."""
    from acados_b200.condensing import BlockCondenser
    from acados_b200.ocp_qp import PackedBatch
    from oracle import oracle_binding as ob
    red = PackedBatch(qps)
    if cond_N >= FULL_N:
        return ob.oracle_solve(P.Batch(red.shape, red.layout, red.qp, "reduced"), o)
    bc = BlockCondenser(red.shape, cond_N)
    return ob.oracle_solve(P.Batch(bc.cshape, bc.clay, bc.condense(red.qp), "condensed"), o)


# ---- comparisons ----------------------------------------------------------------------------------------------------------

def _same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _assert_clean_bits(idx, sol, info, csol, cinfo, stat=None, cstat=None):
    """QPs idx of a poisoned run against the same QPs of the clean run: solution, summary and statistics bit for bit."""
    assert _same_bits(sol[idx], csol[idx]), "a clean QP of the poisoned batch changed"
    for f in info.dtype.names:
        assert _same_bits(info[f][idx], cinfo[f][idx]), f
    if stat is not None:
        assert _same_bits(stat[idx], cstat[idx])


def _unconstrained_branch_writes(L):
    """Columns of a solution record the reference's unconstrained branch writes (OCP_QP_FACT_SOLVE_KKT_UNCONSTR,
    x_ocp_qp_kkt.c): u, x and pi.  It leaves the slacks, lam and t as they were in the caller's ocp_qp_out, so there the
    reference's values are those of an earlier solve (zeros on a fresh object), not a result."""
    m = np.zeros(L.sol_stride, dtype=bool)
    for k in range(L.shape.N + 1):
        m[L.off["ux"][k]:L.off["ux"][k] + L.shape.nv(k)] = True
        m[L.off["pi"][k]:L.off["pi"][k] + L.size["pi"][k]] = True
    return m


def _masked_rows(b):
    """(nbatch, sol_stride): the lam and t entries of the rows each QP masks out (dmask = 0)."""
    L, sh = b.layout, b.shape
    m = np.zeros((b.nbatch, L.sol_stride), dtype=bool)
    for k in range(sh.N + 1):
        off = L.view(b.qp, "dmask", k) == 0.0
        for f in ("lam", "t"):
            m[:, L.off[f][k]:L.off[f][k] + off.shape[1]] = off
    return m


def _assert_solution_close(b, s1, s2):
    """The whole-solution bar of tests/test_oracle_vs_reference.py, |s1 - s2| <= 1e-6 max(1, max |s2|), over the entries of the
    rows that are not masked out; on the lam and t of masked rows (t is the distance to a bound of +-1e10 there, which would set
    the scale of the whole bar) the same bar entry by entry, 1e-6 max(1, |s2|)."""
    m = _masked_rows(b)
    d = np.abs(s1 - s2)
    assert np.max(d[~m]) <= 1e-6 * max(1.0, np.max(np.abs(s2[~m]))), np.max(d[~m])
    assert (d[m] <= 1e-6 * np.maximum(1.0, np.abs(s2[m]))).all()


def _oracle_reference_bars(b, s1, i1, s2, i2):
    """tests/test_oracle_vs_reference.py's bars, per QP, where both solutions are finite."""
    assert np.array_equal(i1["status"], i2["status"]), (i1["status"], i2["status"])
    assert np.array_equal(i1["iter"], i2["iter"]), (i1["iter"], i2["iter"])
    cols = np.where((i2["iter"] == 0)[:, None], _unconstrained_branch_writes(b.layout)[None, :], True)
    assert np.array_equal(np.isfinite(s1) & cols, np.isfinite(s2) & cols)
    fin = np.isfinite(s2).all(axis=1)
    if not fin.any():
        return
    du = np.max(np.abs(b.layout.u_traj(s1[fin]) - b.layout.u_traj(s2[fin])), axis=1)
    conv = i2["status"][fin] == 0
    assert du[conv].max(initial=0.0) <= TOL_U, du
    assert du.max() <= 1e-8, du
    _assert_solution_close(_sub(b, np.nonzero(fin)[0]), s1[fin], s2[fin])


def _digest(qp):
    """SHA-256 of the whole records (NaN and inf included), as 32 bytes."""
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(qp).tobytes()).digest(), dtype=np.uint8)


# ---- the reference's answers ----------------------------------------------------------------------------------------------

def reference_answers():
    """What the reference returns, each QP solved by its own fresh reference object (one QP per ref_solve call: the harness
    creates its solver memory per call).  The generator of tests/golden/reference/nonfinite.npz."""
    from oracle import oracle_binding as ob
    from acados_b200.ocp_qp import PackedBatch
    from acados_b200.problems import Batch
    out = {}

    def per_qp(b, o):
        sols, infos = [], []
        for q in range(b.nbatch):
            s, i, _ = ob.ref_solve(_sub(b, [q]), o, nthreads=1)
            sols.append(s); infos.append(i)
        return np.concatenate(sols), np.concatenate(infos)

    for fam in FAMILIES:
        for itref in ITREF:
            o = default_opts(itref_corr_max=itref)
            _, bad = poisoned(fam)
            for tag, b in (("poisoned", bad), ("masked_inf", masked_infinity(fam))):
                key = f"{fam}_{tag}_itref{itref}"
                s, i = per_qp(b, o)
                out.update({key + "_qp_sha256": _digest(b.qp), key + "_iter": i["iter"], key + "_status": i["status"],
                            key + "_u": b.layout.u_traj(s), key + "_sol": s.astype(np.float32)})
    o = default_opts()
    for tag, qps in (("poisoned", poison_full(full_qps())), ("masked_inf", full_qps(masked=True))):
        full = PackedBatch(qps, eliminate=False)
        idxe0 = [int(i) for i in qps[0].idxe[0]]
        for cond_N in (FULL_N, FULL_COARSE):
            infos = [ob.ref_solve_xcond(Batch(full.shape, full.layout, np.ascontiguousarray(full.qp[[q]]), "full"), idxe0, cond_N, o)[1]
                     for q in range(len(qps))]
            key = f"xcond_{tag}_N{cond_N}"
            out.update({key + "_qp_sha256": _digest(full.qp), key + "_iter": np.concatenate(infos)["iter"], key + "_status": np.concatenate(infos)["status"]})
    return out


def _stored(key, b=None, qp=None):
    """The reference's answers stored under ``key``, after checking that the records they were taken on (those of batch b, or
    the full-shape records qp) are still the ones the builders make."""
    g = np.load(GOLD, allow_pickle=False)
    qp = b.qp if b is not None else qp
    assert _same_bits(_digest(qp), g[key + "_qp_sha256"]), "generator drifted from the stored inputs"
    info = np.zeros(len(g[key + "_iter"]), dtype=[("status", np.int32), ("iter", np.int32)])
    info["status"], info["iter"] = g[key + "_status"], g[key + "_iter"]
    if key + "_sol" not in g:
        return None, info
    # the solution is stored in float32 (NaN and inf kept), the inputs in float64 (compared to 1e-10)
    sol, u, col = g[key + "_sol"].astype(np.float64), g[key + "_u"], 0
    for k in range(b.shape.N + 1):
        nu = b.shape.nu[k]
        b.layout.view(sol, "ux", k)[:, :nu] = u[:, col:col + nu]
        col += nu
    return sol, info


# ---- CPU: the oracle against the reference --------------------------------------------------------------------------------

@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("itref", ITREF)
@pytest.mark.parametrize("tag", ["poisoned", "masked_inf"])
def test_oracle_matches_reference_on_nonfinite_data(built, family, itref, tag):
    """Per QP: the reference's status and iteration count, the same finite entries in the solution, and where both are finite
    the bars of test_oracle_vs_reference.py.  Every poisoned QP ends with NAN_SOL; the clean ones converge."""
    from oracle import oracle_binding as ob
    o = default_opts(itref_corr_max=itref)
    b = poisoned(family)[1] if tag == "poisoned" else masked_infinity(family)
    s1, i1 = ob.oracle_solve(b, o)
    s2, i2 = _stored(f"{family}_{tag}_itref{itref}", b)
    _oracle_reference_bars(b, s1, i1, s2, i2)
    if tag == "poisoned":
        bad = np.array(sorted(POISONED))
        assert (i1["status"][bad] == NAN_SOL).all(), i1["status"]
        assert (np.delete(i1["status"], bad) == 0).all()
    else:
        assert (i1["status"] == 0).all()
    if ob.have_ref():                                           # the stored answers are still what the reference returns
        for q in (0, 1, 7, 13):
            s, i, _ = ob.ref_solve(_sub(b, [q]), o, nthreads=1)
            assert i["status"][0] == i2["status"][q] and i["iter"][0] == i2["iter"][q]
            assert _same_bits(np.isfinite(s[0]), np.isfinite(s2[q]))


@pytest.mark.parametrize("tag", ["poisoned", "masked_inf"])
@pytest.mark.parametrize("cond_N", [FULL_N, FULL_COARSE])
def test_host_chain_matches_reference_xcond(built, tag, cond_N):
    """The QPs as posed (x0 a stage-0 equality; defect 1 and a NaN x0): the host chain (elimination, condensing, the oracle's
    IPM) against the reference's whole xcond path, one QP per reference object: same status (the reference's is acados') and
    iteration count per QP."""
    from acados_b200.ocp_qp import PackedBatch
    from test_host_pipeline import ACADOS_STATUS
    qps = poison_full(full_qps()) if tag == "poisoned" else full_qps(masked=True)
    _, i1 = _full_oracle(qps, cond_N, default_opts())
    _, i2 = _stored(f"xcond_{tag}_N{cond_N}", qp=PackedBatch(qps, eliminate=False).qp)
    assert [ACADOS_STATUS[int(s)] for s in i1["status"]] == i2["status"].tolist(), (i1["status"], i2["status"])
    assert np.array_equal(i1["iter"], i2["iter"]), (i1["iter"], i2["iter"])
    if tag == "poisoned":
        assert (i1["status"][sorted(FULL_POISONED)] == NAN_SOL).all()
        assert (np.delete(i1["status"], sorted(FULL_POISONED)) == 0).all()


def test_reference_carries_a_nan_into_later_solves(built):
    """Observed behaviour of the reference, recorded: one reference object (one solver memory, one ocp_qp_out, reused as acados
    reuses them across SQP iterations) that has solved a poisoned QP of the rand_soft shape returns NAN_SOL after one iteration
    for every QP it solves afterwards, the clean ones included, while the same clean QPs solved alone converge.  This is why
    the stored answers are taken one QP per object, and why 'a later solve is not disturbed' is a property the CUDA routes are
    tested for on their own (test_no_carry_over_*)."""
    from oracle import oracle_binding as ob
    if not ob.have_ref():
        pytest.skip("oracle/_ref not built (needs the reference sources)")
    o = default_opts()
    clean, bad = poisoned("rand_soft")
    _, one = ob.ref_solve(bad, o, nthreads=1)[:2]               # the whole batch on one object, in order
    _, alone = _stored("rand_soft_poisoned_itref2", bad)
    after = np.arange(2, NBATCH, 2)                             # the clean QPs that come after the first poisoned one
    assert (alone["status"][after] == 0).all()
    assert (one["status"][after] == NAN_SOL).all() and (one["iter"][after] == 1).all(), one
    assert one["status"][0] == 0 and one["iter"][0] == alone["iter"][0]


# ---- CPU: the throughput kernel's body on the warp emulation --------------------------------------------------------------

def _emul_run(family, itref, order, out):
    """Subprocess body: the poisoned and the clean batch through ob.fast_emul_solve with rr off and on."""
    from oracle import oracle_binding as ob
    clean, bad = poisoned(family)
    o = default_opts(itref_corr_max=itref)
    res = {}
    for rr in (0, 1):
        for tag, b in (("clean", clean), ("bad", bad)):
            s, i, st, r = ob.fast_emul_solve(b, o, g=FAST_G[family], order=order, want_stat=True, rr=bool(rr))
            res.update({f"{tag}{rr}_sol": s, f"{tag}{rr}_info": i, f"{tag}{rr}_stat": st, f"{tag}{rr}_redo": r})
    np.savez(out, **res)


@pytest.mark.parametrize("family", list(FAST_G))
@pytest.mark.parametrize("itref", ITREF)
@pytest.mark.parametrize("order", [0, 1])
def test_throughput_kernel_emulation_on_poisoned_batch(built, tmp_path, family, itref, order):
    """Run in a subprocess with a timeout, so that a QP that never leaves a ring fails the test instead of hanging it.  Each
    poisoned QP gets the oracle's status and iteration count or is handed back; a QP is handed back only where the kernel must
    hand it back (no active constraint: defect 7, or a failed linear-system test, which needs itref_corr_max > 0); every clean
    QP has the bits of the clean batch (solution, summary, statistics); the iteration-sliced schedule changes no bit."""
    from oracle import oracle_binding as ob
    out = str(tmp_path / "emul.npz")
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; "
            f"import test_nonfinite_data as t; t._emul_run({family!r}, {itref}, {order}, {out!r})")
    r = subprocess.run([sys.executable, "-c", code], timeout=600, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    e = dict(np.load(out, allow_pickle=False))
    o = default_opts(itref_corr_max=itref)
    _, bad = poisoned(family)
    _, oinfo = ob.oracle_solve(bad, o)
    bad_idx = np.array(sorted(POISONED))
    clean_idx = np.delete(np.arange(NBATCH), bad_idx)
    for rr in (0, 1):
        info, redo = e[f"bad{rr}_info"], e[f"bad{rr}_redo"]
        keep = np.setdiff1d(np.arange(NBATCH), redo)
        assert (info["status"][redo] == HANDED_BACK).all()
        assert np.array_equal(info["status"][keep], oinfo["status"][keep]), (info["status"], oinfo["status"])
        assert np.array_equal(info["iter"][keep], oinfo["iter"][keep]), (info["iter"], oinfo["iter"])
        # the unconstrained QP is always handed back; others only through the linear-system test's refinement
        unc = [q for q, d in POISONED.items() if d == "unconstrained_rq_nan"]
        assert set(unc) <= set(redo.tolist())
        assert set(redo.tolist()) <= set(bad_idx.tolist()), redo
        if itref == 0:
            assert redo.tolist() == unc, redo
        # the clean batch's own hand-backs (none on these families) are the clean QPs' hand-backs in the poisoned batch
        assert np.array_equal(np.intersect1d(redo, clean_idx), e[f"clean{rr}_redo"])
        _assert_clean_bits(clean_idx, e[f"bad{rr}_sol"], info, e[f"clean{rr}_sol"], e[f"clean{rr}_info"],
                           e[f"bad{rr}_stat"], e[f"clean{rr}_stat"])
    for f in ("sol", "info", "stat", "redo"):
        assert _same_bits(e[f"bad0_{f}"], e[f"bad1_{f}"]), f"rr changed {f}"


# ---- GPU ------------------------------------------------------------------------------------------------------------------

ROUTES = {"fast_rr0": dict(rr=0), "fast_rr2": dict(rr=2), "generic_w1": dict(fast=0, warps=1), "generic_w2": dict(fast=0, warps=2),
          "generic_w4": dict(fast=0, warps=4), "generic_spill": dict(fast=0, spill=1)}


def _solver(b, route, nbatch=None):
    from acados_b200.binding import CuipmSolver
    s = CuipmSolver(b.shape, nbatch or b.nbatch)
    for k, v in ROUTES[route].items():
        s.set_tuning(k, v)
    return s


def _run(b, o, route):
    s = _solver(b, route)
    sol, info, stat = s.solve(b.qp, o, want_stat=True)
    hb = s.last_handed_back
    s.close()
    return sol, info, stat, hb


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("itref", ITREF)
def test_poisoned_batch_on_every_kernel_route(built, family, itref):
    """Throughput kernel (rr 0 and 2), generic kernel at 1, 2 and 4 warps, generic kernel with global scratch: the oracle's
    status and iteration count on every poisoned QP, and the clean QPs bit-identical to the route's run of the clean batch."""
    from oracle import oracle_binding as ob
    o = default_opts(itref_corr_max=itref)
    clean, bad = poisoned(family)
    _, oinfo = ob.oracle_solve(bad, o)
    bad_idx = np.array(sorted(POISONED))
    clean_idx = np.delete(np.arange(NBATCH), bad_idx)
    handed = {}
    for route in ROUTES:
        sol, info, stat, hb = _run(bad, o, route)
        csol, cinfo, cstat, _ = _run(clean, o, route)
        assert np.array_equal(info["status"], oinfo["status"]), (route, info["status"], oinfo["status"])
        assert np.array_equal(info["iter"], oinfo["iter"]), (route, info["iter"], oinfo["iter"])
        assert (info["status"][bad_idx] == NAN_SOL).all()
        _assert_clean_bits(clean_idx, sol, info, csol, cinfo, stat, cstat)
        handed[route] = hb
    # which QPs the throughput kernel hands back: the solver reports a count only, so each QP is solved on its own as well; the
    # decision depends on the QP alone, hence the batch's count is the size of that set, the same under both schedules
    for route in ("fast_rr0", "fast_rr2"):
        s = _solver(bad, route, nbatch=1)
        which = []
        for q in range(NBATCH):
            s.solve(np.ascontiguousarray(bad.qp[[q]]), o)
            if s.last_handed_back:
                which.append(q)
        s.close()
        print(f"{family} itref_corr_max={itref} {route} handed back: {which}")
        assert handed[route] == len(which)
        assert set(which) <= set(bad_idx.tolist())
        if family in FAST_G:
            unc = [q for q, d in POISONED.items() if d == "unconstrained_rq_nan"]
            assert set(unc) <= set(which) and (itref > 0 or which == unc), which
        else:
            assert which == []                                  # shapes the throughput kernel does not take
        handed[route + "_set"] = which
    assert handed["fast_rr0_set"] == handed["fast_rr2_set"]


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_masked_infinity_on_every_kernel_route(built, family):
    """One-sided bounds as acados passes them (dmask = 0, +-1e10 in d): the oracle's iteration counts and statuses, and
    tests/test_parity_gpu.py's bars on the solution."""
    from oracle import oracle_binding as ob
    from test_parity_gpu import _tol_default
    b = masked_infinity(family)
    for itref in ITREF:
        o = default_opts(itref_corr_max=itref)
        osol, oinfo = ob.oracle_solve(b, o)
        assert (oinfo["status"] == 0).all()
        for route in ROUTES:
            sol, info, _, _ = _run(b, o, route)
            assert np.array_equal(info["iter"], oinfo["iter"]) and np.array_equal(info["status"], oinfo["status"]), route
            du = np.max(np.abs(b.layout.u_traj(sol) - b.layout.u_traj(osol)))
            assert du <= _tol_default("c2" if family == "chain_mass" else family), (route, du)
            _assert_solution_close(b, sol, osol)


HOST_N = 1024
HOST_CHUNKS = 8                                                 # cuipm_solve_host's chunks (each on its own stream) from 512 QPs on
HOST_WHERE = [37 + 140 * i for i in range(len(DEFECTS))]        # spread over chunks 0 .. 6 of 128 QPs
# launches per chunk: the repack, the throughput kernel (one launch, or rr_first + rr_loop on the rings), the generic kernel over
# the QPs handed back
HOST_LAUNCHES = {0: 3 * HOST_CHUNKS, 2: 4 * HOST_CHUNKS}


def _host_runs(b, o):
    """cuipm_solve_host on b with the single-launch schedule and with the iteration-sliced one forced in every chunk (a chunk of
    128 QPs is below what the device holds at once, so the default would not take the rings): {rr: (sol, info, handed back)}."""
    out = {}
    for rr in (2, 0):
        s = _solver(b, f"fast_rr{rr}")
        sol, info = s.solve(b.qp, o)
        assert s.last_launch_count == HOST_LAUNCHES[rr], (rr, s.last_launch_count)
        out[rr] = (sol, info, s.last_handed_back)
        s.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("itref", ITREF)
def test_poisoned_batch_through_the_host_pipeline(built, itref):
    """cuipm_solve_host at n = 1024 (eight chunks on concurrent streams; every chunk on its own rings and ring counters with
    rr = 2) and the plugin's batched entry on the same records: the poisoned QPs get the oracle's status and iteration count
    (ACADOS_NAN_DETECTED through the plugin), the clean ones the bits of the clean batch under the same schedule; both schedules
    give the same bits and hand back as many QPs."""
    from oracle import oracle_binding as ob
    o = default_opts(itref_corr_max=itref)
    clean, bad = poisoned("chain_mass", HOST_N, HOST_WHERE)
    bad_idx = np.array(HOST_WHERE)
    clean_idx = np.delete(np.arange(HOST_N), bad_idx)
    _, oinfo = ob.oracle_solve(_sub(bad, bad_idx), o)
    assert (oinfo["status"] == NAN_SOL).all()
    runs, cruns = _host_runs(bad, o), _host_runs(clean, o)
    for rr in (2, 0):
        sol, info, hb = runs[rr]
        assert np.array_equal(info["status"][bad_idx], oinfo["status"]) and np.array_equal(info["iter"][bad_idx], oinfo["iter"])
        _assert_clean_bits(clean_idx, sol, info, cruns[rr][0], cruns[rr][1])
        want = len(DEFECTS) if itref > 0 else 1                 # every poisoned QP, or the unconstrained one only
        assert want <= hb <= want + cruns[rr][2], (hb, cruns[rr][2])
    assert _same_bits(runs[2][0], runs[0][0]) and _same_bits(runs[2][1], runs[0][1]) and runs[2][2] == runs[0][2]
    sol, info = runs[0][:2]
    csol = cruns[0][0]
    from integration import plugin_bench as pb
    if not pb.available():
        pytest.skip("libplugin_bench.so did not travel")
    p = pb.PluginBatch(bad, o)
    p.run(2)
    psol, piter, pstatus = p.solutions()
    p.close()
    assert np.array_equal(piter, info["iter"])
    assert (pstatus[bad_idx] == ACADOS_NAN_DETECTED).all() and (pstatus[clean_idx] == 0).all()
    for f in ("ux", "pi", "lam", "t"):
        assert _same_bits(bad.layout.gather(psol, f)[clean_idx], bad.layout.gather(csol, f)[clean_idx]), f


@pytest.mark.gpu
@pytest.mark.parametrize("itref", ITREF)
def test_masked_infinity_through_the_host_pipeline(built, itref):
    """The masked-infinity family at n = 1024 through cuipm_solve_host under both schedules and through the plugin's batched
    entry: the oracle's iteration counts and statuses on a sample, tests/test_parity_gpu.py's bars on it, the same bits from
    both schedules and from the plugin."""
    from oracle import oracle_binding as ob
    o = default_opts(itref_corr_max=itref)
    b = masked_infinity("chain_mass", HOST_N)
    runs = _host_runs(b, o)
    sol, info = runs[0][:2]
    assert _same_bits(runs[2][0], sol) and _same_bits(runs[2][1], info)
    idx = np.arange(0, HOST_N, 37)
    sb = _sub(b, idx)
    osol, oinfo = ob.oracle_solve(sb, o)
    assert np.array_equal(info["iter"][idx], oinfo["iter"]) and np.array_equal(info["status"][idx], oinfo["status"])
    assert (oinfo["status"] == 0).all()
    # a sample at the default tolerances: held as test_full_size_properties_c2 holds its slice
    d = np.max(np.abs(b.layout.u_traj(sol[idx]) - b.layout.u_traj(osol)), axis=1)
    assert (d <= TOL_U).mean() >= 0.9 and d.max() <= 5e-9, (d.max(), (d <= TOL_U).mean())
    _assert_solution_close(sb, sol[idx], osol)
    from integration import plugin_bench as pb
    if not pb.available():
        pytest.skip("libplugin_bench.so did not travel")
    p = pb.PluginBatch(b, o)
    p.run(2)
    psol, piter, pstatus = p.solutions()
    p.close()
    assert np.array_equal(piter, info["iter"]) and (pstatus == 0).all()
    for f in ("ux", "pi", "lam", "t"):
        assert _same_bits(b.layout.gather(psol, f), b.layout.gather(sol, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("itref", ITREF)
def test_handed_back_count_is_the_last_solves(built, itref):
    """cuipm_last_handed_back after a solve of fewer chunks than the one before, and after a solve the throughput kernel does not
    take, reports that solve's hand-backs only: the counters of the chunks a solve leaves unused, or of the throughput kernel
    when the generic kernel solved everything, no longer carry an earlier solve's counts."""
    clean, bad = poisoned("chain_mass", HOST_N, HOST_WHERE)
    o = default_opts(itref_corr_max=itref)
    s = _solver(bad, "fast_rr0")
    s.solve(bad.qp, o)                                          # eight chunks, hand-backs in chunks 0 .. 6
    assert s.last_handed_back >= 1
    small = _sub(clean, np.arange(NBATCH))
    s.solve(small.qp, o)                                        # one chunk of clean QPs
    one = s.last_handed_back
    s.set_tuning("fast", 0)
    s.solve(bad.qp, o)                                          # the generic kernel over everything
    none = s.last_handed_back
    s.close()
    _, _, _, want = _run(small, o, "fast_rr0")
    assert one == want and none == 0, (one, want, none)


def _xcond_run(qps, cond_N, o, xc=None):
    from acados_b200.binding import CuipmXcond
    from acados_b200.ocp_qp import PackedBatch
    full = PackedBatch(qps, eliminate=False)
    own = xc is None
    if own:
        xc = CuipmXcond(full.shape, [int(i) for i in qps[0].idxe[0]], cond_N, len(qps))
    sol, info, stat = xc.solve(full.qp, o, want_stat=True)
    if own:
        xc.close()
    return sol, info, stat


@pytest.mark.gpu
@pytest.mark.parametrize("cond_N", [FULL_N, FULL_COARSE])
@pytest.mark.parametrize("itref", ITREF)
def test_poisoned_qps_through_the_xcond_chain(built, cond_N, itref):
    """A NaN gradient and a NaN x0 in QPs as posed, through the device chain (reduce, condense, IPM, expand, restore) and
    through the tensor front end over it: the host chain's status and iteration count on the poisoned QPs, and full-shape
    solutions of the clean QPs bit-identical to the chain's run of the clean QPs."""
    import torch
    from acados_b200.ocp_qp import OcpQpOptions
    from test_device_batch import _tensor_solver
    o = default_opts(itref_corr_max=itref)
    qps = full_qps()
    bad_qps = poison_full(qps)
    bad_idx = np.array(sorted(FULL_POISONED))
    clean_idx = np.delete(np.arange(len(qps)), bad_idx)
    _, oinfo = _full_oracle(bad_qps, cond_N, o)
    csol, cinfo, cstat = _xcond_run(qps, cond_N, o)
    sol, info, stat = _xcond_run(bad_qps, cond_N, o)
    assert np.array_equal(info["status"], oinfo["status"]) and np.array_equal(info["iter"], oinfo["iter"]), (info, oinfo)
    assert (info["status"][bad_idx] == NAN_SOL).all()
    _assert_clean_bits(clean_idx, sol, info, csol, cinfo, stat, cstat)
    opts = OcpQpOptions(cond_N=cond_N if cond_N < FULL_N else None)
    tb, _ = _tensor_solver(bad_qps, opts)
    tb.c_opts.itref_corr_max = itref
    status = tb.solve().cpu().numpy()
    torch.cuda.synchronize()
    assert (status[bad_idx] == ACADOS_NAN_DETECTED).all() and (status[clean_idx] == 0).all()
    assert _same_bits(tb._sol.cpu().numpy()[clean_idx], csol[clean_idx])
    tinfo = tb.info
    assert np.array_equal(tinfo["iter"], info["iter"]) and np.array_equal(tinfo["status"], info["status"])
    tb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cond_N", [FULL_N, FULL_COARSE])
@pytest.mark.parametrize("itref", ITREF)
def test_masked_infinity_through_the_xcond_chain(built, cond_N, itref):
    """One-sided bounds with +-1e10 masked values in QPs as posed, through the device chain and the tensor front end over it:
    the host chain's iteration counts and statuses, inputs within tests/test_parity_gpu.py's bar of the host chain's expanded
    solution, and the tensor front end's solutions bit-identical to the chain's."""
    import torch
    from acados_b200.condensing import BlockCondenser
    from acados_b200.ocp_qp import OcpQpOptions, PackedBatch
    from test_device_batch import _tensor_solver
    from test_parity_gpu import _tol_default
    o = default_opts(itref_corr_max=itref)
    qps = full_qps(masked=True)
    osol, oinfo = _full_oracle(qps, cond_N, o)
    red = PackedBatch(qps)
    if cond_N < FULL_N:
        osol = BlockCondenser(red.shape, cond_N).expand(red.qp, osol)
    sol, info, _ = _xcond_run(qps, cond_N, o)
    assert (oinfo["status"] == 0).all()
    assert np.array_equal(info["iter"], oinfo["iter"]) and np.array_equal(info["status"], oinfo["status"])
    full = PackedBatch(qps, eliminate=False)
    du = np.max(np.abs(full.layout.u_traj(sol) - red.layout.u_traj(osol)))
    assert du <= _tol_default("c2"), du
    tb, _ = _tensor_solver(qps, OcpQpOptions(cond_N=cond_N if cond_N < FULL_N else None))
    tb.c_opts.itref_corr_max = itref
    status = tb.solve().cpu().numpy()
    torch.cuda.synchronize()
    assert (status == 0).all()
    assert _same_bits(tb._sol.cpu().numpy(), sol)
    tinfo = tb.info
    assert np.array_equal(tinfo["iter"], info["iter"])
    tb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["fast_rr0", "fast_rr2", "generic_w1"])
def test_no_carry_over_on_one_solver(built, route):
    """The poisoned batch, then the clean batch with warm_start = 0 on the same object (work records, rings and their counters,
    hand-back list kept from the first solve): the bits of a fresh object's solve of the clean batch."""
    o = default_opts(warm_start=0)
    clean, bad = poisoned("chain_mass")
    want, winfo, wstat, _ = _run(clean, o, route)
    s = _solver(clean, route)
    s.solve(bad.qp, o, want_stat=True)
    sol, info, stat = s.solve(clean.qp, o, want_stat=True)
    s.close()
    _assert_clean_bits(np.arange(NBATCH), sol, info, want, winfo, stat, wstat)


@pytest.mark.gpu
@pytest.mark.parametrize("cond_N", [FULL_N, FULL_COARSE])
def test_no_carry_over_on_one_xcond_object(built, cond_N):
    """The same on one CuipmXcond, whose previous solution is the warm start of its next solve when warm_start >= 2."""
    from acados_b200.binding import CuipmXcond
    from acados_b200.ocp_qp import PackedBatch
    o = default_opts(warm_start=0)
    qps = full_qps()
    want, winfo, wstat = _xcond_run(qps, cond_N, o)
    full = PackedBatch(qps, eliminate=False)
    xc = CuipmXcond(full.shape, [int(i) for i in qps[0].idxe[0]], cond_N, len(qps))
    _xcond_run(poison_full(qps), cond_N, o, xc)
    sol, info, stat = _xcond_run(qps, cond_N, o, xc)
    xc.close()
    _assert_clean_bits(np.arange(len(qps)), sol, info, want, winfo, stat, wstat)
