"""QPs posed as torch tensors on the GPU: the device-side record assembly (cuipm_xcond_assemble_device), the device-buffer
entries of the xcond chain, and the front end over both (tensor_batch.OcpQpTensorBatchSolver).

CPU part: the assembly kernel's body, run sequentially on the host (tests/assemble_emul.cpp), writes the bits of the host packer
(PackedBatch(eliminate=False).qp) for every source layout, and refuses bad sources; the front end's argument checks raise
before anything is launched.  GPU part: the kernel gives the same bits, and the tensor front end gives the bits of
OcpQpBatchSolver in solutions, summaries and statistics."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from acados_b200.problems import Layout
from acados_b200.binding import FIELD_IDS, INFO_DTYPE, CuipmSrc
from acados_b200.ocp_qp import DYNAMICS_FIELDS, OcpQp, OcpQpBatchSolver, OcpQpOptions, PackedBatch
from test_ocp_qp_mirror import random_ocp_qp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "acados_b200", "csrc")
DATA_FIELDS = tuple(FIELD_IDS)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emul") / "libassemble_emul.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
                    "-o", out, os.path.join(ROOT, "tests", "assemble_emul.cpp"), os.path.join(CSRC, "cuipm_host.cpp")],
                   check=True)
    lib = C.CDLL(out)
    lib.emul_assemble.argtypes = [C.c_void_p, C.c_int, C.POINTER(CuipmSrc), C.c_int, C.c_void_p]
    lib.emul_assemble.restype = C.c_int
    lib.emul_assemble_error.restype = C.c_char_p
    return lib


# ---- QP families -------------------------------------------------------------------------------------------------------

def _masked(rng, qps):
    for q in qps:
        for k in range(q.N + 1):
            for f in ("lbu_mask", "ubx_mask", "lg_mask", "lls_mask"):
                m = q._f[f][k]
                if m.size:
                    q.set(f, k, (rng.random(m.size) > 0.3).astype(float))
    return qps


def _varying(rng, N=5, nx=3, nu=2):
    """nb, ng and ns change from stage to stage; stage 2 has no constraint at all."""
    qp = OcpQp(N)
    for k in range(N + 1):
        nuk = nu if k < N else 0
        qp.set("Q", k, np.eye(nx) + 0.1 * rng.standard_normal((nx, nx)))   # not symmetric: the packer copies as given
        qp.set("R", k, np.eye(nuk) + 0.1 * rng.standard_normal((nuk, nuk)))
        qp.set("S", k, rng.standard_normal((nuk, nx)))
        qp.set("q", k, rng.standard_normal(nx))
        qp.set("r", k, rng.standard_normal(nuk))
        if k < N:
            qp.set("A", k, rng.standard_normal((nx, nx)))
            qp.set("B", k, rng.standard_normal((nx, nuk)))
            qp.set("b", k, rng.standard_normal(nx))
        if k == 0:
            qp.set("idxb", 0, list(range(nuk + nx)))
            x0 = rng.standard_normal(nx)
            qp.set("lbu", 0, -np.ones(nuk)); qp.set("ubu", 0, np.ones(nuk))
            qp.set("lbx", 0, x0); qp.set("ubx", 0, x0)
            qp.set("idxe", 0, list(range(nuk, nuk + nx)))
        elif k != 2:
            nbu, nbx, ng = k % 2 * nuk, k % 3 + (k == N), k % 2 + 1
            qp.set("idxb", k, list(range(nbu)) + [nuk + i for i in range(nbx)])
            qp.set("lbu", k, -rng.random(nbu)); qp.set("ubu", k, rng.random(nbu) + 0.0 * (k == 1))
            qp.set("lbx", k, -rng.random(nbx)); qp.set("ubx", k, np.zeros(nbx))   # zeros: -0.0 after negation
            qp.set("C", k, rng.standard_normal((ng, nx))); qp.set("D", k, rng.standard_normal((ng, nuk)))
            qp.set("lg", k, -rng.random(ng)); qp.set("ug", k, rng.random(ng))
            if k % 2 and nbx:
                ns = 2
                qp.set("idxs_rev", k, [-1] * nbu + [0] + [-1] * (nbx - 1) + [1] + [-1] * (ng - 1))
                for f in ("zl", "zu", "Zl", "Zu", "lls", "lus"):
                    qp.set(f, k, rng.random(ns))
    qp.make_consistent()
    return qp


def _unconstrained(rng, N=4, nx=3, nu=2):
    qp = OcpQp(N)
    for k in range(N + 1):
        nuk = nu if k < N else 0
        qp.set("Q", k, np.eye(nx)); qp.set("R", k, np.eye(nuk)); qp.set("q", k, rng.standard_normal(nx))
        qp.set("r", k, rng.standard_normal(nuk))
        if k < N:
            qp.set("A", k, rng.standard_normal((nx, nx))); qp.set("B", k, rng.standard_normal((nx, nuk)))
            qp.set("b", k, rng.standard_normal(nx))
    qp.make_consistent()
    return qp


FAMILIES = {
    "random_soft_general_masked": lambda rng: _masked(rng, [random_ocp_qp(rng, soft=True, general=True) for _ in range(3)]),
    "stage_varying": lambda rng: [_varying(rng) for _ in range(3)],
    "unconstrained": lambda rng: [_unconstrained(rng) for _ in range(3)],
    "hard_and_soft_stages": lambda rng: [random_ocp_qp(rng, N=5, soft=True, general=False) for _ in range(3)],
}


def _existing(qp):
    """(field, stage) pairs with at least one element: the sources the assembly takes."""
    return [(f, k) for f in DATA_FIELDS for k in range(qp.N + (0 if f in DYNAMICS_FIELDS else 1)) if qp._f[f][k].size > 0]


def _src(f, k, arr, batched=True):
    """A source for numpy array arr: (nbatch, *dims) if batched, else (*dims) broadcast; any strides."""
    st = [s // 8 for s in arr.strides]
    sb = st.pop(0) if batched else 0
    sr, sc = (st[0], st[1]) if len(st) == 2 else (st[0], 0)
    return (FIELD_IDS[f], k, arr.ctypes.data, sb, sr, sc)


def _run(emul, shape, nbatch, srcs):
    arr = (CuipmSrc * max(1, len(srcs)))(*[CuipmSrc(*s) for s in srcs])
    out = np.full((nbatch, Layout(shape).qp_stride), np.nan)
    rc = emul.emul_assemble(C.byref(shape.as_ctypes()), nbatch, arr, len(srcs), out.ctypes.data)
    return rc, out


def _stacked_sources(qps):
    """One batched source per (field, stage), plus the arrays behind them (kept alive by the caller)."""
    keep, srcs = [], []
    for f, k in _existing(qps[0]):
        a = np.stack([np.asarray(q._f[f][k], dtype=float) for q in qps])
        keep.append(a)
        srcs.append(_src(f, k, a))
    return srcs, keep


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


# ---- CPU: the kernel body against the host packer ----------------------------------------------------------------------

@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_emulated_assembly_matches_the_packer(emul, family):
    qps = FAMILIES[family](np.random.default_rng(5))
    want = PackedBatch(qps, eliminate=False)
    srcs, keep = _stacked_sources(qps)
    rc, out = _run(emul, want.shape, len(qps), srcs)
    assert rc == 0, emul.emul_assemble_error().decode()
    assert np.array_equal(_bits(out), _bits(want.qp))


def test_emulated_assembly_source_layouts(emul):
    """Broadcast sources (batch stride 0), transposed and sliced views and stage stacks give the same bits."""
    rng = np.random.default_rng(9)
    qps = [random_ocp_qp(rng, soft=True, general=True) for _ in range(4)]
    for k in range(qps[0].N):                      # dynamics shared by the batch: broadcast
        for q in qps[1:]:
            q.set("A", k, qps[0].A[k]); q.set("B", k, qps[0].B[k])
    want = PackedBatch(qps, eliminate=False)
    N, keep, srcs = qps[0].N, [], []
    for f, k in _existing(qps[0]):
        a = np.stack([np.asarray(q._f[f][k], dtype=float) for q in qps])
        if f in ("A", "B"):
            a = np.ascontiguousarray(a[0])
            srcs.append(_src(f, k, a, batched=False))
        elif f in ("Q", "C"):                      # stored transposed, passed as a transposed view
            t = np.ascontiguousarray(np.swapaxes(a, 1, 2))
            keep.append(t)
            srcs.append(_src(f, k, np.swapaxes(t, 1, 2)))
            continue
        elif f in ("r", "lbu", "Zl"):              # every other column of a wider array, batch-minor
            w = np.zeros((a.shape[1] * 2, a.shape[0]))
            w[::2] = a.T
            keep.append(w)
            srcs.append(_src(f, k, w[::2].T))
            continue
        elif f == "q":
            continue                               # below: one stack over the stages
        else:
            srcs.append(_src(f, k, a))
        keep.append(a)
    qs = np.stack([np.stack([q.q[k] for k in range(N + 1)]) for q in qps])   # (nbatch, N+1, nx)
    srcs += [(FIELD_IDS["q"], k, qs.ctypes.data + 8 * k * qs.strides[1] // 8, qs.strides[0] // 8, qs.strides[2] // 8, 0)
             for k in range(N + 1)]
    rc, out = _run(emul, want.shape, len(qps), srcs)
    assert rc == 0, emul.emul_assemble_error().decode()
    assert np.array_equal(_bits(out), _bits(want.qp))


def test_emulated_assembly_without_sources_is_the_empty_record(emul):
    qp = random_ocp_qp(np.random.default_rng(1), soft=True, general=True)
    sh = PackedBatch([qp], eliminate=False).shape
    rc, out = _run(emul, sh, 2, [])
    assert rc == 0 and np.array_equal(_bits(out), _bits(Layout(sh).new_qp(2)))


def test_emulated_assembly_refuses_bad_sources(emul):
    qp = random_ocp_qp(np.random.default_rng(2), N=4, soft=True, general=True)
    sh = PackedBatch([qp], eliminate=False).shape
    a = np.zeros((2, 8, 8))
    ok = _src("q", 1, a[:, 0, :4])
    for bad, why in (([ok, ok], "given twice"),
                     ([_src("A", 4, a[:, :4, :4])], "does not exist"),      # dynamics at N
                     ([_src("zl", 0, a[:, 0, :2])], "does not exist"),      # no slacks at stage 0
                     ([(FIELD_IDS["S"], 4, a.ctypes.data, 0, 1, 1)], "does not exist"),   # no inputs at N
                     ([(FIELD_IDS["q"], 1, a.ctypes.data, 8, -1, 0)], "negative stride"),
                     ([(FIELD_IDS["q"], 9, a.ctypes.data, 8, 1, 0)], "out of range"),
                     ([(99, 1, a.ctypes.data, 8, 1, 0)], "no such field")):
        rc, out = _run(emul, sh, 2, bad)
        assert rc == -1 and why in emul.emul_assemble_error().decode(), (why, emul.emul_assemble_error())
    rc, _ = _run(emul, sh, 2, [_src("q", 1, a[:, 0, 3::-1])])              # a reversed view: negative strides
    assert rc == -1 and "negative stride" in emul.emul_assemble_error().decode()


# ---- CPU: the front end's argument checks (no launch, no device needed) ----------------------------------------------

def test_tensor_front_end_checks_its_arguments():
    import torch
    from acados_b200.tensor_batch import TensorFields
    qp = random_ocp_qp(np.random.default_rng(3), N=4, nx=4, nu=2, soft=True, general=True)
    tf = TensorFields(qp, 8, device=0)
    with pytest.raises(TypeError, match="float64"):
        tf.resolve("lbx", 0, torch.zeros(8, 4, dtype=torch.float32))
    with pytest.raises(TypeError, match="torch.Tensor"):
        tf.resolve("lbx", 0, np.zeros((8, 4)))
    with pytest.raises(ValueError, match="shape"):
        tf.resolve("lbx", 0, torch.zeros(8, 3, dtype=torch.float64))
    with pytest.raises(ValueError, match="shape"):
        tf.resolve("q", None, torch.zeros(8, 4, 4, dtype=torch.float64))    # 5 stages carry q
    with pytest.raises(ValueError, match="on cpu"):
        tf.resolve("lbx", 0, torch.zeros(8, 4, dtype=torch.float64))
    with pytest.raises(ValueError, match="on cpu"):
        tf.resolve("A", 1, torch.zeros(4, 4, dtype=torch.float64))          # broadcast shape, but on the host
    for f in ("idxb", "idxs_rev", "idxe"):
        with pytest.raises(ValueError, match="index field"):
            tf.resolve(f, 0, torch.zeros(8, 4, dtype=torch.float64))
    with pytest.raises(ValueError, match="does not exist"):
        tf.resolve("A", 4, torch.zeros(4, 4, dtype=torch.float64))          # dynamics at N
    with pytest.raises(ValueError, match="does not exist"):
        tf.resolve("zl", 0, torch.zeros(2, dtype=torch.float64))            # no slacks at stage 0
    with pytest.raises(ValueError, match="not recognized"):
        tf.resolve("x0", 0, torch.zeros(4, dtype=torch.float64))


# ---- GPU ----------------------------------------------------------------------------------------------------------------

def _tensor_solver(qps, opts, stage_none=("q",)):
    """An OcpQpTensorBatchSolver on qps[0]'s structure with every field set from the batch's values (fields in stage_none
    as one stack over the stages); returns the solver and the tensors behind it."""
    import torch
    from acados_b200.tensor_batch import OcpQpTensorBatchSolver
    tb = OcpQpTensorBatchSolver(qps[0], len(qps), opts)
    ts = {}
    for f, k in _existing(qps[0]):
        if f in stage_none:
            continue
        ts[(f, k)] = torch.from_numpy(np.stack([np.asarray(q._f[f][k], dtype=float) for q in qps])).cuda()
        tb.set(f, k, ts[(f, k)])
    for f in stage_none:
        stages = sorted(tb.fields.dims[f])
        ts[(f, None)] = torch.from_numpy(np.stack([np.stack([q._f[f][k] for k in stages]) for q in qps])).cuda()
        tb.set(f, None, ts[(f, None)])
    return tb, ts


def _same_solution(b, tb, N):
    for k in range(N + 1):
        for f in ("x", "u", "sl", "su", "lam", "t") + (("pi",) if k < N else ()):
            assert _bits(tb.get(k, f).cpu().numpy()).tobytes() == _bits(b.get(k, f)).tobytes(), (k, f)
    want, got = b.info, tb.info
    for f in ("status", "iter", "res_max", "mu", "obj", "dual_gap", "lq_count"):
        assert got[f].tobytes() == want[f].tobytes(), f
    assert tb.stat.cpu().numpy().tobytes() == b.stat.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("family", sorted(FAMILIES) + ["chain_mass_sized"])
def test_device_assembly_matches_the_packer(built, family):
    import torch
    rng = np.random.default_rng(21)
    qps = ([random_ocp_qp(rng, N=40, nx=21, nu=3, soft=True, general=False) for _ in range(16)] if family == "chain_mass_sized"
           else FAMILIES[family](rng))
    tb, _ = _tensor_solver(qps, OcpQpOptions())
    rec = tb.assemble()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(rec.cpu().numpy()), _bits(PackedBatch(qps, eliminate=False).qp))
    tb.close()


def _new_data(rng, qps):
    """New x0 and cost gradients: what an MPC loop changes from one step to the next."""
    for q in qps:
        x0 = q.lbx[0] + 0.05 * rng.standard_normal(q.lbx[0].shape)
        q.set("lbx", 0, x0); q.set("ubx", 0, x0)
        for k in range(q.N + 1):
            q.set("q", k, q.q[k] + 0.01 * rng.standard_normal(q.q[k].shape))


@pytest.mark.gpu
@pytest.mark.parametrize("solver,cond_N", [("PARTIAL_CONDENSING_CUIPM", None), ("PARTIAL_CONDENSING_CUIPM", 5),
                                           ("FULL_CONDENSING_CUIPM", None)])
def test_tensor_solver_matches_the_batch_solver(built, solver, cond_N):
    """Cold solve, in-place tensor update, warm_start = 2 solve: bit-identical to OcpQpBatchSolver on the same QPs."""
    import torch
    rng = np.random.default_rng(31)
    qps = [random_ocp_qp(rng, N=12, nx=5, nu=2, soft=True, general=True) for _ in range(64)]
    mk = lambda: OcpQpOptions(qp_solver=solver, cond_N=cond_N)
    b = OcpQpBatchSolver(qps, mk())
    tb, ts = _tensor_solver(qps, mk())
    st = b.solve()
    tst = tb.solve()
    assert np.array_equal(tst.cpu().numpy(), st)
    _same_solution(b, tb, qps[0].N)
    _new_data(rng, qps)
    b.update(qps)
    ts[("lbx", 0)].copy_(torch.from_numpy(np.stack([q.lbx[0] for q in qps])))
    ts[("ubx", 0)].copy_(torch.from_numpy(np.stack([q.ubx[0] for q in qps])))
    ts[("q", None)].copy_(torch.from_numpy(np.stack([np.stack(q.q) for q in qps])))
    b.c_opts.warm_start = tb.c_opts.warm_start = 2
    st = b.solve()
    tst = tb.solve()
    assert np.array_equal(tst.cpu().numpy(), st)
    _same_solution(b, tb, qps[0].N)
    b.close(); tb.close()


@pytest.mark.gpu
def test_tensor_solver_split_matches_the_batch_solver(built):
    """condense_lhs, a new x0 set in place, condense_rhs_and_solve: the bits of OcpQpBatchSolver's split."""
    import torch
    rng = np.random.default_rng(41)
    qps = [random_ocp_qp(rng, N=10, nx=4, nu=2, soft=True, general=True) for _ in range(32)]
    b = OcpQpBatchSolver(qps, OcpQpOptions(cond_N=3))
    tb, ts = _tensor_solver(qps, OcpQpOptions(cond_N=3))
    b.condense_lhs(); tb.condense_lhs()
    for q in qps:
        x0 = q.lbx[0] + 0.1
        q.set("lbx", 0, x0); q.set("ubx", 0, x0)
    b.update(qps)
    ts[("lbx", 0)].add_(0.1); ts[("ubx", 0)].add_(0.1)
    st = b.condense_rhs_and_solve()
    tst = tb.condense_rhs_and_solve()
    assert np.array_equal(tst.cpu().numpy(), st)
    _same_solution(b, tb, qps[0].N)
    b.close(); tb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cond_N", [None, 4])
def test_xcond_device_entry_matches_the_host_entry(built, cond_N):
    """cuipm_xcond_solve_device on records copied to the device: the bits of cuipm_xcond_solve_host, statistics included;
    sensitivities through the chain's solver afterwards are the same too."""
    import torch
    from acados_b200.binding import STAT_M, CuipmXcond, _CLayout, default_opts
    rng = np.random.default_rng(51)
    qps = [random_ocp_qp(rng, N=10, soft=True, general=True) for _ in range(48)]
    full = PackedBatch(qps, eliminate=False)
    idxe0, nb = [int(i) for i in qps[0].idxe[0]], len(qps)
    o = default_opts()
    xh = CuipmXcond(full.shape, idxe0, cond_N or full.N, nb)
    xd = CuipmXcond(full.shape, idxe0, cond_N or full.N, nb)
    sol, info, stat = xh.solve(full.qp, o, want_stat=True)
    d_qp = torch.from_numpy(full.qp).cuda()
    d_sol = torch.zeros((nb, full.layout.sol_stride), dtype=torch.float64, device="cuda")
    d_info = torch.zeros((nb, INFO_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    d_stat = torch.zeros((nb, o.stat_max + 1, STAT_M), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    xd.solve_device(nb, d_qp.data_ptr(), d_sol.data_ptr(), d_info.data_ptr(), o, d_stat.data_ptr(), sync=True)
    assert d_sol.cpu().numpy().tobytes() == sol.tobytes()
    got = d_info.cpu().numpy().view(INFO_DTYPE).reshape(nb)
    for f in ("status", "iter", "res_max", "mu", "obj", "dual_gap", "lq_count"):
        assert got[f].tobytes() == info[f].tobytes(), f
    assert d_stat.cpu().numpy().tobytes() == stat.tobytes()
    lib = xh.lib
    sh_h, sh_d = xh.solver_handle, xd.solver_handle
    sol_stride = C.cast(lib.cuipm_get_layout(sh_h), C.POINTER(_CLayout)).contents.sol_stride
    seed = np.random.default_rng(7).standard_normal((nb, sol_stride))
    for adjoint in (0, 1):
        a, d = np.zeros_like(seed), np.zeros_like(seed)
        assert lib.cuipm_sens_host(sh_h, nb, seed.ctypes.data, a.ctypes.data, adjoint, C.byref(o)) == 0
        assert lib.cuipm_sens_host(sh_d, nb, seed.ctypes.data, d.ctypes.data, adjoint, C.byref(o)) == 0
        assert a.tobytes() == d.tobytes()
    xh.close(); xd.close()


@pytest.mark.gpu
def test_tensor_solver_orders_itself_after_the_current_stream(built):
    """Inputs written by a torch kernel on a non-default current stream right before solve, no synchronise in between: the
    results are those of a synchronised run."""
    import torch
    rng = np.random.default_rng(61)
    qps = [random_ocp_qp(rng, N=10, nx=4, nu=2, soft=True, general=True) for _ in range(64)]
    tb, ts = _tensor_solver(qps, OcpQpOptions())
    x0 = ts[("lbx", 0)].clone()
    tb.solve()
    torch.cuda.synchronize()
    ref_x = [tb.get(k, "x").clone() for k in range(qps[0].N + 1)]
    ref_stat = tb.stat.clone()
    ts[("lbx", 0)].zero_(); ts[("ubx", 0)].zero_()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)              # keeps the stream busy so that an unordered solve would read the zeros
        ts[("lbx", 0)].copy_(x0); ts[("ubx", 0)].copy_(x0)
        tb.solve()
        xs = [tb.get(k, "x") * 1.0 for k in range(qps[0].N + 1)]
        stat = tb.stat * 1.0
    torch.cuda.synchronize()
    for k in range(qps[0].N + 1):
        assert torch.equal(xs[k], ref_x[k]), k
    assert torch.equal(stat, ref_stat)
    tb.close()
