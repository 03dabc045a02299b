"""ctypes binding of the C ABI in ``include/cuipm.h`` (libcuipm.so, built in-tree by ``__graft_entry__.build``).

The library is the product: hand-written sm_90a CUDA kernels behind plain-C entry points.  There is no
CPU fallback -- if the shared object is missing, or no CUDA device is present, the solve calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .problems import Batch, Layout, Shape

_HERE = os.path.dirname(os.path.abspath(__file__))
def host_threads() -> int:
    """Host threads this process can actually run at once: the affinity mask, capped by the cgroup CPU quota (a container may
    see 128 CPUs and be allowed 16 CPUs' worth of time; a thread team sized from the mask then spends its quota spinning)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = max(1, min(n, int(-(-int(quota) // int(period)))))
    except Exception:  # noqa: BLE001
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = max(1, min(n, -(-q // per)))
        except Exception:  # noqa: BLE001
            pass
    return n


LIB_PATH = os.environ.get("CUIPM_LIB") or os.path.join(_HERE, "csrc", "libcuipm.so")

STAT_M = 20
STATUS_NAMES = {0: "SUCCESS", 1: "MAX_ITER", 2: "MIN_STEP", 3: "NAN_SOL", 4: "INCONS_EQ"}
MODES = {"SPEED_ABS": 0, "SPEED": 1, "BALANCE": 2, "ROBUST": 3}


class CuipmOpts(C.Structure):
    """Mirror of ``struct cuipm_opts``."""
    _fields_ = [("mode", C.c_int), ("iter_max", C.c_int), ("stat_max", C.c_int), ("mu0", C.c_double),
                ("alpha_min", C.c_double), ("res_g_max", C.c_double), ("res_b_max", C.c_double),
                ("res_d_max", C.c_double), ("res_m_max", C.c_double), ("dual_gap_max", C.c_double),
                ("reg_prim", C.c_double), ("lam_min", C.c_double), ("t_min", C.c_double), ("tau_min", C.c_double),
                ("lam0_min", C.c_double), ("t0_min", C.c_double), ("pred_corr", C.c_int), ("cond_pred_corr", C.c_int),
                ("itref_pred_max", C.c_int), ("itref_corr_max", C.c_int), ("lq_fact", C.c_int), ("warm_start", C.c_int),
                ("abs_form", C.c_int), ("comp_dual_sol_eq", C.c_int), ("comp_res_exit", C.c_int),
                ("split_step", C.c_int), ("var_init_scheme", C.c_int), ("t_lam_min", C.c_int), ("t0_init", C.c_int),
                ("m_relax", C.c_double)]


class CuipmInfo(C.Structure):
    """Mirror of ``struct cuipm_info``."""
    _fields_ = [("status", C.c_int), ("iter", C.c_int), ("res_max", C.c_double * 4), ("mu", C.c_double),
                ("obj", C.c_double), ("dual_gap", C.c_double), ("lq_count", C.c_int), ("reserved", C.c_int)]


INFO_DTYPE = np.dtype([("status", np.int32), ("iter", np.int32), ("res_max", np.float64, (4,)), ("mu", np.float64),
                       ("obj", np.float64), ("dual_gap", np.float64), ("lq_count", np.int32), ("reserved", np.int32)],
                      align=True)
assert INFO_DTYPE.itemsize == C.sizeof(CuipmInfo)

# enum cuipm_field: the per-field sources of cuipm_xcond_assemble_device, under AcadosOcpQp's field names
FIELD_IDS = {f: i for i, f in enumerate(("A", "B", "b", "Q", "R", "S", "q", "r", "lbu", "ubu", "lbx", "ubx", "C", "D", "lg", "ug",
                                         "Zl", "Zu", "zl", "zu", "lls", "lus", "lbu_mask", "ubu_mask", "lbx_mask", "ubx_mask",
                                         "lg_mask", "ug_mask", "lls_mask", "lus_mask"))}


class CuipmSrc(C.Structure):
    """Mirror of ``struct cuipm_src``: one field of one stage, element (r, c) of QP q at ptr[q*s_batch + r*s_row + c*s_col]."""
    _fields_ = [("field", C.c_int), ("stage", C.c_int), ("ptr", C.c_void_p), ("s_batch", C.c_longlong), ("s_row", C.c_longlong),
                ("s_col", C.c_longlong)]


_lib: Optional[C.CDLL] = None


def load_library(path: str = LIB_PATH) -> C.CDLL:
    """Loads libcuipm.so; raises if the extension has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
                           "g.build()'); the cuipm solver has no CPU fallback")
    lib = C.CDLL(path)
    vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.c_int
    lib.cuipm_opts_set_default.argtypes = [C.POINTER(CuipmOpts), ip]
    lib.cuipm_opts_set_default_acados.argtypes = [C.POINTER(CuipmOpts), ip]
    lib.cuipm_opts_set.argtypes = [C.POINTER(CuipmOpts), C.c_char_p, vp]
    lib.cuipm_opts_set.restype = ip
    lib.cuipm_opts_get.argtypes = [C.POINTER(CuipmOpts), C.c_char_p, vp]
    lib.cuipm_opts_get.restype = ip
    lib.cuipm_layout_create.argtypes = [vp]
    lib.cuipm_layout_create.restype = vp
    lib.cuipm_layout_destroy.argtypes = [vp]
    lib.cuipm_create.argtypes = [vp, ip, ip]
    lib.cuipm_create.restype = vp
    lib.cuipm_destroy.argtypes = [vp]
    lib.cuipm_get_layout.argtypes = [vp]
    lib.cuipm_get_layout.restype = vp
    lib.cuipm_last_error.restype = C.c_char_p
    lib.cuipm_solve_host.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(CuipmOpts)]
    lib.cuipm_solve_host.restype = ip
    lib.cuipm_solve_host_async.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(CuipmOpts)]
    lib.cuipm_solve_host_async.restype = ip
    lib.cuipm_wait.argtypes = [vp]
    lib.cuipm_wait.restype = ip
    lib.cuipm_solve_device.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(CuipmOpts), ip]
    lib.cuipm_solve_device.restype = ip
    for name in ("cuipm_device_qp_buffer", "cuipm_device_sol_buffer", "cuipm_device_info_buffer", "cuipm_stream"):
        getattr(lib, name).argtypes = [vp]
        getattr(lib, name).restype = vp
    lib.cuipm_get_ric.argtypes = [vp, ip, C.c_char_p, ip, vp, ip, ip]
    lib.cuipm_get_ric.restype = ip
    lib.cuipm_last_launch_count.argtypes = [vp]
    lib.cuipm_last_launch_count.restype = ip
    lib.cuipm_last_kernel_ms.argtypes = [vp]
    lib.cuipm_last_kernel_ms.restype = C.c_float
    lib.cuipm_sens_host.argtypes = [vp, ip, vp, vp, ip, C.POINTER(CuipmOpts)]
    lib.cuipm_sens_host.restype = ip
    lib.cuipm_sens_device.argtypes = [vp, ip, vp, vp, vp, ip, C.POINTER(CuipmOpts), ip]
    lib.cuipm_sens_device.restype = ip
    lib.cuipm_reducer_create.argtypes = [vp, ip, C.POINTER(C.c_int), ip]
    lib.cuipm_reducer_create.restype = vp
    lib.cuipm_reducer_destroy.argtypes = [vp]
    for name in ("cuipm_reducer_reduced_shape", "cuipm_reducer_full_layout", "cuipm_reducer_reduced_layout"):
        getattr(lib, name).argtypes = [vp]
        getattr(lib, name).restype = vp
    lib.cuipm_reduce_device.argtypes = [vp, ip, vp, vp, vp]
    lib.cuipm_reduce_device.restype = ip
    lib.cuipm_restore_device.argtypes = [vp, ip, vp, vp, vp, C.c_double, C.c_double, vp]
    lib.cuipm_restore_device.restype = ip
    lib.cuipm_condenser_create.argtypes = [vp, ip, ip]
    lib.cuipm_condenser_create.restype = vp
    lib.cuipm_condenser_destroy.argtypes = [vp]
    lib.cuipm_condenser_condensed_shape.argtypes = [vp]
    lib.cuipm_condenser_condensed_shape.restype = vp
    lib.cuipm_condense_device.argtypes = [vp, ip, vp, vp, vp]
    lib.cuipm_condense_device.restype = ip
    for f in (lib.cuipm_condense_lhs_device, lib.cuipm_condense_rhs_device):
        f.argtypes = [vp, ip, vp, vp, vp]
        f.restype = ip
    lib.cuipm_expand_device.argtypes = [vp, ip, vp, vp, vp, vp]
    lib.cuipm_expand_device.restype = ip
    lib.cuipm_xcond_create.argtypes = [vp, ip, C.POINTER(C.c_int), ip, ip, ip]
    lib.cuipm_xcond_create.restype = vp
    lib.cuipm_xcond_destroy.argtypes = [vp]
    lib.cuipm_xcond_solver.argtypes = [vp]
    lib.cuipm_xcond_solver.restype = vp
    for f in (lib.cuipm_xcond_solve_host, lib.cuipm_xcond_condense_rhs_and_solve_host):
        f.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(CuipmOpts)]
        f.restype = ip
    lib.cuipm_xcond_condense_lhs_host.argtypes = [vp, ip, vp]
    lib.cuipm_xcond_condense_lhs_host.restype = ip
    for f in (lib.cuipm_xcond_solve_device, lib.cuipm_xcond_condense_rhs_and_solve_device):
        f.argtypes = [vp, ip, vp, vp, vp, vp, C.POINTER(CuipmOpts), ip]
        f.restype = ip
    lib.cuipm_xcond_condense_lhs_device.argtypes = [vp, ip, vp, ip]
    lib.cuipm_xcond_condense_lhs_device.restype = ip
    lib.cuipm_xcond_assemble_device.argtypes = [vp, ip, C.POINTER(CuipmSrc), ip, vp, ip]
    lib.cuipm_xcond_assemble_device.restype = ip
    lib.cuipm_set_tuning.argtypes = [vp, C.c_char_p, ip]
    lib.cuipm_set_tuning.restype = ip
    lib.cuipm_last_handed_back.argtypes = [vp]
    lib.cuipm_last_handed_back.restype = ip
    lib.cuipm_last_main_kernel_ms.argtypes = [vp]
    lib.cuipm_last_main_kernel_ms.restype = C.c_float
    _lib = lib
    return lib


def default_opts(mode: str = "BALANCE", acados: bool = True, **overrides) -> CuipmOpts:
    """Options as the reference's plugin would hold them (``acados=True``: HPIPM mode defaults plus the acados
    overrides, i.e. what PARTIAL_CONDENSING_HPIPM runs with; keyword overrides use the struct field names)."""
    lib = load_library()
    o = CuipmOpts()
    (lib.cuipm_opts_set_default_acados if acados else lib.cuipm_opts_set_default)(C.byref(o), MODES[mode])
    for k, v in overrides.items():
        if not hasattr(o, k):
            raise KeyError(k)
        setattr(o, k, v)
    if o.stat_max < o.iter_max:
        o.stat_max = o.iter_max
    return o


class _CLayout(C.Structure):
    _fields_ = ([("N", C.c_int), ("qp_stride", C.c_size_t)]
                + [(n, C.POINTER(C.c_size_t)) for n in ("qp_stage", "off_BAt", "off_RSQ", "off_DCt", "off_b", "off_rq",
                                                          "off_d", "off_dmask", "off_Z", "off_z")]
                + [("sol_stride", C.c_size_t)]
                + [(n, C.POINTER(C.c_size_t)) for n in ("sol_stage", "off_ux", "off_pi", "off_lam", "off_t")])


def c_layout_as_dict(ptr: int, N: int) -> dict:
    """Reads a ``cuipm_layout*`` into python lists (used to cross-check the numpy Layout)."""
    l = C.cast(ptr, C.POINTER(_CLayout)).contents
    out = {"qp_stride": l.qp_stride, "sol_stride": l.sol_stride}
    for n, _ in _CLayout._fields_:
        if n in ("N", "qp_stride", "sol_stride"):
            continue
        cnt = N + 2 if n.endswith("_stage") else N + 1
        out[n] = [getattr(l, n)[i] for i in range(cnt)]
    return out


class CuipmSolver:
    """Batched OCP-QP solver on one CUDA device (thin object wrapper over the C ABI)."""

    def __init__(self, shape: Shape, max_batch: int, device: int = 0):
        self.lib = load_library()
        self.shape = shape
        self.layout = Layout(shape)
        self.max_batch = max_batch
        self._cshape = shape.as_ctypes()
        self.handle = self.lib.cuipm_create(C.byref(self._cshape), max_batch, device)
        if not self.handle:
            raise RuntimeError("cuipm_create failed: " + self.lib.cuipm_last_error().decode())

    def close(self):
        if self.handle:
            self.lib.cuipm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"cuipm error {rc}: " + self.lib.cuipm_last_error().decode())

    def solve(self, qp: np.ndarray, opts: Optional[CuipmOpts] = None, sol0: Optional[np.ndarray] = None,
              want_stat: bool = False):
        """Host-buffer solve (H2D, kernel, D2H inside): returns (sol, info[, stat])."""
        opts = opts or default_opts()
        nb = qp.shape[0]
        assert qp.dtype == np.float64 and qp.flags.c_contiguous and qp.shape[1] == self.layout.qp_stride
        sol = np.zeros((nb, self.layout.sol_stride)) if sol0 is None else np.ascontiguousarray(sol0, dtype=np.float64).copy()
        info = np.zeros(nb, dtype=INFO_DTYPE)
        stat = np.zeros((nb, opts.stat_max + 1, STAT_M)) if want_stat else None
        rc = self.lib.cuipm_solve_host(self.handle, nb, qp.ctypes.data, sol.ctypes.data, info.ctypes.data,
                                       stat.ctypes.data if want_stat else None, C.byref(opts))
        self._check(rc)
        return (sol, info, stat) if want_stat else (sol, info)

    def solve_host_async(self, nbatch: int, h_qp: int, h_sol: int, h_info: int, opts: CuipmOpts, h_stat: int = 0):
        """Enqueue a host-buffer solve (raw pointers to PINNED host memory) and return; ``wait()`` completes it."""
        self._check(self.lib.cuipm_solve_host_async(self.handle, nbatch, h_qp, h_sol, h_info, h_stat or None, C.byref(opts)))

    def wait(self):
        self._check(self.lib.cuipm_wait(self.handle))

    def solve_device(self, nbatch: int, d_qp: int, d_sol: int, d_info: int, opts: CuipmOpts, sync: bool = True,
                     d_stat: int = 0):
        self._check(self.lib.cuipm_solve_device(self.handle, nbatch, d_qp, d_sol, d_info, d_stat or None,
                                                C.byref(opts), 1 if sync else 0))

    def sens(self, seed: np.ndarray, opts: Optional[CuipmOpts] = None, adjoint: bool = False) -> np.ndarray:
        """Forward / adjoint solution sensitivities for one seed per QP of the preceding ``solve`` (records in the
        solution layout: (seed_g, seed_b, seed_d, seed_m) in the (ux, pi, lam, t) slots)."""
        opts = opts or default_opts()
        seed = np.ascontiguousarray(seed, dtype=np.float64)
        assert seed.ndim == 2 and seed.shape[1] == self.layout.sol_stride
        out = np.zeros_like(seed)
        self._check(self.lib.cuipm_sens_host(self.handle, seed.shape[0], seed.ctypes.data, out.ctypes.data,
                                             1 if adjoint else 0, C.byref(opts)))
        return out

    def sens_device(self, nbatch: int, d_qp: int, d_seed: int, d_sens: int, opts: CuipmOpts, adjoint: bool = False,
                    sync: bool = True):
        self._check(self.lib.cuipm_sens_device(self.handle, nbatch, d_qp, d_seed, d_sens, 1 if adjoint else 0,
                                               C.byref(opts), 1 if sync else 0))

    def set_tuning(self, key: str, value: int):
        self._check(self.lib.cuipm_set_tuning(self.handle, key.encode(), value))

    @property
    def last_kernel_ms(self) -> float:
        return float(self.lib.cuipm_last_kernel_ms(self.handle))

    @property
    def last_main_kernel_ms(self) -> float:
        return float(self.lib.cuipm_last_main_kernel_ms(self.handle))

    @property
    def last_handed_back(self) -> int:
        return int(self.lib.cuipm_last_handed_back(self.handle))

    @property
    def last_launch_count(self) -> int:
        return int(self.lib.cuipm_last_launch_count(self.handle))

    def get_ric(self, iqp: int, field: str, stage: int, shape2):
        out = np.zeros(shape2[::-1])  # column-major (size1 x size2)
        self._check(self.lib.cuipm_get_ric(self.handle, iqp, field.encode(), stage, out.ctypes.data, shape2[0], shape2[1]))
        return out.T


def _shape_from_c(ptr: int) -> Shape:
    """Python copy of a ``const cuipm_shape *`` owned by a C object."""
    class _CS(C.Structure):
        _fields_ = [("N", C.c_int)] + [(n, C.POINTER(C.c_int)) for n in ("nx", "nu", "nb", "ng", "ns")] + \
                   [("idxb", C.POINTER(C.POINTER(C.c_int))), ("idxs_rev", C.POINTER(C.POINTER(C.c_int)))]
    cs = C.cast(ptr, C.POINTER(_CS)).contents
    N = cs.N
    g = lambda a: [int(a[k]) for k in range(N + 1)]
    nx, nu, nb, ng, ns = g(cs.nx), g(cs.nu), g(cs.nb), g(cs.ng), g(cs.ns)
    return Shape(N, nx, nu, nb, ng, ns, [[int(cs.idxb[k][i]) for i in range(nb[k])] for k in range(N + 1)],
                 [[int(cs.idxs_rev[k][i]) for i in range(nb[k] + ng[k])] for k in range(N + 1)])


class CuipmCondenser:
    """Partial (block) condensing / expansion on the device (``cuipm_condenser_*``, include/cuipm.h)."""

    def __init__(self, shape: Shape, cond_N: int, device: int = 0):
        self.lib = load_library()
        self.shape = shape
        self._cshape = shape.as_ctypes()
        self.handle = self.lib.cuipm_condenser_create(C.byref(self._cshape), cond_N, device)
        if not self.handle:
            raise RuntimeError("cuipm_condenser_create failed: " + self.lib.cuipm_last_error().decode())
        self.condensed_shape = _shape_from_c(self.lib.cuipm_condenser_condensed_shape(self.handle))
        self.layout, self.condensed_layout = Layout(shape), Layout(self.condensed_shape)

    def condense(self, nbatch: int, d_qp: int, d_qp_cond: int, stream: int = 0):
        if self.lib.cuipm_condense_device(self.handle, nbatch, d_qp, d_qp_cond, stream or None) != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def condense_lhs(self, nbatch: int, d_qp: int, d_qp_cond: int, stream: int = 0):
        """Condenses the QPs and keeps the prediction matrices of every stage on the device (the preparation phase of an SQP-RTI
        step: ``condense_lhs`` of the reference's xcond solver)."""
        if self.lib.cuipm_condense_lhs_device(self.handle, nbatch, d_qp, d_qp_cond, stream or None) != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def condense_rhs(self, nbatch: int, d_qp: int, d_qp_cond: int, stream: int = 0):
        """Refreshes the vectors of the condensed records from records with the same matrices and new vectors (the feedback
        phase: ``condense_rhs`` of the reference's xcond solver)."""
        if self.lib.cuipm_condense_rhs_device(self.handle, nbatch, d_qp, d_qp_cond, stream or None) != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def expand(self, nbatch: int, d_qp: int, d_sol_cond: int, d_sol: int, stream: int = 0):
        if self.lib.cuipm_expand_device(self.handle, nbatch, d_qp, d_sol_cond, d_sol, stream or None) != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def close(self):
        if self.handle:
            self.lib.cuipm_condenser_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CuipmXcond:
    """The whole xcond chain on the device behind one object (``cuipm_xcond_*``, include/cuipm.h): records of the shape the
    user poses in, solutions of that shape out; one pass, or the SQP-RTI split ``condense_lhs`` / ``condense_rhs_and_solve``."""

    def __init__(self, full_shape: Shape, idxe0, cond_N: int, max_batch: int, device: int = 0):
        self.lib = load_library()
        self.full_shape, self.layout = full_shape, Layout(full_shape)
        self._cshape = full_shape.as_ctypes()
        idx = (C.c_int * max(1, len(idxe0)))(*[int(i) for i in idxe0])
        self.handle = self.lib.cuipm_xcond_create(C.byref(self._cshape), len(idxe0), idx, cond_N, max_batch, device)
        if not self.handle:
            raise RuntimeError("cuipm_xcond_create failed: " + self.lib.cuipm_last_error().decode())

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def _solve(self, fn, qp_full, opts, want_stat):
        qp_full = np.ascontiguousarray(qp_full, dtype=np.float64)
        nb = qp_full.shape[0]
        sol = np.zeros((nb, self.layout.sol_stride))
        info = np.zeros(nb, dtype=INFO_DTYPE)
        stat = np.zeros((nb, opts.stat_max + 1, STAT_M)) if want_stat else None
        self._check(fn(self.handle, nb, qp_full.ctypes.data, sol.ctypes.data, info.ctypes.data,
                       stat.ctypes.data if want_stat else None, C.byref(opts)))
        return (sol, info, stat) if want_stat else (sol, info)

    def solve(self, qp_full, opts: CuipmOpts, want_stat: bool = False):
        """One pass: returns (sol, info[, stat]); with warm_start >= 2 the solve starts from this object's previous solution."""
        return self._solve(self.lib.cuipm_xcond_solve_host, qp_full, opts, want_stat)

    def condense_lhs(self, qp_full):
        qp_full = np.ascontiguousarray(qp_full, dtype=np.float64)
        self._check(self.lib.cuipm_xcond_condense_lhs_host(self.handle, qp_full.shape[0], qp_full.ctypes.data))

    def condense_rhs_and_solve(self, qp_full, opts: CuipmOpts, want_stat: bool = False):
        return self._solve(self.lib.cuipm_xcond_condense_rhs_and_solve_host, qp_full, opts, want_stat)

    # device-buffer entries: device pointers, work enqueued on ``stream``, a synchronise only with sync=True
    def solve_device(self, nbatch: int, d_qp: int, d_sol: int, d_info: int, opts: CuipmOpts, d_stat: int = 0, sync: bool = False):
        self._check(self.lib.cuipm_xcond_solve_device(self.handle, nbatch, d_qp, d_sol, d_info, d_stat or None, C.byref(opts),
                                                      1 if sync else 0))

    def condense_lhs_device(self, nbatch: int, d_qp: int, sync: bool = False):
        self._check(self.lib.cuipm_xcond_condense_lhs_device(self.handle, nbatch, d_qp, 1 if sync else 0))

    def condense_rhs_and_solve_device(self, nbatch: int, d_qp: int, d_sol: int, d_info: int, opts: CuipmOpts, d_stat: int = 0,
                                      sync: bool = False):
        self._check(self.lib.cuipm_xcond_condense_rhs_and_solve_device(self.handle, nbatch, d_qp, d_sol, d_info, d_stat or None,
                                                                       C.byref(opts), 1 if sync else 0))

    def assemble_device(self, nbatch: int, src, nsrc: int, d_qp: int, sync: bool = False):
        """Records of the full shape from per-field sources (a ``CuipmSrc`` array; include/cuipm.h)."""
        self._check(self.lib.cuipm_xcond_assemble_device(self.handle, nbatch, src, nsrc, d_qp, 1 if sync else 0))

    @property
    def solver_handle(self) -> int:
        """The inner ``cuipm_solver *`` (statistics, sensitivities: ``cuipm_xcond_solver``)."""
        return self.lib.cuipm_xcond_solver(self.handle)

    @property
    def stream(self) -> int:
        """The ``cudaStream_t`` the device entries enqueue on."""
        return self.lib.cuipm_stream(self.solver_handle)

    @property
    def last_kernel_ms(self) -> float:
        return float(self.lib.cuipm_last_kernel_ms(self.lib.cuipm_xcond_solver(self.handle)))

    def close(self):
        if self.handle:
            self.lib.cuipm_xcond_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CuipmReducer:
    """Stage-0 equality elimination / restore on the device (``cuipm_reducer_*``, include/cuipm.h): maps QP records of
    the shape the user poses (x0 a stage-0 equality) to records of the reduced shape and solutions back."""

    def __init__(self, full_shape: Shape, idxe0, device: int = 0):
        self.lib = load_library()
        self.full_shape = full_shape
        self._cshape = full_shape.as_ctypes()
        idx = (C.c_int * max(1, len(idxe0)))(*[int(i) for i in idxe0])
        self.handle = self.lib.cuipm_reducer_create(C.byref(self._cshape), len(idxe0), idx, device)
        if not self.handle:
            raise RuntimeError("cuipm_reducer_create failed: " + self.lib.cuipm_last_error().decode())
        self.reduced_shape = _shape_from_c(self.lib.cuipm_reducer_reduced_shape(self.handle))
        self.full_layout, self.reduced_layout = Layout(full_shape), Layout(self.reduced_shape)

    def reduce(self, nbatch: int, d_qp_full: int, d_qp_red: int, stream: int = 0):
        rc = self.lib.cuipm_reduce_device(self.handle, nbatch, d_qp_full, d_qp_red, stream or None)
        if rc != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def restore(self, nbatch: int, d_qp_full: int, d_sol_red: int, d_sol_full: int, lam_min: float, t_min: float, stream: int = 0):
        rc = self.lib.cuipm_restore_device(self.handle, nbatch, d_qp_full, d_sol_red, d_sol_full, lam_min, t_min, stream or None)
        if rc != 0:
            raise RuntimeError(self.lib.cuipm_last_error().decode())

    def close(self):
        if self.handle:
            self.lib.cuipm_reducer_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
