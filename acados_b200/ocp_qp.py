"""Host-side mirror of the reference's Python QP interface for the cuipm path.

``OcpQp`` carries an OCP-structured QP under the field names of ``acados_template.AcadosOcpQp``
(reference: interfaces/acados_template/acados_template/acados_ocp_qp.py:23-436 -- ``set``, ``make_consistent``,
``from_dict`` / ``from_json`` with zero-padded ``<field>_<stage>`` keys), ``OcpQpSolver`` mirrors
``AcadosOcpQpSolver`` (acados_ocp_qp_solver.py:51-510: ``solve``, ``get``, ``get_stats``, ``get_cost``,
``get_iterate``), and ``OcpQpBatchSolver`` is the batched form the reference does not have: many structurally
identical QPs, one launch.

What happens between the user's QP and the kernel is what the reference's xcond layer does for
PARTIAL_CONDENSING_HPIPM (acados/ocp_qp/ocp_qp_xcond_solver.c:523-669 in front of ocp_qp_partial_condensing.c:523-689):
the stage-0 state bounds marked as equalities (``idxe``: x0 = lbx_0) are eliminated before the solve
(d_ocp_qp_reduce_eq_dof, external/hpipm/ocp_qp/x_ocp_qp_red.c:278-560), the QP is block-condensed to cond_N stages if
cond_N < N, and after the solve the solution is expanded and the eliminated states are restored, multipliers included
(d_ocp_qp_restore_eq_dof, :848-994).  The data are packed into the cuipm QP records (include/cuipm.h, HPIPM's
conventions: BAt = [B'; A'], RSQ = [R S; S' Q] lower, DCt = [D'; C'], d = [lb, lg, -ub, -ug, lls, lus]); on the GPU
the uncondensed QP is usually the cheaper one to factorise, so cond_N defaults to N as in the reference.

By default the records travel as posed and that whole chain runs on the device in one cuipm_xcond object
(binding.CuipmXcond, acados_b200/csrc/cuipm_xcond.cu).  ``device_reduce=False`` runs the elimination and the restore
here, vectorised over the batch in numpy, and the condensing in acados_b200/condensing.py, and solves the records with
binding.CuipmSolver; the tests hold the device route to it.  Either way the solve is CUDA: no CPU fallback.
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np

from .binding import STAT_M, CuipmOpts, CuipmSolver, CuipmXcond, default_opts
from .problems import Layout, Shape

DYNAMICS_FIELDS = ("A", "B", "b")
COST_FIELDS = ("Q", "R", "S", "q", "r", "zl", "zu", "Zl", "Zu")
CONSTRAINT_FIELDS = ("idxb", "lbu", "ubu", "lbx", "ubx", "C", "D", "lg", "ug", "idxs_rev", "lls", "lus", "lbu_mask",
                     "ubu_mask", "lbx_mask", "ubx_mask", "lg_mask", "ug_mask", "lls_mask", "lus_mask", "idxe")
ALL_FIELDS = DYNAMICS_FIELDS + COST_FIELDS + CONSTRAINT_FIELDS
MATRIX_FIELDS = ("A", "B", "Q", "R", "S", "C", "D")
INT_FIELDS = ("idxb", "idxs_rev", "idxe")
MASK_FIELDS = tuple(f for f in CONSTRAINT_FIELDS if f.endswith("_mask"))


@dataclass
class OcpQpDims:
    N: int
    nx: np.ndarray
    nu: np.ndarray
    nbx: np.ndarray
    nbu: np.ndarray
    nb: np.ndarray
    ng: np.ndarray
    ns: np.ndarray
    nbxe: np.ndarray


class OcpQp:
    """OCP-structured QP, stage by stage (same fields and meaning as the reference's ``AcadosOcpQp``)."""

    def __init__(self, N: int):
        self.N = N
        self._f: Dict[str, list] = {f: [None] * (N + 1) for f in ALL_FIELDS}
        z = np.zeros(N + 1, dtype=int)
        self.dims = OcpQpDims(N, *(z.copy() for _ in range(8)))

    def __getattr__(self, name):
        f = self.__dict__.get("_f")
        if f is not None and name in f:
            return f[name]
        raise AttributeError(name)

    def set(self, field_name: str, stage: int, value):
        if stage < 0 or stage > self.N:
            raise ValueError(f"Stage {stage} is out of bounds for N={self.N}.")
        if field_name in DYNAMICS_FIELDS and stage == self.N:
            raise ValueError(f"Dynamics fields cannot be set at terminal stage N={self.N}.")
        if field_name not in ALL_FIELDS:
            raise ValueError(f"Field name {field_name} is not recognized.")
        a = np.asarray(value, dtype=int if field_name in INT_FIELDS else float)
        if field_name in MATRIX_FIELDS:
            if a.ndim != 2:
                a = a.reshape(0, 0) if a.size == 0 else np.atleast_2d(a)
        else:
            a = a.reshape(-1)
        self._f[field_name][stage] = a

    def make_consistent(self, assert_dims: bool = True):
        """Fills unset fields with empty arrays (masks with ones, idxs_rev with -1), derives the dimensions and checks
        them (reference: acados_ocp_qp.py:294-379)."""
        N, d = self.N, self.dims
        nx_next = None
        for k in range(N + 1):
            for f in ALL_FIELDS:
                if f in DYNAMICS_FIELDS and k == N:
                    continue
                if self._f[f][k] is None:
                    self.set(f, k, np.zeros((0, 0)) if f in MATRIX_FIELDS else np.zeros(0))
            nx, nu = self.Q[k].shape[0], self.R[k].shape[0]
            d.nx[k], d.nu[k] = nx, nu
            d.nbx[k], d.nbu[k] = len(self.lbx[k]), len(self.lbu[k])
            d.nb[k] = d.nbx[k] + d.nbu[k]
            d.ng[k], d.ns[k] = len(self.lg[k]), len(self.lls[k])
            d.nbxe[k] = len(self.idxe[k])
            for f, n in (("lbu_mask", d.nbu[k]), ("ubu_mask", d.nbu[k]), ("lbx_mask", d.nbx[k]), ("ubx_mask", d.nbx[k]),
                         ("lg_mask", d.ng[k]), ("ug_mask", d.ng[k]), ("lls_mask", d.ns[k]), ("lus_mask", d.ns[k])):
                if len(self._f[f][k]) == 0 and n > 0:
                    self._f[f][k] = np.ones(n)
            if len(self.idxs_rev[k]) == 0 and d.nb[k] + d.ng[k] > 0:
                self._f["idxs_rev"][k] = -np.ones(d.nb[k] + d.ng[k], dtype=int)
            if self.S[k].size == 0 and nu > 0:
                self._f["S"][k] = np.zeros((nu, nx))
            if self.C[k].size == 0 and d.ng[k] == 0:
                self._f["C"][k] = np.zeros((0, nx))
            if self.D[k].size == 0:
                self._f["D"][k] = np.zeros((d.ng[k], nu))
            if not assert_dims:
                continue
            assert self.q[k].shape == (nx,) and self.r[k].shape == (nu,), f"Inconsistent dimensions in q / r at stage {k}."
            assert self.S[k].shape == (nu, nx) or nu == 0, f"Inconsistent dimensions in S matrix at stage {k}."
            if k < N:
                if nx_next is not None:
                    assert nx == nx_next, f"Inconsistent dimensions between consecutive A matrices at stage {k}."
                nx_next = self.A[k].shape[0]
                assert self.A[k].shape == (nx_next, nx) and self.B[k].shape == (nx_next, nu) and self.b[k].shape == (nx_next,), \
                    f"Inconsistent dynamics dimensions at stage {k}."
            elif nx_next is not None:
                assert nx == nx_next, "Inconsistent terminal state dimension."
            assert len(self.idxb[k]) == d.nb[k], f"Inconsistent number of bound constraint indices at stage {k}."
            assert len(self.ubu[k]) == d.nbu[k] and len(self.ubx[k]) == d.nbx[k] and len(self.ug[k]) == d.ng[k]
            assert self.C[k].shape == (d.ng[k], nx) and self.D[k].shape == (d.ng[k], nu), f"Inconsistent general constraints at stage {k}."
            assert len(self.idxs_rev[k]) == d.nb[k] + d.ng[k], f"Inconsistent number of slack variable indices at stage {k}."
            for f in ("zl", "zu", "Zl", "Zu", "lus", "lls_mask", "lus_mask"):
                assert self._f[f][k].shape == (d.ns[k],), f"Inconsistent dimensions in {f} at stage {k}."
            for i in self.idxe[k]:
                if i < d.nbu[k] or i >= d.nb[k]:
                    raise ValueError(f"Equality constraint index {i} at stage {k} does not correspond to x bound, this is not supported yet.")

    def has_slacks(self) -> bool:
        return bool(np.any(self.dims.ns > 0))

    def has_masks(self) -> bool:
        return any(np.any(m == 0.0) for f in MASK_FIELDS for m in self._f[f] if m is not None)

    # ---- (de)serialisation: the reference's key scheme '<field>_<zero-padded stage>' ----------------------------
    @classmethod
    def from_dict(cls, qp_dict) -> "OcpQp":
        N = len([k for k in qp_dict if k.startswith("Q_")]) - 1
        w = len(str(N + 1))
        bad = [k for k in qp_dict if (s := k.split("_")[-1]).isdigit() and len(s) != w]
        if bad:
            raise ValueError(f"Keys {bad} do not follow the expected format with zero-padded stage indices.")
        qp = cls(N)
        for f in ALL_FIELDS:
            for k in range(N + (0 if f in DYNAMICS_FIELDS else 1)):
                key = f"{f}_{k:0{w}d}"
                if key in qp_dict:
                    qp.set(f, k, qp_dict[key])
        qp.make_consistent()
        return qp

    @classmethod
    def from_json(cls, json_file_path: Optional[str] = None, json_data: Optional[dict] = None) -> "OcpQp":
        if json_data is None:
            if json_file_path is None:
                raise ValueError("Either json_file_path or json_data must be provided to from_json.")
            with open(json_file_path, "r") as f:
                json_data = json.load(f)
        return cls.from_dict(json_data)

    def to_dict(self) -> dict:
        w = len(str(self.N + 1))
        out = {}
        for f in ALL_FIELDS:
            for k in range(self.N + (0 if f in DYNAMICS_FIELDS else 1)):
                v = self._f[f][k]
                if v is not None:
                    out[f"{f}_{k:0{w}d}"] = v.tolist()
        return out

    def get_hessian_block(self, stage: int) -> np.ndarray:
        """[R S; S' Q] of one stage, slack Hessians appended (reference: acados_ocp_qp.py:437-452)."""
        nu, nx = self.dims.nu[stage], self.dims.nx[stage]
        H = np.zeros((nu + nx, nu + nx))
        H[:nu, :nu], H[nu:, nu:] = self.R[stage], self.Q[stage]
        if nu > 0:
            H[:nu, nu:], H[nu:, :nu] = self.S[stage], self.S[stage].T
        if self.dims.ns[stage] > 0:
            Z = np.diag(np.concatenate([self.Zl[stage], self.Zu[stage]]))
            H = np.block([[H, np.zeros((nu + nx, Z.shape[0]))], [np.zeros((Z.shape[0], nu + nx)), Z]])
        return H


@dataclass
class OcpQpOptions:
    """The reference's ``AcadosOcpQpOptions`` fields that reach this path (acados_ocp_qp_options.py)."""
    qp_solver: str = "PARTIAL_CONDENSING_CUIPM"
    hpipm_mode: str = "BALANCE"
    iter_max: int = 50
    tol_stat: float = 1e-6
    tol_eq: float = 1e-8
    tol_ineq: float = 1e-8
    tol_comp: float = 1e-8
    warm_start: int = 0
    mu0: float = 1.0
    t0_init: int = 2
    cond_N: Optional[int] = None
    print_level: int = 0

    def make_consistent(self, N: int):
        if self.qp_solver in ("FULL_CONDENSING_CUIPM", "FULL_CONDENSING_HPIPM"):
            # full condensing = one block: every state but the terminal one is eliminated (cond_N = 1; the reference's
            # ocp_qp_full_condensing.c:450-645 -> d_cond_qp_cond also drops x_N and hands a dense_qp to dense_qp_hpipm; here the
            # 2-stage QP [all inputs | x_N] goes through the same OCP interior-point kernel, so the QP and its solution are the
            # same, the iterates -- and hence iteration counts -- are not those of the dense solver)
            self.cond_N = 1
        elif self.qp_solver not in ("PARTIAL_CONDENSING_CUIPM", "PARTIAL_CONDENSING_HPIPM"):
            raise ValueError(f"qp_solver {self.qp_solver} is not served by this backend (PARTIAL_CONDENSING_CUIPM, FULL_CONDENSING_CUIPM; "
                             "the *_HPIPM names are accepted as aliases so that existing scripts switch over).")
        if self.cond_N is not None and not 1 <= self.cond_N <= N:
            raise ValueError(f"cond_N must be in 1..N={N}")
        if self.hpipm_mode != "BALANCE":
            raise ValueError("hpipm_mode: only BALANCE (the acados default) selects code paths that exist here")

    def to_cuipm(self) -> CuipmOpts:
        return default_opts(self.hpipm_mode, iter_max=self.iter_max, stat_max=max(self.iter_max, 50), res_g_max=self.tol_stat,
                            res_b_max=self.tol_eq, res_d_max=self.tol_ineq, res_m_max=self.tol_comp,
                            warm_start=self.warm_start, mu0=self.mu0, t0_init=self.t0_init)


# -----------------------------------------------------------------------------------------------------------------
# packing: structurally identical QPs -> one batch of cuipm records (with the stage-0 equality elimination)
# -----------------------------------------------------------------------------------------------------------------

class PackedBatch:
    """Records of a batch plus what is needed to restore the eliminated stage-0 states afterwards."""

    def __init__(self, qps: Sequence[OcpQp], eliminate: bool = True):
        """eliminate=False keeps stage 0 as posed (records of the FULL shape, x0 still a pair of coinciding bounds): the
        input format of the device-side elimination (binding.CuipmReducer)."""
        q0 = qps[0]
        for q in qps:
            q.make_consistent()
        self.qps, self.N, self.nbatch = list(qps), q0.N, len(qps)
        N, d = q0.N, q0.dims
        for q in qps[1:]:
            same = q.N == N and all(np.array_equal(getattr(q.dims, f), getattr(d, f)) for f in ("nx", "nu", "nbx", "nbu", "ng", "ns", "nbxe"))
            same = same and all(np.array_equal(q.idxb[k], q0.idxb[k]) and np.array_equal(q.idxs_rev[k], q0.idxs_rev[k])
                                and np.array_equal(q.idxe[k], q0.idxe[k]) for k in range(N + 1))
            if not same:
                raise ValueError("all QPs of a batch must share dimensions and index maps (idxb, idxs_rev, idxe)")
        if any(d.nbxe[k] > 0 for k in range(1, N + 1)):
            raise ValueError("idxe at stages > 0 is not supported (the reference eliminates stage-0 states only)")
        # stage 0: eliminated state components E (through their bounds), kept ones F
        nu0, nx0 = int(d.nu[0]), int(d.nx[0])
        eb = np.asarray(q0.idxe[0], dtype=int) if eliminate else np.zeros(0, dtype=int)   # positions in the bound list
        self.elim_b = eb
        self.E = np.asarray(q0.idxb[0], dtype=int)[eb] - nu0 if len(eb) else np.zeros(0, dtype=int)   # state indices
        self.F = np.setdiff1d(np.arange(nx0), self.E)
        keep_b = np.setdiff1d(np.arange(int(d.nb[0])), eb)
        self.keep_b = keep_b
        if len(eb) and np.any(np.asarray(q0.idxs_rev[0])[eb] >= 0):
            raise ValueError("a softened bound cannot be marked as an equality")
        # reduced shape
        remap0 = -np.ones(nu0 + nx0, dtype=int)
        remap0[:nu0] = np.arange(nu0)
        remap0[nu0 + self.F] = nu0 + np.arange(len(self.F))
        nx = [len(self.F)] + [int(v) for v in d.nx[1:]]
        nu = [int(v) for v in d.nu]
        idxb = [[int(remap0[i]) for i in np.asarray(q0.idxb[0], dtype=int)[keep_b]]] + [[int(i) for i in q0.idxb[k]] for k in range(1, N + 1)]
        nb = [len(i) for i in idxb]
        ng = [int(v) for v in d.ng]
        ns = [int(v) for v in d.ns]
        rev0 = np.asarray(q0.idxs_rev[0], dtype=int)
        rev = [[int(i) for i in np.concatenate([rev0[keep_b], rev0[int(d.nb[0]):]])]] + [[int(i) for i in q0.idxs_rev[k]] for k in range(1, N + 1)]
        self.shape = Shape(N, nx, nu, nb, ng, ns, idxb, rev)
        self.layout = Layout(self.shape)
        self.qp = self.layout.new_qp(self.nbatch)
        self.x0E = np.zeros((self.nbatch, len(self.E)))
        self._fill()

    def _stack(self, f, k):
        return np.stack([q._f[f][k] for q in self.qps])

    def _fill(self):
        L, N, sh = self.layout, self.N, self.shape
        d = self.qps[0].dims
        E, F, kb = self.E, self.F, self.keep_b
        for k in range(N + 1):
            nu, nxf = int(d.nu[k]), int(d.nx[k])
            R, S, Q = self._stack("R", k), self._stack("S", k), self._stack("Q", k)
            r, q = self._stack("r", k), self._stack("q", k)
            C, D = self._stack("C", k), self._stack("D", k)
            lb = np.concatenate([self._stack("lbu", k), self._stack("lbx", k)], axis=1)
            ub = np.concatenate([self._stack("ubu", k), self._stack("ubx", k)], axis=1)
            lbm = np.concatenate([self._stack("lbu_mask", k), self._stack("lbx_mask", k)], axis=1)
            ubm = np.concatenate([self._stack("ubu_mask", k), self._stack("ubx_mask", k)], axis=1)
            lg, ug = self._stack("lg", k), self._stack("ug", k)
            xsel = np.arange(nxf)
            if k == 0 and len(E):
                xE = lb[:, self.elim_b]                                  # x0 = lbx_0 on the eliminated components
                self.x0E = xE
                r = r + np.einsum("bue,be->bu", S[:, :, E], xE) if nu > 0 else r
                q = (q + np.einsum("bfe,be->bf", Q[:, :, E], xE))[:, F]
                lg = lg - np.einsum("bge,be->bg", C[:, :, E], xE)
                ug = ug - np.einsum("bge,be->bg", C[:, :, E], xE)
                Q, S, C = Q[:, F][:, :, F], S[:, :, F], C[:, :, F]
                lb, ub, lbm, ubm = lb[:, kb], ub[:, kb], lbm[:, kb], ubm[:, kb]
                xsel = F
            nx = len(xsel)
            H = L.view(self.qp, "RSQ", k)
            H[:, :nu, :nu], H[:, nu:, nu:] = R, Q
            if nu > 0 and nx > 0:
                H[:, :nu, nu:] = S
                H[:, nu:, :nu] = np.swapaxes(S, 1, 2)
            L.view(self.qp, "rq", k)[:] = np.concatenate([r, q], axis=1)
            if k < N:
                A, B, b = self._stack("A", k), self._stack("B", k), self._stack("b", k)
                if k == 0 and len(E):
                    b = b + np.einsum("bne,be->bn", A[:, :, E], self.x0E)
                    A = A[:, :, F]
                BA = L.view(self.qp, "BAt", k)              # (nbatch, nx_next, nu+nx): row j = column j of [B'; A']
                BA[:, :, :nu], BA[:, :, nu:] = B, A
                L.view(self.qp, "b", k)[:] = b
            ngk = sh.ng[k]
            if ngk > 0:
                DC = L.view(self.qp, "DCt", k)
                DC[:, :, :nu], DC[:, :, nu:] = D, C
            nsk = sh.ns[k]
            L.view(self.qp, "d", k)[:] = np.concatenate([lb, lg, -ub, -ug, self._stack("lls", k), self._stack("lus", k)], axis=1)
            L.view(self.qp, "dmask", k)[:] = np.concatenate([lbm, self._stack("lg_mask", k), ubm, self._stack("ug_mask", k),
                                                             self._stack("lls_mask", k), self._stack("lus_mask", k)], axis=1)
            if nsk > 0:
                L.view(self.qp, "Z", k)[:] = np.concatenate([self._stack("Zl", k), self._stack("Zu", k)], axis=1)
                L.view(self.qp, "z", k)[:] = np.concatenate([self._stack("zl", k), self._stack("zu", k)], axis=1)

    # ---- solution of the reduced QPs -> per-stage arrays of the original QPs -------------------------------------
    def unpack(self, sol: np.ndarray, lam_min: float = 1e-16, t_min: float = 1e-16) -> Dict[str, List[np.ndarray]]:
        """Returns {'u','x','pi','lam','t','sl','su'}: lists over stages of (nbatch, dim) arrays in the ORIGINAL QP's
        dimensions; lam / t in HPIPM's order (lb, lg, ub, ug, ls, us).  The multipliers of the eliminated stage-0 bounds
        are recovered from stationarity as the reference does (x_ocp_qp_red.c:948-966)."""
        L, N, sh = self.layout, self.N, self.shape
        d = self.qps[0].dims
        out = {f: [] for f in ("u", "x", "pi", "lam", "t", "sl", "su")}
        for k in range(N + 1):
            nu, ns = sh.nu[k], sh.ns[k]
            ux = L.view(sol, "ux", k)
            lam, t = L.view(sol, "lam", k).copy(), L.view(sol, "t", k).copy()
            x = ux[:, nu:nu + sh.nx[k]]
            if k == 0 and len(self.E):
                nx0, nb0, ng0 = int(d.nx[0]), int(d.nb[0]), int(d.ng[0])
                xf = np.zeros((self.nbatch, nx0))
                xf[:, self.F], xf[:, self.E] = x, self.x0E
                x = xf
                nbr = sh.nb[0]
                lam_f = np.full((self.nbatch, 2 * (nb0 + ng0 + ns)), lam_min)
                t_f = np.full((self.nbatch, 2 * (nb0 + ng0 + ns)), t_min)
                for src, dst in ((lam, lam_f), (t, t_f)):
                    dst[:, self.keep_b] = src[:, :nbr]
                    dst[:, nb0:nb0 + ng0] = src[:, nbr:nbr + ng0]
                    dst[:, nb0 + ng0 + self.keep_b] = src[:, nbr + ng0:2 * nbr + ng0]
                    dst[:, 2 * nb0 + ng0:] = src[:, 2 * nbr + ng0:]
                # stationarity of the original stage 0 without the eliminated bounds: its x_E rows are their multipliers
                q0s = self.qps
                u0 = ux[:, :nu]
                v = np.concatenate([u0, x], axis=1)
                g = np.concatenate([self._stack("r", 0), self._stack("q", 0)], axis=1)
                H = np.stack([q.get_hessian_block(0)[:nu + nx0, :nu + nx0] for q in q0s])
                res = g + np.einsum("bij,bj->bi", H, v)
                if N > 0:
                    BAt = np.concatenate([np.swapaxes(self._stack("B", 0), 1, 2), np.swapaxes(self._stack("A", 0), 1, 2)], axis=1)
                    res += np.einsum("bin,bn->bi", BAt, L.view(sol, "pi", 0))
                dl = lam_f[:, nb0 + ng0:2 * (nb0 + ng0)] - lam_f[:, :nb0 + ng0]
                idxb0 = np.asarray(q0s[0].idxb[0], dtype=int)
                np.add.at(res, (slice(None), idxb0), dl[:, :nb0])
                if ng0 > 0:
                    DCt = np.concatenate([np.swapaxes(self._stack("D", 0), 1, 2), np.swapaxes(self._stack("C", 0), 1, 2)], axis=1)
                    res += np.einsum("big,bg->bi", DCt, dl[:, nb0:])
                tmp = res[:, nu + self.E]
                lam_f[:, self.elim_b] = np.where(tmp >= 0, tmp, lam_min)
                lam_f[:, nb0 + ng0 + self.elim_b] = np.where(tmp >= 0, lam_min, -tmp)
                lam, t = lam_f, t_f
            out["u"].append(ux[:, :nu].copy())
            out["x"].append(np.array(x))
            out["sl"].append(ux[:, nu + sh.nx[k]:nu + sh.nx[k] + ns].copy())
            out["su"].append(ux[:, nu + sh.nx[k] + ns:nu + sh.nx[k] + 2 * ns].copy())
            if k < N:
                out["pi"].append(L.view(sol, "pi", k).copy())
            out["lam"].append(lam)
            out["t"].append(t)
        return out


# -----------------------------------------------------------------------------------------------------------------
# solvers
# -----------------------------------------------------------------------------------------------------------------

class OcpQpBatchSolver:
    """Solves a batch of structurally identical QPs in one launch of the CUDA path."""

    def __init__(self, qps: Sequence[OcpQp], opts: Optional[OcpQpOptions] = None, device: int = 0, device_reduce: bool = True):
        """device_reduce: run the whole chain -- stage-0 equality elimination, block condensing for cond_N < N, solve, expansion
        and restore -- on the GPU in one cuipm_xcond object (binding.CuipmXcond): the records travel as posed, the reduced and
        condensed records never exist on the host.  False runs the elimination, the restore and the condensing on the host
        (numpy) and solves with binding.CuipmSolver."""
        self.opts = opts or OcpQpOptions()
        self.opts.make_consistent(qps[0].N)
        self.device, self.device_reduce = device, device_reduce
        self.c_opts = self.opts.to_cuipm()
        self._cond_N = self.opts.cond_N if self.opts.cond_N is not None else qps[0].N
        self._load(qps)
        if device_reduce:
            self._solver = CuipmXcond(self.packed.shape, self._idxe0, self._cond_N, len(qps), device)
        else:
            self._solver = CuipmSolver(self._cond.cshape if self._cond is not None else self.packed.shape, len(qps), device)
        self._sol = None
        self.info = None
        self.stat = None
        self.result = None

    def _load(self, qps):
        self._idxe0 = [int(i) for i in qps[0].idxe[0]]
        self._cond = None
        if self.device_reduce:
            self.packed = PackedBatch(qps, eliminate=False)          # records as posed
        else:
            self.packed = PackedBatch(qps)
            if self._cond_N < self.packed.N:
                # block condensing on the host (acados_b200/condensing.py, numpy)
                from .condensing import BlockCondenser
                self._cond = BlockCondenser(self.packed.shape, self._cond_N)
                self._cqp = self._cond.condense(self.packed.qp)

    @property
    def N(self) -> int:
        return self.packed.N

    def update(self, qps: Sequence[OcpQp]):
        """New data, same structure (an SQP / RL sweep re-solving with updated linearisations).  The device chain and the solver
        hold index maps and buffers of the structure they were built for: a batch of another size, other dimensions, bound /
        slack index maps or stage-0 equalities is refused rather than solved with stale maps."""
        old, old_idxe, old_nb = self.packed.shape, [int(i) for i in self._idxe0], self.packed.nbatch
        self._load(qps)
        new = self.packed.shape
        same = (len(qps) == old_nb and [int(i) for i in qps[0].idxe[0]] == old_idxe and new.N == old.N
                and all(list(getattr(new, f)) == list(getattr(old, f)) for f in ("nx", "nu", "nb", "ng", "ns"))
                and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(new.idxb, old.idxb))
                and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(new.idxs_rev, old.idxs_rev)))
        if not same:
            raise ValueError("OcpQpBatchSolver.update: the new batch does not have the structure (batch size, dimensions, idxb, "
                             "idxs_rev, idxe) this solver was built for; create a new solver")

    def _require_device_condensing(self, name):
        if not (self.device_reduce and self._cond_N < self.N):
            raise RuntimeError(f"{name}: needs the device path with cond_N < N")

    def condense_lhs(self) -> None:
        """Preparation phase of an SQP-RTI step (``ocp_qp_xcond_solver``'s condense_lhs, ocp_qp_xcond_solver.c:591-627): the QPs
        loaded last are reduced and condensed on the device and the condensed records -- with the prediction matrices of every
        stage -- stay there.  Device path with cond_N < N only."""
        self._require_device_condensing("condense_lhs")
        self._solver.condense_lhs(self.packed.qp)

    def condense_rhs_and_solve(self) -> np.ndarray:
        """Feedback phase (``condense_rhs_and_solve``, ocp_qp_xcond_solver.c:629-669): the QPs loaded last (``update``: same
        matrices as at ``condense_lhs``, new vectors) refresh the vectors of the resident condensed records, which are then solved
        and expanded.  Returns the acados status per QP."""
        self._require_device_condensing("condense_rhs_and_solve")
        sol, self.info, self.stat = self._solver.condense_rhs_and_solve(self.packed.qp, self.c_opts, want_stat=True)
        self.result = self.packed.unpack(sol)
        return self._status()

    def solve(self) -> np.ndarray:
        """Returns the acados status per QP (0 success, 2 max iter, 3 min step, 1 NaN; ocp_qp_hpipm.c:398-404).  With
        warm_start >= 2 the solve starts from the previous solve's solution in the solver's (reduced or condensed) layout."""
        if self.device_reduce:
            sol, self.info, self.stat = self._solver.solve(self.packed.qp, self.c_opts, want_stat=True)
            self.result = self.packed.unpack(sol)
            return self._status()
        warm = self._sol if self.c_opts.warm_start >= 2 else None
        qp = self._cqp if self._cond is not None else self.packed.qp
        self._sol, self.info, self.stat = self._solver.solve(qp, self.c_opts, sol0=warm, want_stat=True)
        sol = self._cond.expand(self.packed.qp, self._sol) if self._cond is not None else self._sol
        self.result = self.packed.unpack(sol, self.c_opts.lam_min, self.c_opts.t_min)
        return self._status()

    def _status(self) -> np.ndarray:
        return np.array([{0: 0, 1: 2, 2: 3, 3: 1, 4: 9}.get(int(s), -1) for s in self.info["status"]])

    def get(self, stage: int, field: str) -> np.ndarray:
        if field not in ("x", "u", "pi", "lam", "sl", "su", "t"):
            raise ValueError(f"get(stage={stage}, field={field}): invalid field")
        if stage < 0 or stage > self.N or (field == "pi" and stage == self.N):
            raise ValueError(f"get(stage={stage}, field={field}): stage out of range")
        return self.result[field][stage]

    def get_stats(self, field: str):
        if field == "iter":
            return self.info["iter"].copy()
        if field == "statistics":
            return self.stat
        if field in ("time_qp_solver_call", "time_tot"):
            return self._solver.last_kernel_ms * 1e-3
        raise NotImplementedError(f"get_stats() does not support field '{field}' yet.")

    def close(self):
        self._solver.close()


class OcpQpSolver:
    """Single-QP front end with the reference's method names (``AcadosOcpQpSolver``)."""

    def __init__(self, qp: OcpQp, opts: Optional[OcpQpOptions] = None, verbose: bool = False, device: int = 0,
                 device_reduce: bool = True):
        self.qp = qp
        self._b = OcpQpBatchSolver([qp], opts, device, device_reduce)
        self._status = None

    @property
    def N(self) -> int:
        return self.qp.N

    @property
    def qp_solver_name(self) -> str:
        return self._b.opts.qp_solver

    def solve(self) -> int:
        self._b.update([self.qp])
        self._status = int(self._b.solve()[0])
        return self._status

    def get(self, stage_: int, field_: str, unique_duals: bool = True) -> np.ndarray:
        if field_ not in ("x", "u", "pi", "lam", "sl", "su"):
            raise ValueError(f"OcpQpSolver.get(stage={stage_}, field={field_}): '{field_}' is an invalid argument.")
        if not isinstance(stage_, int):
            raise TypeError(f"OcpQpSolver.get(stage={stage_}, field={field_}): stage index must be an integer.")
        if stage_ == self.N and field_ == "pi":
            raise KeyError(f"OcpQpSolver.get(stage={stage_}, field={field_}): field does not exist at final stage.")
        out = self._b.get(stage_, field_)[0].copy()
        if field_ == "lam" and unique_duals and stage_ == 0:
            d = self.qp.dims
            hard = int(d.ng[0] + d.nb[0])
            u = out[hard:2 * hard] - out[:hard]
            out[:hard], out[hard:2 * hard] = np.maximum(0.0, -u), np.maximum(0.0, u)
        return out

    def get_stats(self, field_: str):
        v = self._b.get_stats(field_)
        if field_ == "iter":
            return int(v[0])
        if field_ == "statistics":
            return v[0, :int(self._b.info["iter"][0]) + 1, :STAT_M].copy()
        return v

    def get_cost(self) -> float:
        return float(self.get_stats("statistics")[-1, 12])

    def get_iterate(self) -> Dict[str, List[np.ndarray]]:
        return {f: [self.get(k, f) for k in range(self.N + (0 if f == "pi" else 1))] for f in ("x", "u", "sl", "su", "pi", "lam")}

    def close(self):
        self._b.close()
