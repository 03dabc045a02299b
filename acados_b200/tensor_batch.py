"""Batches of OCP QPs posed as torch tensors on the GPU.

``OcpQpTensorBatchSolver`` is the device-resident counterpart of ``ocp_qp.OcpQpBatchSolver``: a template ``OcpQp`` fixes the
structure (dimensions, ``idxb``, ``idxs_rev``, ``idxe``) and supplies every field's default value, and ``set`` hands over CUDA
float64 tensors for any data field of any stage -- one value per QP, or one value broadcast to the batch.  ``solve`` assembles
the full-shape QP records on the device from those tensors (``cuipm_xcond_assemble_device``, acados_b200/csrc/cuipm_assemble.cu)
and runs the xcond chain on them (``cuipm_xcond_solve_device``: stage-0 elimination, block condensing for cond_N < N, the
interior-point solve, expansion, restore).  Nothing goes through the host and nothing waits for the GPU: the work is ordered
after torch's current stream and torch's current stream after it, so the outputs can feed later torch work directly.

``set`` keeps a reference to the tensor and every ``solve`` reads its contents at that time: a loop that updates its tensors in
place (a new x0, a new reference) calls ``solve`` again and nothing else.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from .binding import FIELD_IDS, INFO_DTYPE, STAT_M, CuipmSrc, CuipmXcond
from .ocp_qp import DYNAMICS_FIELDS, INT_FIELDS, OcpQp, OcpQpOptions, PackedBatch

# cuipm status -> acados status (as OcpQpBatchSolver._status)
_ACADOS_STATUS = (0, 2, 3, 1, 9)


class TensorFields:
    """Which data fields exist at which stages of a template's structure, and what a tensor for one of them must look like.
    ``resolve`` checks a ``set`` call before anything is launched: wrong input raises ``ValueError`` or ``TypeError``."""

    def __init__(self, template: OcpQp, nbatch: int, device: int = 0):
        template.make_consistent()
        self.N, self.nbatch, self.device = template.N, int(nbatch), torch.device("cuda", device)
        d = template.dims
        for k in range(self.N + 1):
            idxb, nbu = np.asarray(template.idxb[k], dtype=int), int(d.nbu[k])
            if np.any(idxb[:nbu] >= d.nu[k]) or np.any(idxb[nbu:] < d.nu[k]):
                raise ValueError(f"idxb at stage {k}: the input bounds (lbu / ubu) must come first, then the state bounds")
        # field -> {stage: shape} where the field has at least one element (the stages the device assembly accepts it at)
        self.dims = {}
        for f in FIELD_IDS:
            for k in range(self.N + (0 if f in DYNAMICS_FIELDS else 1)):
                a = template._f[f][k]
                if a.size > 0:
                    self.dims.setdefault(f, {})[k] = tuple(a.shape)

    def resolve(self, field: str, stage: Optional[int], value):
        """[(stage, element offset into value, s_batch, s_row, s_col)] for ``set(field, stage, value)``; stage None: every
        stage the field exists at, value (nbatch, n_stages, ...) or (n_stages, ...)."""
        if field in INT_FIELDS:
            raise ValueError(f"set: {field} is an index field; the template fixes the structure")
        if field not in FIELD_IDS:
            raise ValueError(f"set: field {field} is not recognized")
        have = self.dims.get(field, {})
        if stage is None:
            stages = sorted(have)
            if not stages:
                raise ValueError(f"set: field {field} exists at no stage of this structure")
            if len({have[k] for k in stages}) != 1:
                raise ValueError(f"set: field {field} has different dimensions at different stages; set it stage by stage")
            core = (len(stages),) + have[stages[0]]
        else:
            if not isinstance(stage, (int, np.integer)) or stage not in have:
                raise ValueError(f"set: field {field} does not exist at stage {stage} of this structure")
            stages, core = [int(stage)], have[int(stage)]
        if not isinstance(value, torch.Tensor):
            raise TypeError(f"set({field}): expected a torch.Tensor, got {type(value).__name__}")
        if value.dtype != torch.float64:
            raise TypeError(f"set({field}): expected a float64 tensor, got {value.dtype}")
        shape = tuple(value.shape)
        if shape == (self.nbatch,) + core:
            batched = True
        elif shape == core:
            batched = False
        else:
            raise ValueError(f"set({field}, {stage}): shape {shape}; expected {(self.nbatch,) + core} or {core}")
        if value.device != self.device:
            raise ValueError(f"set({field}): the tensor is on {value.device}, the solver on {self.device}")
        st = list(value.stride())
        sb = st.pop(0) if batched else 0
        s_stage = st.pop(0) if stage is None else 0
        sr, sc = (st[0], st[1]) if len(st) == 2 else (st[0], 0)
        return [(k, i * s_stage, sb, sr, sc) for i, k in enumerate(stages)]


class OcpQpTensorBatchSolver:
    """Solves ``nbatch`` QPs of a template's structure whose data are CUDA tensors (see the module docstring)."""

    def __init__(self, template: OcpQp, nbatch: int, opts: Optional[OcpQpOptions] = None, device: int = 0):
        self.fields = TensorFields(template, nbatch, device)
        self.opts = opts or OcpQpOptions()
        self.opts.make_consistent(template.N)
        self.c_opts = self.opts.to_cuipm()
        self.nbatch, self.N = int(nbatch), template.N
        packed = PackedBatch([template], eliminate=False)   # the full shape, as OcpQpBatchSolver derives it
        self.shape, self.layout = packed.shape, packed.layout
        self._cond_N = self.opts.cond_N if self.opts.cond_N is not None else self.N
        self._xc = CuipmXcond(self.shape, [int(i) for i in template.idxe[0]], self._cond_N, self.nbatch, device)
        dev = self.fields.device
        # the template's values, uploaded once: the broadcast default source of every (field, stage)
        keys = [(f, k) for f, per in self.fields.dims.items() for k in per]
        arrs = [np.ascontiguousarray(template._f[f][k], dtype=np.float64) for f, k in keys]
        offs = np.cumsum([0] + [a.size for a in arrs])
        self._tpl = torch.from_numpy(np.concatenate([a.ravel() for a in arrs])).to(dev)
        self._src = (CuipmSrc * len(keys))()
        self._slot = {}
        for i, ((f, k), a, o) in enumerate(zip(keys, arrs, offs)):
            sr, sc = (a.shape[1], 1) if a.ndim == 2 else (1, 0)
            self._src[i] = CuipmSrc(FIELD_IDS[f], k, self._tpl.data_ptr() + 8 * int(o), 0, sr, sc)
            self._slot[(f, k)] = i
        self._set = {}                                       # slot -> (tensor, element offset)
        self.records = torch.empty((self.nbatch, self.layout.qp_stride), dtype=torch.float64, device=dev)
        self._sol = torch.zeros((self.nbatch, self.layout.sol_stride), dtype=torch.float64, device=dev)
        self._info = torch.zeros((self.nbatch, INFO_DTYPE.itemsize), dtype=torch.uint8, device=dev)
        self.stat = torch.zeros((self.nbatch, self.c_opts.stat_max + 1, STAT_M), dtype=torch.float64, device=dev)
        self._stream = torch.cuda.ExternalStream(self._xc.stream, device=dev)
        self._lut = torch.tensor(_ACADOS_STATUS, dtype=torch.int32, device=dev)

    def set(self, field: str, stage: Optional[int], value: torch.Tensor) -> None:
        """Data of ``field`` (AcadosOcpQp's names and orientation) at ``stage`` -- or, with stage None, at every stage it exists
        at -- for every QP: a CUDA float64 tensor (nbatch, *dims), or (*dims) broadcast to the batch.  Any strides are
        accepted.  The tensor is referenced, not copied: each solve reads its contents at that time."""
        for k, off, sb, sr, sc in self.fields.resolve(field, stage, value):
            slot = self._slot[(field, k)]
            self._set[slot] = (value, off)
            s = self._src[slot]
            s.s_batch, s.s_row, s.s_col = sb, sr, sc

    def _enqueue(self, work) -> None:
        cur = torch.cuda.current_stream(self.fields.device)
        self._stream.wait_stream(cur)                       # inputs written by torch before this call
        for slot, (t, off) in self._set.items():
            self._src[slot].ptr = t.data_ptr() + 8 * off
        self._xc.assemble_device(self.nbatch, self._src, len(self._src), self.records.data_ptr())
        work()
        cur.wait_stream(self._stream)                       # outputs safe for later torch work

    def assemble(self) -> torch.Tensor:
        """Only the record assembly: ``records`` (nbatch, qp_stride) from the tensors set and the template's values."""
        self._enqueue(lambda: None)
        return self.records

    def _solve_args(self):
        return (self.nbatch, self.records.data_ptr(), self._sol.data_ptr(), self._info.data_ptr(), self.c_opts,
                self.stat.data_ptr())

    def solve(self) -> torch.Tensor:
        """Assembles and solves; returns the acados status per QP (CUDA int32).  With warm_start >= 2 the solve starts from
        the previous solve's solution in the solver's (reduced or condensed) layout."""
        self._enqueue(lambda: self._xc.solve_device(*self._solve_args()))
        return self._status()

    def _require_condensing(self, name):
        if self._cond_N >= self.N:
            raise RuntimeError(f"{name}: needs cond_N < N")

    def condense_lhs(self) -> None:
        """Preparation phase of an SQP-RTI step: the QPs as set now are reduced and condensed, and the condensed records stay
        on the device (as OcpQpBatchSolver.condense_lhs)."""
        self._require_condensing("condense_lhs")
        self._enqueue(lambda: self._xc.condense_lhs_device(self.nbatch, self.records.data_ptr()))

    def condense_rhs_and_solve(self) -> torch.Tensor:
        """Feedback phase: same matrices as at condense_lhs, new vectors; returns the acados status per QP."""
        self._require_condensing("condense_rhs_and_solve")
        self._enqueue(lambda: self._xc.condense_rhs_and_solve_device(*self._solve_args()))
        return self._status()

    @property
    def info(self) -> np.ndarray:
        """The per-QP summaries of the last solve (copied to the host: synchronises)."""
        return self._info.cpu().numpy().view(INFO_DTYPE).reshape(self.nbatch)

    def _status(self) -> torch.Tensor:
        s = self._info.view(torch.int32)[:, 0]
        ok = (s >= 0) & (s < len(_ACADOS_STATUS))
        return torch.where(ok, self._lut[s.clamp(0, len(_ACADOS_STATUS) - 1).long()], torch.full_like(s, -1))

    def get(self, stage: int, field: str) -> torch.Tensor:
        """(nbatch, dim) view of the full solution records: x, u, sl, su, pi, lam, t (lam / t in HPIPM's order)."""
        if field not in ("x", "u", "pi", "lam", "sl", "su", "t"):
            raise ValueError(f"get(stage={stage}, field={field}): invalid field")
        if stage < 0 or stage > self.N or (field == "pi" and stage == self.N):
            raise ValueError(f"get(stage={stage}, field={field}): stage out of range")
        L, sh = self.layout, self.shape
        nu, nx, ns = sh.nu[stage], sh.nx[stage], sh.ns[stage]
        lo, n = {"u": (L.off["ux"][stage], nu), "x": (L.off["ux"][stage] + nu, nx), "sl": (L.off["ux"][stage] + nu + nx, ns),
                 "su": (L.off["ux"][stage] + nu + nx + ns, ns), "pi": (L.off["pi"][stage], L.size["pi"][stage]),
                 "lam": (L.off["lam"][stage], L.size["lam"][stage]), "t": (L.off["t"][stage], L.size["t"][stage])}[field]
        return self._sol[:, lo:lo + n]

    def get_stats(self, field: str):
        if field == "iter":
            return self._info.view(torch.int32)[:, 1]
        if field == "statistics":
            return self.stat
        raise NotImplementedError(f"get_stats() does not support field '{field}' yet.")

    @property
    def xcond(self) -> CuipmXcond:
        """The cuipm_xcond object (its solver: sensitivities, Riccati getters)."""
        return self._xc

    def close(self):
        self._xc.close()
