"""acados_b200 -- H100-native batched OCP-QP interior-point solver (cuipm) behind acados' ocp_qp plugin surface.

Only what the hot path needs lives here: ``csrc/`` (CUDA kernels + the C ABI of include/cuipm.h),
``plugin/`` (the plain-C acados qp_solver plugin that calls the C ABI), ``binding`` (ctypes), ``problems``
(shapes, record layout, synthetic batches), ``ocp_qp`` (host-side mirror of the reference's
AcadosOcpQp / AcadosOcpQpSolver interface for this path), ``condensing`` (batched partial condensing, records to
records) and ``sharding`` (batch slices across ranks).
"""
from .problems import Batch, Layout, Shape  # noqa: F401
