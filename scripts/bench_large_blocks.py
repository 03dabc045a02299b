"""Throughput of condensed QPs whose stage blocks do not fit in shared memory (the generic kernel's global-scratch variant).

For each case -- a benchmark configuration (problems.named_config) condensed to cond_N blocks -- prints one JSON line with the
device-resident QP/s of the condensed solve (CUDA events around `steps` solves on the solver's stream, after `warmup` solves),
the same QPs solved uncondensed for context, the scratch bytes per QP and the card's name and power limit.  Condensing itself
(cuipm_condense_device) runs once, before the timed region, and is timed separately.

    python scripts/bench_large_blocks.py [--steps 5] [--warmup 2] [--case c2:1:1024 ...]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DEFAULT_CASES = ["c2:1:1024", "c4:2:1024", "c5:5:256", "c5:1:32"]


def scratch_bytes(shape) -> tuple:
    """(shared memory the on-chip kernel would need, scratch per QP of the global-scratch variant) in bytes: the stage-block
    buffers sm_M + sm_AL + sm_C of acados_b200/csrc/cuipm_plan.h, and those plus the vector area sm_V."""
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
    return 8 * (M + AL + Cb + V), 8 * (M + AL + Cb)


def device_qps(solver, nb, d_qp, d_sol, d_info, opts, steps, warmup, torch):
    """QP/s of `steps` device-resident solves between two CUDA events on the solver's stream; mean iterations of the last."""
    from acados_b200.binding import INFO_DTYPE
    stream = torch.cuda.ExternalStream(solver.lib.cuipm_stream(solver.handle))
    for _ in range(warmup):
        solver.solve_device(nb, d_qp.data_ptr(), d_sol.data_ptr(), d_info.data_ptr(), opts, sync=False)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        ev0.record()
    for _ in range(steps):
        solver.solve_device(nb, d_qp.data_ptr(), d_sol.data_ptr(), d_info.data_ptr(), opts, sync=False)
    with torch.cuda.stream(stream):
        ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    info = np.frombuffer(d_info.cpu().numpy().tobytes(), dtype=INFO_DTYPE)
    return nb * steps / (ms * 1e-3), ms / steps, info


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        phys = int(vis.split(",")[0]) if vis and vis.split(",")[0].strip().isdigit() else 0
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(phys)) / 1000.0
    except Exception:  # noqa: BLE001
        return None


def run_case(name, cond_N, nb, steps, warmup, torch):
    from acados_b200 import problems as P
    from acados_b200.binding import INFO_DTYPE, CuipmCondenser, CuipmSolver, default_opts
    b = P.named_config(name, nb)
    opts = default_opts()
    d_qp = torch.from_numpy(b.qp).cuda()
    # condensed records, made on the device
    dc = CuipmCondenser(b.shape, cond_N)
    cshape, clay = dc.condensed_shape, dc.condensed_layout
    d_cqp = torch.zeros((nb, clay.qp_stride), dtype=torch.float64, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dc.condense(nb, d_qp.data_ptr(), d_cqp.data_ptr())          # first call allocates the condenser's scratch
    torch.cuda.synchronize()
    e0.record()
    dc.condense(nb, d_qp.data_ptr(), d_cqp.data_ptr())
    e1.record()
    torch.cuda.synchronize()
    condense_ms = e0.elapsed_time(e1)
    dc.close()
    smem_b, scratch_b = scratch_bytes(cshape)
    # the solver's rule (GenericPath::create): the device's opt-in limit less the largest static shared memory of the on-chip
    # generic-kernel instances.  1312 B is that figure as `-Xptxas -v` reports it for cuipm_solve_kernel at W = 2 and 4 on sm_90a
    # (Ctx and g_red in cuipm_kernel.cu); it changes with Ctx, and this field only labels the report
    spill = smem_b > torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1312
    out = {"case": f"{name} cond_N={cond_N}", "nbatch": nb, "cond_shape": {"N": cshape.N, "nmax": max(x + u for x, u in zip(cshape.nx, cshape.nu)),
                                                                          "ngmax": max(cshape.ng)},
           "on_chip_bytes_needed": smem_b, "spill": spill, "scratch_bytes_per_qp": scratch_b if spill else 0,
           "condense_ms": round(condense_ms, 3)}
    s = CuipmSolver(cshape, nb)
    d_sol = torch.zeros((nb, clay.sol_stride), dtype=torch.float64, device="cuda")
    d_info = torch.zeros(nb * INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    qps, ms, info = device_qps(s, nb, d_cqp, d_sol, d_info, opts, steps, warmup, torch)
    s.close()
    out.update({"qps_condensed": round(qps, 1), "ms_per_solve_condensed": round(ms, 3), "iters_mean_condensed": float(info["iter"].mean()),
                "converged_condensed": int((info["status"] == 0).sum())})
    del d_cqp, d_sol
    # the same QPs uncondensed, for context
    s = CuipmSolver(b.shape, nb)
    d_sol = torch.zeros((nb, b.layout.sol_stride), dtype=torch.float64, device="cuda")
    qps, ms, info = device_qps(s, nb, d_qp, d_sol, d_info, opts, steps, warmup, torch)
    s.close()
    out.update({"qps_uncondensed": round(qps, 1), "ms_per_solve_uncondensed": round(ms, 3), "iters_mean_uncondensed": float(info["iter"].mean())})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--case", action="append", help="config:cond_N:nbatch (default: %s)" % " ".join(DEFAULT_CASES))
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    import torch
    from acados_b200.binding import load_library
    load_library()
    dev = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    for c in args.case or DEFAULT_CASES:
        name, cond_N, nb = c.split(":")
        r = run_case(name, int(cond_N), int(nb), args.steps, args.warmup, torch)
        r.update(dev)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
