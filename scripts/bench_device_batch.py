"""QPs posed on the host versus QPs posed as CUDA tensors, on chain-mass-sized QPs.

Workload: nx = 21, nu = 3, N = 40, x0 a stage-0 equality, soft bounds on every state (ns = 21 per stage), at batch 4096; once
without condensing and once with cond_N = 5.  Each step changes x0 and the state reference (the cost gradient q), as an MPC or
RL loop does.  Timings, each the median over the steps:
  (a) OcpQpBatchSolver.update + solve: the batch as numpy OcpQp objects, packed on the host, solved through the xcond chain
  (b) OcpQpTensorBatchSolver: only the x0 and reference tensors are rewritten in place per step; solve, then a synchronise
  (c) the assembly kernel alone (CUDA events over many launches), as bytes written + bytes read per second
(a) and (b) must give the same bits (solutions, iteration counts, statuses).  The card name and power limit are printed with
the numbers.  ``python scripts/bench_device_batch.py [--nbatch 4096] [--steps 3]`` (a step of (a) takes seconds of host time)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NX, NU, N = 21, 3, 40


def template(seed=0):
    from acados_b200.ocp_qp import OcpQp
    rng = np.random.default_rng(seed)
    qp = OcpQp(N)
    A = np.eye(NX) + 0.05 * rng.standard_normal((NX, NX)) / np.sqrt(NX)
    B = rng.standard_normal((NX, NU)) / np.sqrt(NX)
    for k in range(N + 1):
        nu = NU if k < N else 0
        qp.set("Q", k, np.eye(NX)); qp.set("R", k, 0.1 * np.eye(nu)); qp.set("S", k, np.zeros((nu, NX)))
        qp.set("q", k, np.zeros(NX)); qp.set("r", k, np.zeros(nu))
        if k < N:
            qp.set("A", k, A); qp.set("B", k, B[:, :nu]); qp.set("b", k, np.zeros(NX))
        qp.set("idxb", k, list(range(nu + NX)))
        qp.set("lbu", k, -np.ones(nu)); qp.set("ubu", k, np.ones(nu))
        if k == 0:
            qp.set("lbx", 0, np.zeros(NX)); qp.set("ubx", 0, np.zeros(NX)); qp.set("idxe", 0, list(range(nu, nu + NX)))
        else:
            qp.set("lbx", k, -np.ones(NX)); qp.set("ubx", k, np.ones(NX))
            qp.set("idxs_rev", k, [-1] * nu + list(range(NX)))
            for f, v in (("zl", 1e2), ("zu", 1e2), ("Zl", 1e2), ("Zu", 1e2), ("lls", 0.0), ("lus", 0.0)):
                qp.set(f, k, v * np.ones(NX))
    qp.make_consistent()
    return qp


def step_data(rng, nbatch):
    """x0 (nbatch, NX) and the reference gradient q (nbatch, N+1, NX) of one step."""
    return 0.5 * rng.standard_normal((nbatch, NX)), 0.1 * rng.standard_normal((nbatch, N + 1, NX))


def host_qps(tpl, x0, qref):
    """The batch as OcpQp objects: the template's arrays shared, x0 and q per QP."""
    from acados_b200.ocp_qp import OcpQp
    out = []
    for i in range(x0.shape[0]):
        q = OcpQp(N)
        q._f = {f: list(v) for f, v in tpl._f.items()}
        q._f["lbx"][0] = q._f["ubx"][0] = x0[i]
        q._f["q"] = list(qref[i])
        out.append(q)
    return out


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def run(nbatch, cond_N, steps, warmup):
    import torch
    from acados_b200.ocp_qp import OcpQpBatchSolver, OcpQpOptions
    from acados_b200.tensor_batch import OcpQpTensorBatchSolver
    tpl = template()
    rng = np.random.default_rng(1)
    data = [step_data(rng, nbatch) for _ in range(warmup + steps)]
    opts = lambda: OcpQpOptions(cond_N=cond_N)
    # (a) host objects -> OcpQpBatchSolver
    b = OcpQpBatchSolver(host_qps(tpl, *data[0]), opts())
    ta = []
    for i, (x0, qref) in enumerate(data):
        qps = host_qps(tpl, x0, qref)
        t0 = time.perf_counter()
        b.update(qps)
        b.solve()
        ta.append(time.perf_counter() - t0)
        print(f"cond_N={cond_N or N} (a) step {i}: {1e3 * ta[-1]:.1f} ms", flush=True)
    # (b) tensors -> OcpQpTensorBatchSolver
    tb = OcpQpTensorBatchSolver(tpl, nbatch, opts())
    dev = [(torch.from_numpy(x0).cuda(), torch.from_numpy(q).cuda()) for x0, q in data]
    x0_t = torch.zeros((nbatch, NX), dtype=torch.float64, device="cuda")
    q_t = torch.zeros((nbatch, N + 1, NX), dtype=torch.float64, device="cuda")
    tb.set("lbx", 0, x0_t); tb.set("ubx", 0, x0_t); tb.set("q", None, q_t)
    torch.cuda.synchronize()
    tt = []
    for x0, q in dev:
        t0 = time.perf_counter()
        x0_t.copy_(x0); q_t.copy_(q)
        tb.solve()
        torch.cuda.synchronize()
        tt.append(time.perf_counter() - t0)
    # same bits as (a) on the last step
    same = bool(np.array_equal(tb.info["iter"], b.info["iter"]) and np.array_equal(tb.info["status"], b.info["status"]))
    for k in range(N + 1):
        for f in ("x", "u", "lam") + (("pi",) if k < N else ()):
            same &= tb.get(k, f).cpu().numpy().tobytes() == np.ascontiguousarray(b.get(k, f)).tobytes()
    # (c) the assembly alone
    reps = 20
    tb.assemble()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        tb.assemble()
    e1.record()
    torch.cuda.synchronize()
    asm_ms = e0.elapsed_time(e1) / reps
    written = nbatch * tb.layout.qp_stride * 8
    read = 0
    for f, per in tb.fields.dims.items():
        for k, shape in per.items():
            per_qp = int(np.prod(shape)) * 8
            read += per_qp * (nbatch if (f, k) in (("lbx", 0), ("ubx", 0)) or f == "q" else 1)
    b.close(); tb.close()
    med = lambda v: float(np.median(v[warmup:]))
    return {"cond_N": cond_N or N, "nbatch": nbatch, "same_bits": same,
            "a_host_update_solve_ms": 1e3 * med(ta), "b_tensor_solve_ms": 1e3 * med(tt),
            "c_assemble_ms": asm_ms, "c_assemble_GBps": (written + read) / asm_ms * 1e-6,
            "c_bytes_written": written, "c_bytes_read": read}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nbatch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, pl = card()
    res = []
    for c in (None, 5):
        res.append(dict(run(a.nbatch, c, a.steps, a.warmup), gpu=name, power_limit=pl))
        print(json.dumps(res[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not all(r["same_bits"] for r in res):
        sys.exit("the tensor route and the host route disagree")


if __name__ == "__main__":
    main()
