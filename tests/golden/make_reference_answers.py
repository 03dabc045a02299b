"""Stores what the unmodified reference (oracle/_ref, built from the reference sources by oracle/Makefile) returns on the
cases that tests/test_oracle_vs_reference.py compares the oracle with, so that those comparisons run where the reference
is not built:
  reference/tau_min.npz   acados' ``tau_min`` option (test_oracle_matches_reference_with_tau_min): iteration counts,
                          statuses, input trajectories;
  reference/lq_cases.npz  the near-singular instances of the LQ refactorisation (test_oracle_lq_refactorisation):
                          iteration counts, statuses, LQ counts, input trajectories (float64), the whole solution and the
                          per-iteration statistics (float32: they are compared to 1e-6 and 1e-4 relative).
  reference/nonfinite.npz poisoned batches and the masked-infinity family of tests/test_nonfinite_data.py, each QP solved by
                          its own reference object (test_nonfinite_data.reference_answers): iteration counts, statuses, input
                          trajectories (float64), the whole solution (float32, NaN and inf kept) and a SHA-256 of the records
                          solved; per-QP statuses and iteration counts of the reference's xcond path on the QPs as posed.
  python tests/golden/make_reference_answers.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from acados_b200.binding import default_opts  # noqa: E402
from oracle import oracle_binding as ob  # noqa: E402
from test_oracle_vs_reference import CASES, LQ_CASES, TAU_MIN_CASES, TAU_MIN_VALUES  # noqa: E402

assert ob.have_ref(), "build oracle/_ref first: make -C oracle"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference")
os.makedirs(OUT, exist_ok=True)

out = {}
for name in TAU_MIN_CASES:
    b = CASES[name]()
    for tau in TAU_MIN_VALUES:
        sol, info, _ = ob.ref_solve(b, default_opts(m_relax=tau), nthreads=1)
        key = f"{name}_{tau:g}"
        out.update({key + "_qp_head": np.asarray(b.qp[:, :16]), key + "_iter": info["iter"], key + "_status": info["status"],
                    key + "_u": b.layout.u_traj(sol)})
        print(key, "iters", info["iter"].tolist(), "status", info["status"].tolist())
np.savez_compressed(os.path.join(OUT, "tau_min.npz"), **out)

out = {}
for name, make in LQ_CASES.items():
    b = make()
    sol, info, stat, _ = ob.ref_solve(b, default_opts(lq_fact=1), want_stat=True, nthreads=1)
    rows = int(info["iter"].max()) + 1
    out.update({name + "_qp_head": np.asarray(b.qp[:, :16]), name + "_iter": info["iter"], name + "_status": info["status"],
                name + "_lq_count": info["lq_count"], name + "_u": b.layout.u_traj(sol), name + "_sol": sol.astype(np.float32),
                name + "_stat": stat[:, :rows, :14].astype(np.float32)})
    print(name, "iters", info["iter"].tolist(), "lq", info["lq_count"].tolist())
np.savez_compressed(os.path.join(OUT, "lq_cases.npz"), **out)

from test_nonfinite_data import reference_answers  # noqa: E402

out = reference_answers()
for key in sorted(k for k in out if k.endswith("_status")):
    print(key[:-7], "iters", out[key[:-7] + "_iter"].tolist(), "status", out[key].tolist())
np.savez_compressed(os.path.join(OUT, "nonfinite.npz"), **out)
