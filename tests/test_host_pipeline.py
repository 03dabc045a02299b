"""Host-side plumbing around the solver: the plugin's batched entry, whose host threads submit the chunks of a large batch
through cuipm_solve_host_chunk, and the xcond chain, which solves in the device buffers of its own solver."""
import ctypes as C

import numpy as np
import pytest

from acados_b200 import problems
from acados_b200.binding import CuipmSolver, default_opts
from acados_b200.ocp_qp import PackedBatch
from test_ocp_qp_mirror import random_ocp_qp

# cuipm status -> acados status (ocp_qp_cuipm.c: acados_status; acados/utils/types.h)
ACADOS_STATUS = {0: 0, 1: 2, 2: 3, 3: 1, 4: 9}


@pytest.mark.gpu
def test_plugin_batch_entry_chunks_match_the_solver(built):
    """ocp_qp_cuipm_batch_solve at n = 1024: eight chunks, each submitted by whichever host thread unpacked its last QP.
    Solutions, iteration counts and statuses are bit-identical to cuipm_solve_host on the same records and options."""
    from integration import plugin_bench as pb
    if not pb.available():
        pytest.skip("libplugin_bench.so did not travel")
    b = problems.chain_mass(1024, N=20)
    o = default_opts()
    s = CuipmSolver(b.shape, b.nbatch)
    sol, info = s.solve(b.qp, o)
    s.close()
    p = pb.PluginBatch(b, o)
    p.run(2)                                  # the second call reuses the solver and the page-locked staging
    psol, piter, pstatus = p.solutions()
    p.close()
    assert np.array_equal(piter, info["iter"])
    assert np.array_equal(pstatus, [ACADOS_STATUS[int(st)] for st in info["status"]])
    for f in ("ux", "pi", "lam", "t"):
        assert b.layout.gather(psol, f).tobytes() == b.layout.gather(sol, f).tobytes(), f


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True])
def test_xcond_solver_sensitivities_use_the_chains_records(built, adjoint):
    """After cuipm_xcond_solve_host without condensing, cuipm_sens_host on cuipm_xcond_solver(x) differentiates the QPs the chain
    just solved: bit-identical to a plain solver of the reduced shape run on the device reducer's records of the same QPs."""
    import torch
    from acados_b200.binding import CuipmReducer, CuipmXcond
    rng = np.random.default_rng(11)
    qps = [random_ocp_qp(rng, soft=True, general=True) for _ in range(32)]
    full = PackedBatch(qps, eliminate=False)
    idxe0 = [int(i) for i in qps[0].idxe[0]]
    o = default_opts()
    xc = CuipmXcond(full.shape, idxe0, full.N, len(qps))              # cond_N = N: no block condensing
    _, xinfo = xc.solve(full.qp, o)
    r = CuipmReducer(full.shape, idxe0)
    d_full = torch.from_numpy(full.qp).cuda()
    d_red = torch.zeros((len(qps), r.reduced_layout.qp_stride), dtype=torch.float64, device="cuda")
    r.reduce(len(qps), d_full.data_ptr(), d_red.data_ptr())
    torch.cuda.synchronize()
    s = CuipmSolver(r.reduced_shape, len(qps))
    _, info = s.solve(d_red.cpu().numpy(), o)
    r.close()
    assert xinfo.tobytes() == info.tobytes()
    seed = np.random.default_rng(17).standard_normal((len(qps), r.reduced_layout.sol_stride))
    want = s.sens(seed, o, adjoint=adjoint)
    s.close()
    got = np.zeros_like(seed)
    lib = xc.lib
    assert lib.cuipm_sens_host(lib.cuipm_xcond_solver(xc.handle), len(qps), seed.ctypes.data, got.ctypes.data, int(adjoint),
                               C.byref(o)) == 0, lib.cuipm_last_error().decode()
    xc.close()
    assert got.tobytes() == want.tobytes()
