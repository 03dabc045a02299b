// assemble_emul.cpp -- TEST INFRASTRUCTURE ONLY (compiled by tests/test_device_batch.py into a temporary directory).
//
// Runs the product's record-assembly code (acados_b200/csrc/cuipm_assemble_core.h, the body of the CUDA kernel) on the host with
// a sequential execution policy, with the product's table building and source checks, so that the CPU test-suite can hold the
// kernel's index maps to the host packer (ocp_qp.PackedBatch) without a GPU.  The product never calls this.
#include <string>
#include <vector>

#include "cuipm_assemble_core.h"

using namespace cuipm_asm;

namespace {
struct SeqExec
{
    template <class F> void for_each(long long n, F f) { for (long long t = 0; t < n; t++) f(t); }
};
std::string g_err;
}  // namespace

extern "C" {

const char *emul_assemble_error(void) { return g_err.c_str(); }

// nbatch records of `sh` into out (nbatch x qp_stride doubles); CUIPM_OK, or CUIPM_ERR_INVALID with the product's message
int emul_assemble(const cuipm_shape *sh, int nbatch, const cuipm_src *src, int nsrc, double *out)
{
    cuipm_layout *L = cuipm_layout_create(sh);
    std::vector<Stage> st;
    std::vector<Src> srcs;
    if (!stage_table(sh, L, st)) { cuipm_layout_destroy(L); g_err = "offsets beyond 32 bits"; return CUIPM_ERR_TOO_LARGE; }
    g_err = enter_sources(st, src, nsrc, srcs);
    if (!g_err.empty()) { cuipm_layout_destroy(L); return CUIPM_ERR_INVALID; }
    Plan P;
    P.st = st.data();
    P.src = srcs.data();
    P.N = sh->N;
    P.qp_stride = (unsigned) L->qp_stride;
    P.total = (long long) nbatch * (long long) L->qp_stride;
    P.out = out;
    SeqExec ex;
    assemble(ex, P);
    cuipm_layout_destroy(L);
    return CUIPM_OK;
}
}
