// cuipm_xcond.cu -- the whole QP chain of acados' xcond solver on the device, behind one C-ABI object: records of the shape the
// user poses (x0 as a stage-0 equality) in, solutions of that shape out.
//   stage-0 equality elimination (cuipm_reduce.cu) -> block condensing for cond_N < N (cuipm_condense.cu) -> interior-point
//   solve (cuipm_api.cu) -> expansion -> restore of the eliminated states and their multipliers
// Reference: ocp_qp_xcond_solver (acados/ocp_qp/ocp_qp_xcond_solver.c:523-669: condensing + qp_solver + expansion, with the
// condense_lhs / condense_rhs_and_solve split of the SQP-RTI phases) in front of ocp_qp_partial_condensing
// (acados/ocp_qp/ocp_qp_partial_condensing.c:523-689).  The intermediate records never leave the device.
#include <cuda_runtime.h>

#include <string>

#include "cuipm.h"
#include "cuipm_internal.h"

using namespace cuipm;

struct cuipm_xcond
{
    int device = 0, max_batch = 0, N = 0, cond_N = 0;
    cuipm_reducer *red = nullptr;
    cuipm_condenser *cond = nullptr;
    cuipm_solver *solver = nullptr;                    // its device buffers hold the records, solutions and summaries it solves
    const cuipm_layout *lf = nullptr, *lr = nullptr;
    double *d_full = nullptr, *d_red = nullptr, *d_sol_red = nullptr, *d_sol_full = nullptr;   // d_red, d_sol_red: condensing only
    int lhs_valid = 0;
};

#define RCX(call) do { int rc_ = (call); if (rc_ != CUIPM_OK) return rc_; } while (0)

extern "C" void cuipm_xcond_destroy(cuipm_xcond *x)
{
    if (!x) return;
    cudaSetDevice(x->device);
    if (x->solver) cuipm_destroy(x->solver);
    if (x->cond) cuipm_condenser_destroy(x->cond);
    if (x->red) cuipm_reducer_destroy(x->red);
    cudaFree(x->d_full); cudaFree(x->d_red); cudaFree(x->d_sol_red); cudaFree(x->d_sol_full);
    delete x;
}

extern "C" cuipm_xcond *cuipm_xcond_create(const cuipm_shape *full, int nbxe0, const int *idxe0, int cond_N, int max_batch, int device)
{
    if (!full || max_batch <= 0 || nbxe0 < 0 || (nbxe0 > 0 && !idxe0)) { set_error("cuipm_xcond_create: bad arguments"); return nullptr; }
    cuipm_xcond *x = new cuipm_xcond();
    x->device = device; x->max_batch = max_batch; x->N = full->N;
    x->cond_N = (cond_N <= 0 || cond_N > full->N) ? full->N : cond_N;
    auto fail = [&]() { cuipm_xcond_destroy(x); return (cuipm_xcond *) nullptr; };
    x->red = cuipm_reducer_create(full, nbxe0, idxe0, device);
    if (!x->red) return fail();
    x->lf = cuipm_reducer_full_layout(x->red);
    x->lr = cuipm_reducer_reduced_layout(x->red);
    const cuipm_shape *ssh = cuipm_reducer_reduced_shape(x->red);
    if (x->cond_N < full->N)
    {
        x->cond = cuipm_condenser_create(ssh, x->cond_N, device);
        if (!x->cond) return fail();
        ssh = cuipm_condenser_condensed_shape(x->cond);
    }
    x->solver = cuipm_create(ssh, max_batch, device);   // zeroes its solutions: the first warm start starts from zeros
    if (!x->solver) return fail();
    const size_t nb = (size_t) max_batch;
    if (cudaSetDevice(device) != cudaSuccess
        || cudaMalloc(&x->d_full, sizeof(double) * x->lf->qp_stride * nb) != cudaSuccess
        || (x->cond && cudaMalloc(&x->d_red, sizeof(double) * x->lr->qp_stride * nb) != cudaSuccess)
        || (x->cond && cudaMalloc(&x->d_sol_red, sizeof(double) * x->lr->sol_stride * nb) != cudaSuccess)
        || cudaMalloc(&x->d_sol_full, sizeof(double) * x->lf->sol_stride * nb) != cudaSuccess)
    {
        set_error("cuipm_xcond_create: device allocation failed (no CPU fallback)");
        return fail();
    }
    return x;
}

extern "C" const cuipm_layout *cuipm_xcond_full_layout(const cuipm_xcond *x) { return x ? x->lf : nullptr; }
extern "C" int cuipm_xcond_cond_N(const cuipm_xcond *x) { return x ? x->cond_N : 0; }
extern "C" cuipm_solver *cuipm_xcond_solver(cuipm_xcond *x) { return x ? x->solver : nullptr; }

// mode 0: one pass; 1: preparation phase only (reduce + condense_lhs); 2: feedback phase (reduce + condense_rhs + solve + ...)
// The solver's own buffers hold its records (reduced, or condensed: condense_rhs refreshes those condense_lhs left there) and its
// solution of the previous call, from which warm starts (warm_start >= 2) start.
static int chain(cuipm_xcond *x, int mode, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info, double *stat,
                 const cuipm_opts *opts)
{
    if (!x || nbatch < 0 || nbatch > x->max_batch || !qp_full || (mode != 1 && (!sol_full || !info || !opts)))
    {
        set_error("cuipm_xcond: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    if (mode == 2 && x->cond && x->lhs_valid < nbatch) { set_error("cuipm_xcond_condense_rhs_and_solve_host: call cuipm_xcond_condense_lhs_host first"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(x->device));
    cuipm_solver *s = x->solver;
    cudaStream_t st = (cudaStream_t) cuipm_stream(s);
    double *d_qp = cuipm_device_qp_buffer(s), *d_sol = cuipm_device_sol_buffer(s);
    cuipm_info *d_info = cuipm_device_info_buffer(s);
    const size_t stat_n = stat ? (size_t) nbatch * CUIPM_STAT_M * (opts->stat_max + 1) : 0;
    double *d_stat = stat ? stat_buffer(s, stat_n) : nullptr;
    if (stat && !d_stat) return CUIPM_ERR_CUDA;
    CK(cudaMemcpyAsync(x->d_full, qp_full, sizeof(double) * x->lf->qp_stride * (size_t) nbatch, cudaMemcpyHostToDevice, st));
    RCX(cuipm_reduce_device(x->red, nbatch, x->d_full, x->cond ? x->d_red : d_qp, st));
    if (x->cond)
    {
        if (mode == 2) RCX(cuipm_condense_rhs_device(x->cond, nbatch, x->d_red, d_qp, st));
        else RCX(cuipm_condense_lhs_device(x->cond, nbatch, x->d_red, d_qp, st));
        if (mode != 2) x->lhs_valid = nbatch;
    }
    if (mode == 1) { CK(cudaStreamSynchronize(st)); return CUIPM_OK; }
    RCX(cuipm_solve_device(s, nbatch, d_qp, d_sol, d_info, d_stat, opts, 0));
    const double *d_sr = d_sol;
    if (x->cond)
    {
        RCX(cuipm_expand_device(x->cond, nbatch, x->d_red, d_sol, x->d_sol_red, st));
        d_sr = x->d_sol_red;
    }
    RCX(cuipm_restore_device(x->red, nbatch, x->d_full, d_sr, x->d_sol_full, opts->lam_min, opts->t_min, st));
    CK(cudaMemcpyAsync(sol_full, x->d_sol_full, sizeof(double) * x->lf->sol_stride * (size_t) nbatch, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(info, d_info, sizeof(cuipm_info) * (size_t) nbatch, cudaMemcpyDeviceToHost, st));
    if (stat) CK(cudaMemcpyAsync(stat, d_stat, sizeof(double) * stat_n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return CUIPM_OK;
}

extern "C" int cuipm_xcond_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info, double *stat,
                                      const cuipm_opts *opts)
{
    return chain(x, 0, nbatch, qp_full, sol_full, info, stat, opts);
}
extern "C" int cuipm_xcond_condense_lhs_host(cuipm_xcond *x, int nbatch, const double *qp_full)
{
    return chain(x, 1, nbatch, qp_full, nullptr, nullptr, nullptr, nullptr);
}
extern "C" int cuipm_xcond_condense_rhs_and_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info,
                                                       double *stat, const cuipm_opts *opts)
{
    return chain(x, 2, nbatch, qp_full, sol_full, info, stat, opts);
}
