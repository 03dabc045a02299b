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

#define RCX(call) do { int rc_ = (call); if (rc_ != CUIPM_OK) return rc_; } while (0)

extern "C" void cuipm_xcond_destroy(cuipm_xcond *x)
{
    if (!x) return;
    cudaSetDevice(x->device);
    if (x->solver) cuipm_destroy(x->solver);
    if (x->cond) cuipm_condenser_destroy(x->cond);
    if (x->red) cuipm_reducer_destroy(x->red);
    asm_free(x);
    cudaFree(x->d_full); cudaFree(x->d_red); cudaFree(x->d_sol_red); cudaFree(x->d_sol_full);
    delete x;
}

extern "C" cuipm_xcond *cuipm_xcond_create(const cuipm_shape *full, int nbxe0, const int *idxe0, int cond_N, int max_batch, int device)
{
    if (!full || max_batch <= 0 || nbxe0 < 0 || (nbxe0 > 0 && !idxe0)) { set_error("cuipm_xcond_create: bad arguments"); return nullptr; }
    cuipm_xcond *x = new cuipm_xcond();
    x->device = device; x->max_batch = max_batch;
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
    if (!x->solver || asm_init(x, full) != CUIPM_OK) return fail();
    const size_t nb = (size_t) max_batch;
    if (cudaSetDevice(device) != cudaSuccess
        || (x->cond && cudaMalloc(&x->d_red, sizeof(double) * x->lr->qp_stride * nb) != cudaSuccess)
        || (x->cond && cudaMalloc(&x->d_sol_red, sizeof(double) * x->lr->sol_stride * nb) != cudaSuccess))
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
// solution of the previous call, from which warm starts (warm_start >= 2) start.  Device pointers; enqueued on the solver's
// stream, nothing waited for.
static int chain_device(cuipm_xcond *x, int mode, int nbatch, const double *d_qp_full, double *d_sol_full, cuipm_info *d_info,
                        double *d_stat, const cuipm_opts *opts)
{
    cuipm_solver *s = x->solver;
    cudaStream_t st = (cudaStream_t) cuipm_stream(s);
    double *d_qp = cuipm_device_qp_buffer(s), *d_sol = cuipm_device_sol_buffer(s);
    RCX(cuipm_reduce_device(x->red, nbatch, d_qp_full, x->cond ? x->d_red : d_qp, st));
    if (x->cond)
    {
        if (mode == 2) RCX(cuipm_condense_rhs_device(x->cond, nbatch, x->d_red, d_qp, st));
        else RCX(cuipm_condense_lhs_device(x->cond, nbatch, x->d_red, d_qp, st));
        if (mode != 2) x->lhs_valid = nbatch;
    }
    if (mode == 1) return CUIPM_OK;
    RCX(cuipm_solve_device(s, nbatch, d_qp, d_sol, d_info, d_stat, opts, 0));
    const double *d_sr = d_sol;
    if (x->cond)
    {
        RCX(cuipm_expand_device(x->cond, nbatch, x->d_red, d_sol, x->d_sol_red, st));
        d_sr = x->d_sol_red;
    }
    return cuipm_restore_device(x->red, nbatch, d_qp_full, d_sr, d_sol_full, opts->lam_min, opts->t_min, st);
}

// the argument checks shared by both kinds of entry; CUIPM_OK, or CUIPM_ERR_INVALID (+ message)
static int chain_check(const cuipm_xcond *x, int mode, int nbatch, const void *qp_full, const void *sol_full, const void *info,
                       const cuipm_opts *opts, const char *name)
{
    if (!x || nbatch < 0 || nbatch > x->max_batch || !qp_full || (mode != 1 && (!sol_full || !info || !opts)))
    {
        set_error(std::string(name) + ": bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    if (mode == 2 && x->cond && x->lhs_valid < nbatch)
    {
        set_error(std::string(name) + ": call the condense_lhs entry first");
        return CUIPM_ERR_INVALID;
    }
    return CUIPM_OK;
}

// host entries: H2D copy, the device chain, D2H copies, synchronise
static int chain_host(cuipm_xcond *x, int mode, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info, double *stat,
                      const cuipm_opts *opts, const char *name)
{
    RCX(chain_check(x, mode, nbatch, qp_full, sol_full, info, opts, name));
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(x->device));
    const size_t nb = (size_t) x->max_batch;
    if ((!x->d_full && cudaMalloc(&x->d_full, sizeof(double) * x->lf->qp_stride * nb) != cudaSuccess)
        || (!x->d_sol_full && cudaMalloc(&x->d_sol_full, sizeof(double) * x->lf->sol_stride * nb) != cudaSuccess))
    {
        set_error(std::string(name) + ": device allocation failed (no CPU fallback)");
        return CUIPM_ERR_CUDA;
    }
    cuipm_solver *s = x->solver;
    cudaStream_t st = (cudaStream_t) cuipm_stream(s);
    cuipm_info *d_info = cuipm_device_info_buffer(s);
    const size_t stat_n = stat ? (size_t) nbatch * CUIPM_STAT_M * (opts->stat_max + 1) : 0;
    double *d_stat = stat ? stat_buffer(s, stat_n) : nullptr;
    if (stat && !d_stat) return CUIPM_ERR_CUDA;
    CK(cudaMemcpyAsync(x->d_full, qp_full, sizeof(double) * x->lf->qp_stride * (size_t) nbatch, cudaMemcpyHostToDevice, st));
    RCX(chain_device(x, mode, nbatch, x->d_full, x->d_sol_full, d_info, d_stat, opts));
    if (mode != 1)
    {
        CK(cudaMemcpyAsync(sol_full, x->d_sol_full, sizeof(double) * x->lf->sol_stride * (size_t) nbatch, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(info, d_info, sizeof(cuipm_info) * (size_t) nbatch, cudaMemcpyDeviceToHost, st));
        if (stat) CK(cudaMemcpyAsync(stat, d_stat, sizeof(double) * stat_n, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    return CUIPM_OK;
}

static int chain_dev(cuipm_xcond *x, int mode, int nbatch, const double *d_qp_full, double *d_sol_full, cuipm_info *d_info,
                     double *d_stat, const cuipm_opts *opts, int sync, const char *name)
{
    RCX(chain_check(x, mode, nbatch, d_qp_full, d_sol_full, d_info, opts, name));
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(x->device));
    RCX(chain_device(x, mode, nbatch, d_qp_full, d_sol_full, d_info, d_stat, opts));
    if (sync) CK(cudaStreamSynchronize((cudaStream_t) cuipm_stream(x->solver)));
    return CUIPM_OK;
}

extern "C" int cuipm_xcond_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info, double *stat,
                                      const cuipm_opts *opts)
{
    return chain_host(x, 0, nbatch, qp_full, sol_full, info, stat, opts, "cuipm_xcond_solve_host");
}
extern "C" int cuipm_xcond_condense_lhs_host(cuipm_xcond *x, int nbatch, const double *qp_full)
{
    return chain_host(x, 1, nbatch, qp_full, nullptr, nullptr, nullptr, nullptr, "cuipm_xcond_condense_lhs_host");
}
extern "C" int cuipm_xcond_condense_rhs_and_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info,
                                                       double *stat, const cuipm_opts *opts)
{
    return chain_host(x, 2, nbatch, qp_full, sol_full, info, stat, opts, "cuipm_xcond_condense_rhs_and_solve_host");
}
extern "C" int cuipm_xcond_solve_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, double *d_sol_full, cuipm_info *d_info,
                                        double *d_stat, const cuipm_opts *opts, int sync)
{
    return chain_dev(x, 0, nbatch, d_qp_full, d_sol_full, d_info, d_stat, opts, sync, "cuipm_xcond_solve_device");
}
extern "C" int cuipm_xcond_condense_lhs_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, int sync)
{
    return chain_dev(x, 1, nbatch, d_qp_full, nullptr, nullptr, nullptr, nullptr, sync, "cuipm_xcond_condense_lhs_device");
}
extern "C" int cuipm_xcond_condense_rhs_and_solve_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, double *d_sol_full,
                                                         cuipm_info *d_info, double *d_stat, const cuipm_opts *opts, int sync)
{
    return chain_dev(x, 2, nbatch, d_qp_full, d_sol_full, d_info, d_stat, opts, sync, "cuipm_xcond_condense_rhs_and_solve_device");
}
