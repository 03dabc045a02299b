// cuipm_condense.cu -- batched partial (block) condensing and expansion on the device: the CUDA instantiation of
// cuipm_condense_core.h (one CTA per QP, a phase = all threads of the CTA + __syncthreads) and its C-ABI entry points.
// Reference: ocp_qp_partial_condensing (acados/ocp_qp/ocp_qp_partial_condensing.c:523-689) -> d_part_cond_qp_cond /
// d_part_cond_qp_expand_sol (external/hpipm/cond/x_part_cond.c:410-866).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>

#include "cuipm.h"
#include "cuipm_condense_plan.h"
#include "cuipm_internal.h"

using namespace cuipm;
using namespace cuipm_cond;

namespace {

struct CtaExec
{
    __device__ int nthreads() const { return (int) blockDim.x; }
    template <class F>
    __device__ void phase(F f)
    {
        f((int) threadIdx.x);
        __syncthreads();
    }
};

// GSCR: the scratch of a block that does not fit in shared memory is QP q's slice of a device buffer (gscr, scr_stride doubles per QP)
template <int MODE, bool GSCR>
__global__ void condense_kernel(Plan P, const double *qp, double *qp2, double *tbuf, double *gscr, size_t scr_stride, int nbatch)
{
    extern __shared__ double sscr[];
    const int q = blockIdx.x;
    if (q >= nbatch) return;
    CtaExec ex;
    double *scr = GSCR ? gscr + (size_t) q * scr_stride : sscr;
    condense_one<MODE>(ex, P, qp + (size_t) q * P.o.qp_stride, qp2 + (size_t) q * P.c.qp_stride, scr,
                       MODE == COND_ALL ? nullptr : tbuf + (size_t) q * P.t_stride);
}

__global__ void expand_kernel(Plan P, const double *qp, const double *sol2, double *sol, int nbatch)
{
    extern __shared__ double scr[];
    const int q = blockIdx.x;
    if (q >= nbatch) return;
    CtaExec ex;
    expand_one(ex, P, qp + (size_t) q * P.o.qp_stride, sol2 + (size_t) q * P.c.sol_stride, sol + (size_t) q * P.o.sol_stride, scr);
}

}  // namespace

struct cuipm_condenser
{
    int device = 0;
    HostPlan hp;
    Plan P{};
    int *d_i = nullptr;
    unsigned *d_u = nullptr;
    size_t smem = 0;              // dynamic shared memory of the condensing kernels (0 with the scratch in global memory)
    size_t smem_exp = 0;          // ... and of the expansion kernel
    double *d_t = nullptr;        // T_j of the QPs of the last lhs pass (t_stride doubles per QP)
    int t_cap = 0, t_valid = 0;   // QPs the buffer holds / QPs the last lhs pass filled
    // condensed blocks whose scratch does not fit in shared memory: the scratch of QP q is d_scr + q * scr_stride (grown on demand, like d_t;
    // calls of one condenser therefore go on one stream, or do not overlap)
    bool gscr = false;
    size_t scr_stride = 0;
    double *d_scr = nullptr;
    int scr_cap = 0;
};

// launches condense_kernel<MODE> with the scratch where the plan needs it
template <int MODE>
static int launch_condense(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, double *tbuf, cudaStream_t stream)
{
    if (!c->gscr)
    {
        const int rc = set_dynamic_smem((const void *) condense_kernel<MODE, false>, c->smem);
        if (rc != CUIPM_OK) return rc;
        condense_kernel<MODE, false><<<nbatch, 128, c->smem, stream>>>(c->P, d_qp, d_qp_cond, tbuf, nullptr, 0, nbatch);
        CK(cudaGetLastError());
        return CUIPM_OK;
    }
    if (c->scr_cap < nbatch)
    {
        CK(cudaStreamSynchronize(stream));
        cudaFree(c->d_scr);
        c->d_scr = nullptr; c->scr_cap = 0;
        CK(cudaMalloc(&c->d_scr, sizeof(double) * c->scr_stride * (size_t) nbatch));
        c->scr_cap = nbatch;
    }
    condense_kernel<MODE, true><<<nbatch, 128, 0, stream>>>(c->P, d_qp, d_qp_cond, tbuf, c->d_scr, c->scr_stride, nbatch);
    CK(cudaGetLastError());
    return CUIPM_OK;
}

extern "C" void cuipm_condenser_destroy(cuipm_condenser *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    cudaFree(c->d_i);
    cudaFree(c->d_u);
    cudaFree(c->d_t);
    cudaFree(c->d_scr);
    delete c;
}

extern "C" cuipm_condenser *cuipm_condenser_create(const cuipm_shape *shape, int cond_N, int device)
{
    if (!shape) { set_error("cuipm_condenser_create: bad arguments"); return nullptr; }
    cuipm_condenser *c = new cuipm_condenser();
    c->device = device;
    if (!build_plan(shape, cond_N, c->hp))
    {
        set_error("cuipm_condenser_create: need 1 <= cond_N <= N (and records within 32-bit offsets)");
        delete c;
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess || cudaMalloc(&c->d_i, sizeof(int) * c->hp.ipool.size()) != cudaSuccess
        || cudaMalloc(&c->d_u, sizeof(unsigned) * c->hp.upool.size()) != cudaSuccess
        || cudaMemcpy(c->d_i, c->hp.ipool.data(), sizeof(int) * c->hp.ipool.size(), cudaMemcpyHostToDevice) != cudaSuccess
        || cudaMemcpy(c->d_u, c->hp.upool.data(), sizeof(unsigned) * c->hp.upool.size(), cudaMemcpyHostToDevice) != cudaSuccess)
    {
        set_error("cuipm_condenser_create: CUDA allocation failed (no CPU fallback)");
        cuipm_condenser_destroy(c);
        return nullptr;
    }
    c->P = c->hp.plan(c->d_i, c->d_u);
    c->smem = sizeof(double) * (size_t) scratch_doubles(c->P);
    c->smem_exp = c->smem;
    // the on-chip scratch must fit every kernel that uses it
    size_t limit = SIZE_MAX;
    for (const void *k : {(const void *) condense_kernel<COND_ALL, false>, (const void *) condense_kernel<COND_LHS, false>,
                          (const void *) condense_kernel<COND_RHS, false>, (const void *) expand_kernel})
    {
        size_t l = 0;
        if (smem_limit(k, &l) != CUIPM_OK) { cuipm_condenser_destroy(c); return nullptr; }
        limit = std::min(limit, l);
    }
    if (c->smem > limit)
    {
        // the scratch goes to a device buffer, one slice per QP; the expansion needs only its first 4 nxmax doubles
        c->gscr = true;
        c->scr_stride = (size_t) ((scratch_doubles(c->P) + 1) & ~1);
        c->smem = 0;
        c->smem_exp = sizeof(double) * (size_t) expand_scratch_doubles(c->P);
    }
    return c;
}

extern "C" const cuipm_shape *cuipm_condenser_condensed_shape(const cuipm_condenser *c) { return c ? &c->hp.cshape : nullptr; }

extern "C" int cuipm_condense_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream)
{
    if (!c || nbatch < 0 || !d_qp || !d_qp_cond) { set_error("cuipm_condense_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(c->device));
    // the masks of a fresh record are 1 and untouched entries of d / Z / z are 0 in the reference's layout: clear, then fill
    CK(cudaMemsetAsync(d_qp_cond, 0, sizeof(double) * c->hp.lc->qp_stride * (size_t) nbatch, (cudaStream_t) stream));
    return launch_condense<COND_ALL>(c, nbatch, d_qp, d_qp_cond, nullptr, (cudaStream_t) stream);
}

// The split of acados' xcond solver (ocp_qp_xcond_solver.c:591-669: condense_lhs in the preparation phase of an SQP-RTI step,
// condense_rhs_and_solve in its feedback phase): the lhs pass condenses the whole QP and keeps the prediction matrices T_j of
// every stage per QP on the device; the rhs pass recomputes the vectors of the condensed records (gradient, dynamics offset,
// shifted bounds, slack gradient) for new b, rq, d, z of the same matrices -- O(nx^2 + nx n2) per stage instead of O(nx^2 n2).
extern "C" int cuipm_condense_lhs_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream)
{
    if (!c || nbatch < 0 || !d_qp || !d_qp_cond) { set_error("cuipm_condense_lhs_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(c->device));
    if (c->t_cap < nbatch)
    {
        CK(cudaStreamSynchronize((cudaStream_t) stream));
        cudaFree(c->d_t);
        c->d_t = nullptr; c->t_cap = 0; c->t_valid = 0;
        CK(cudaMalloc(&c->d_t, sizeof(double) * (size_t) c->P.t_stride * (size_t) nbatch));
        c->t_cap = nbatch;
    }
    CK(cudaMemsetAsync(d_qp_cond, 0, sizeof(double) * c->hp.lc->qp_stride * (size_t) nbatch, (cudaStream_t) stream));
    const int rc = launch_condense<COND_LHS>(c, nbatch, d_qp, d_qp_cond, c->d_t, (cudaStream_t) stream);
    if (rc != CUIPM_OK) return rc;
    c->t_valid = nbatch;
    return CUIPM_OK;
}

extern "C" int cuipm_condense_rhs_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream)
{
    if (!c || nbatch < 0 || !d_qp || !d_qp_cond) { set_error("cuipm_condense_rhs_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch > c->t_valid) { set_error("cuipm_condense_rhs_device: no lhs pass for this many QPs (call cuipm_condense_lhs_device first)"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(c->device));
    return launch_condense<COND_RHS>(c, nbatch, d_qp, d_qp_cond, c->d_t, (cudaStream_t) stream);
}

extern "C" int cuipm_expand_device(cuipm_condenser *c, int nbatch, const double *d_qp, const double *d_sol_cond, double *d_sol, void *stream)
{
    if (!c || nbatch < 0 || !d_qp || !d_sol_cond || !d_sol) { set_error("cuipm_expand_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaMemsetAsync(d_sol, 0, sizeof(double) * c->hp.lo->sol_stride * (size_t) nbatch, (cudaStream_t) stream));
    const int rc = set_dynamic_smem((const void *) expand_kernel, c->smem_exp);
    if (rc != CUIPM_OK) return rc;
    expand_kernel<<<nbatch, 128, c->smem_exp, (cudaStream_t) stream>>>(c->P, d_qp, d_sol_cond, d_sol, nbatch);
    CK(cudaGetLastError());
    return CUIPM_OK;
}
