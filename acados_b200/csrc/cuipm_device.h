// cuipm_device.h -- device-visible problem description shared by the API (host) and the kernels.
#ifndef CUIPM_DEVICE_H_
#define CUIPM_DEVICE_H_

#include <cstddef>

#include "cuipm.h"

namespace cuipm {

struct VOff { unsigned ux, pi, lam, t; };   // offsets (doubles) of a primal-dual point / step
struct ROff { unsigned g, b, d, m; };       // offsets (doubles) of a residual / right-hand side

// One horizon stage: dimensions and the offsets of its arrays inside the QP record (q_*), the solution
// record (sol) and the per-QP work record (everything else).
struct StageDesc
{
    int nx, nu, n, nb, ng, ns, nbg, nc;   // n = nu+nx, nbg = nb+ng, nc = 2*(nb+ng+ns)
    int nx1, nu1, n1;                     // dims of stage k+1 (0 at the last stage)
    int idx_off;                          // ipool[idx_off .. +nb) = idxb, then [.. +nbg) = idxs_rev
    int dup_idxb;                         // idxb has repeated entries: scatter serially
    int pad_;
    unsigned q_BAt, q_RSQ, q_DCt, q_b, q_rq, q_d, q_dmask, q_Z, q_z;
    VOff sol, step, itref;
    ROff res, ires;                       // residual sets 0 and 1; the throughput kernel keeps the affine step (dux, dpi, masked dlam) in ires.g, .b, .d
    unsigned w_rmb, w_L, w_Linv, w_lrow, w_Pb, w_Zsi;
    unsigned q_stage, q_stage_bytes;      // this stage's sub-record inside the QP record (16-byte multiple)
    unsigned w_fac, w_fac_bytes;          // factor part of the work record (L, Linv, lrow, Pb, Zs_inv)
    unsigned w_vec, w_vec_bytes;          // vector part of the work record
    unsigned w_Lxx;                       // work record: copy of the state block Lxx of L (nx x nx, leading dimension nx|1, zero above the
                                          // diagonal) kept by the throughput kernel for its forward sweeps (odd leading dimension: row and
                                          // column accesses both bank-conflict free); sizeof(StageDesc) stays a multiple of 8
};
static_assert(sizeof(StageDesc) % 8 == 0, "StageDesc must be a multiple of 8 bytes");

struct ProbDesc
{
    int N;
    int nmax, nxmax, ngmax, nsmax, nbgmax, ncmax, nvsmax;  // maxima over stages (nvs = n + 2 ns)
    int nct;                                               // total constraint count
    int mid_nx, mid_nu;                                    // (nx, nu) shared by stages 1..N-1 and nx of stage N, or 0,0 if not uniform
    unsigned w_lq;                                         // work record: nmax x (nbgmax + nxmax) scratch of the LQ refactorisation
    unsigned w_bkp;                                        // work record: lam, t of the iterate of the last factorisation, in a record of the solution layout
    int pad_;
    size_t qp_stride, sol_stride, work_stride;
    // shared-memory carve (doubles)
    int sm_M, sm_A, sm_AL, sm_C, sm_V;
    int sm_total;
};

struct LaunchArgs
{
    ProbDesc P;
    const StageDesc *sd;
    const int *ipool;
    const double *qp;
    double *sol;
    double *work;
    cuipm_info *info;
    double *stat;      // may be null
    cuipm_opts o;
    int nbatch;
    // sensitivity launch only: right-hand side and result records (solution layout), forward / adjoint
    const double *seed;
    double *sens;
    int adjoint;
    // second pass behind the throughput kernel: solve only the QPs it handed back (indices redo_list[0 .. *redo_count));
    // both null for a plain launch over the whole batch
    const int *redo_list;
    const int *redo_count;
};

// Arguments of the throughput kernel (cuipm_fast.cu): shapes whose interior stages are uniform need three stage
// descriptors only -- stage 0, stage 1 (stage k = stage 1 shifted by (k-1) strides) and stage N -- which travel as
// kernel parameters (constant bank), so that every array offset is an immediate operand.
struct FastArgs
{
    int N, nbatch, nct;
    int nce, nbe, ns2e, nve;       // even-rounded maxima over the stages: constraints, bounds, 2*slacks, nu+nx+2*ns
    int is;                        // index-pool stride of the interior stages
    int nmaps;                     // index maps kept in shared memory: 3 (stages 0, 1, N: interior stages share theirs) or N+1
    unsigned qs, ss, ws;           // strides (doubles) of an interior stage in the QP / solution / work record
    unsigned w_bkp;                // work record: lam, t of the iterate of the last factorisation (solution layout)
    int vsize;                     // doubles of the per-QP vector pool in shared memory
    int gstride;                   // doubles of shared memory per QP
    size_t qp_stride, sol_stride, work_stride;
    StageDesc s0, s1, sN;
    // kernel-side QP records (written by the repack pass from the caller's records): per stage [BAt with leading dimension
    // ld | RSQ as a full symmetric matrix with leading dimension ld | the vectors b, rq, d, d_mask, Z, z as in the caller's
    // record]; kq = start of the stage (stages 0, 1, N), kqs = stride of the interior stages, kH / kV = offsets of the
    // symmetric Hessian / the vector part inside the stage
    unsigned kq[3], kH[3], kV[3], kqs;
    int ld;
    size_t qpk_stride;
    const double *qpk;
    const int *ipool;
    const double *qp;
    double *sol;
    double *work;
    cuipm_info *info;
    double *stat;                  // may be null
    int *redo_list;                // QPs that need a cold path (LQ refactorisation, iterative refinement, no active constraint):
    int *redo_count;               //   handed to the generic kernel, which solves them from scratch
    int *next_qp;                  // work counter of the persistent warps (zero at launch)
    // iteration-sliced scheduling (cuipm_fast_core.h, rr_first / rr_loop): scalar state of every QP between iterations, the
    // CUIPM_RR_RINGS rings of QPs that go on (one per decade of mu, nbatch slots each, -1 = empty) and their counters
    // {heads, tails, stopped}: CUIPM_RR_CTR ints
    double *rr_state;
    int *rr_ring;
    int *rr_ctr;
    cuipm_opts o;
};

#define CUIPM_RR_RINGS 8
#define CUIPM_RR_CTR 32

// status value the throughput kernel leaves in cuipm_info::status of a QP it hands back (never seen by callers)
#define CUIPM_FAST_REDO 100

// launches the solve kernel with `warps` warps per QP on `stream`; returns cudaError_t as int
int launch_solve(const LaunchArgs &a, int warps, void *stream);
// throughput path: true if a kernel instance exists for interior (nx, nu); fills the shared-memory figures of F
bool fast_available(int nx, int nu, FastArgs &F, int *qp_per_warp);
// caller's QP records -> kernel-side records (F.qpk) for F.nbatch QPs on `stream`; sd = device stage table; returns cudaError_t as int
int launch_repack(const FastArgs &F, const StageDesc *sd, void *stream);
// launches the throughput kernel for F on `stream`; returns cudaError_t as int.  mode 0: a QP stays with its warp; 1 then 2: the two
// launches of the iteration-sliced scheduling (fast_rr_available says whether the instance has them)
int launch_fast(const FastArgs &F, void *stream, int mode);
bool fast_rr_available(int nx, int nu);
// QPs the device holds at once with the throughput kernel of F's shape (0 if unknown)
int fast_resident_qps(const FastArgs &F);
// launches the sensitivity kernel (one substitution with the factorisation the last solve left in the work records)
int launch_sens(const LaunchArgs &a, int warps, void *stream);
// dynamic shared memory (bytes) the kernel needs for P
size_t smem_bytes(const ProbDesc &P);
// largest warps-per-QP value compiled
int max_warps();

}  // namespace cuipm
#endif
