// cuipm_device.h -- device-visible problem description shared by the API (host) and the kernels.
#ifndef CUIPM_DEVICE_H_
#define CUIPM_DEVICE_H_

#include <cstddef>
#include <vector>

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
// launches the sensitivity kernel (one substitution with the factorisation the last solve left in the work records)
int launch_sens(const LaunchArgs &a, int warps, void *stream);

struct FastInstance;   // compiled instance of the throughput kernel (cuipm_fast.cu)

// The throughput path of one solver (cuipm_fast.cu): the plan of its shape, the kernel instance that runs it, the buffers the
// kernel needs besides the solver's records, and the choice of schedule.  Streams and events are cudaStream_t / cudaEvent_t
// passed as void *, so that host-only code can include this header.
struct FastPath
{
    const FastInstance *inst = nullptr;   // null: the shape has no throughput kernel
    FastArgs F{};                         // plan of the shape; enqueue adds the records of each batch
    size_t smem = 0;                      // dynamic shared memory per CTA (bytes)
    int sms = 1;                          // SMs of the solver's device
    int ctas[3] = {1, 1, 1};              // CTAs the device holds at once with this shared memory, per launch mode
    int ring_qps = 0;                     // QPs the device holds at once in mode 0 (0: unknown)
    int nslot = 0;                        // chunks that may run concurrently (one set of counters each)
    int use = 1;                          // tuning key "fast": 0 off
    int rr = 1;                           // tuning key "rr": iteration-sliced scheduling 0 off, 1 when the batch exceeds ring_qps, 2 always
    double *qpk = nullptr;                // kernel-side QP records (repack pass)
    int *redo_list = nullptr;             // QPs handed back to the generic kernel
    int *ctr = nullptr;                   // per slot: hand-back count, work counter of the persistent warps
    double *rr_state = nullptr;           // iteration-sliced scheduling: per-QP scalar state, rings, ring counters per slot
    int *rr_ring = nullptr, *rr_ctr = nullptr;

    // Plans the shape of sd / ipool / P and, if a kernel instance runs it, sizes its shared memory, allocates the buffers for
    // max_batch QPs in nslot concurrent chunks and measures the residency on `device` (the current device).  Returns CUIPM_OK
    // (inst stays null for a shape without a throughput kernel) or an error code with the message set.
    int create(const std::vector<StageDesc> &sd, const std::vector<int> &ipool, const ProbDesc &P, int max_batch, int nslot, int device);
    // One batch or chunk `a` (QPs lo .. lo + a.nbatch - 1 of the solver's buffers, counters of `slot`) on `stream`, if the path
    // takes it (shape, options, 16-byte aligned records): repack, then the throughput kernel; ev_repacked / ev_done, if not null,
    // are recorded after the repack and after the last throughput-kernel launch.  Sets a.redo_list / a.redo_count to the QPs
    // handed back and adds to *launches; leaves `a` as it is if the path does not take the batch.  Returns CUIPM_OK or an error.
    int enqueue(LaunchArgs &a, size_t lo, int slot, void *stream, int *launches, void *ev_repacked, void *ev_done);
    // QPs handed back by the last batch or chunks (inst not null, the solver's streams idle); -1 on error
    int handed_back() const;
    void destroy();
};

}  // namespace cuipm
#endif
