// cuipm_kernel.cu -- the batched OCP-QP interior-point kernel (sm_90a).
//
// One CTA of W warps owns one QP for the whole solve: Mehrotra predictor-corrector iterations around a
// square-root Riccati factorisation / substitution, with residuals, step length, centring and the
// termination test evaluated inside the same launch (reference hot path: HPIPM d_ocp_qp_ipm_solve,
// external/hpipm/ocp_qp/x_ocp_qp_ipm.c:2684-3120, reached from acados/ocp_qp/ocp_qp_hpipm.c:347).
// Stage blocks (Hessian block, dynamics block, Cholesky factor) are staged through shared memory with
// coalesced loads of this QP's contiguous record; the batch of QPs is the grid.
//
// This file is the generic path: any per-stage dimensions, box / general / soft constraints, masks.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <string>

#include "cuipm_device.h"
#include "cuipm_internal.h"

namespace cuipm {

namespace {

#define tid ((int) threadIdx.x)

__device__ __forceinline__ int ev(int n) { return (n + 1) & ~1; }


// Per-CTA solver context.  It lives in static shared memory and is reached by name (never through a pointer), and the
// dynamic shared memory is reached through the extern array below, so that every on-chip access compiles to LDS/STS
// with 32-bit addressing instead of generic loads.
//
// Global-scratch variant (Ker<..., SPILL = true>, for shapes whose buffers exceed the shared memory a block may have): the
// stage-block buffers SM_, SAL_, SC_ are this QP's slice of a device scratch buffer (Ctx::spx), the vector area SV_ and the context
// stay on chip.  The sweeps perform the same arithmetic in the same order on the same operands; only the copies into those
// buffers change, from LDGSTS (cp.async needs a shared destination) to plain loads and stores (cpb8 / cpvb).  __syncthreads /
// __syncwarp order global memory among the CTA's threads as they order shared memory.
struct Ctx
{
    ProbDesc P;
    const StageDesc *SD;
    const int *ipool;
    const double *qp;   // this QP's record (read-only for the whole kernel)
    double *sol;        // this QP's solution record
    double *wk;         // this QP's work record
    cuipm_opts o;
    int mask_constr;
    double nc_mask_inv;
    // descriptors of the stages around the one being processed, slot k & 3: the sweeps read their offsets and dimensions
    // from here (LDS with immediate offsets) instead of chasing the global-memory table
    StageDesc ring[4];
#ifdef CUIPM_PROFILE
    long long prof[16];   // cycles per pass kind (thread 0): 0 res, 1 res_lin, 2 fact_backward, 3 forward, 4 solve_backward, 5 vector passes
#endif
    double *spx;          // global-scratch variant: this QP's slice of the scratch buffer (spill_doubles(P) doubles)
};
__shared__ Ctx g_cx;
__shared__ double g_red[8];
extern __shared__ __align__(16) double g_smem[];
#define CX g_cx
// SPILL is the template parameter of Ker (and of the kernels): a compile-time constant, so the on-chip variant's addresses
// are those of the plain extern array
#define SM_ (SPILL ? CX.spx : g_smem)
#define SAL_ (SM_ + CX.P.sm_M + CX.P.sm_A)
#define SC_ (SM_ + CX.P.sm_M + CX.P.sm_A + CX.P.sm_AL)
#define SV_ (SPILL ? g_smem : g_smem + CX.P.sm_M + CX.P.sm_A + CX.P.sm_AL + CX.P.sm_C)
#ifdef CUIPM_PROFILE
#define PROF_T0() long long t0_ = clock64()
#define PROF_ADD(slot) do { if (tid == 0) CX.prof[slot] += clock64() - t0_; t0_ = clock64(); } while (0)
#else
#define PROF_T0() do {} while (0)
#define PROF_ADD(slot) do {} while (0)
#endif

// Stage dimensions seen by the sweep bodies: RDims reads them from the stage descriptor at run time, SDims<..> makes
// them compile-time constants for the interior stages of a uniform horizon, so that every dot product is fully
// unrolled with immediate address offsets (the generic path spends ~5 integer instructions per matrix element on
// 64-bit address arithmetic).
struct RDims
{
    __device__ __forceinline__ int n(const StageDesc &s) const { return s.n; }
    __device__ __forceinline__ int nu(const StageDesc &s) const { return s.nu; }
    __device__ __forceinline__ int nx1(const StageDesc &s) const { return s.nx1; }
    __device__ __forceinline__ int nu1(const StageDesc &s) const { return s.nu1; }
    __device__ __forceinline__ int n1(const StageDesc &s) const { return s.n1; }
};
template <int NX_, int NU_>
struct SDims   // interior stage k (1 <= k <= N-2) of a horizon with uniform (nx, nu): stage k+1 has the same dims
{
    __device__ __forceinline__ constexpr int n(const StageDesc &) const { return NX_ + NU_; }
    __device__ __forceinline__ constexpr int nu(const StageDesc &) const { return NU_; }
    __device__ __forceinline__ constexpr int nx1(const StageDesc &) const { return NX_; }
    __device__ __forceinline__ constexpr int nu1(const StageDesc &) const { return NU_; }
    __device__ __forceinline__ constexpr int n1(const StageDesc &) const { return NX_ + NU_; }
};

template <int W, int SNX, int SNU, bool SPILL>
struct Ker
{
    static constexpr int NT = 32 * W;
    using SMid = SDims<SNX, SNU>;

    // ---- CTA primitives -------------------------------------------------------------------------
    __device__ __forceinline__ void sync()
    {
        if (W == 1) __syncwarp();
        else __syncthreads();
    }
    __device__ __forceinline__ double wsum(double v)
    {
#pragma unroll 2
        for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
        return v;
    }
    __device__ __noinline__ double rsum(double v)
    {
        v = wsum(v);
        if (W > 1)
        {
            if ((tid & 31) == 0) g_red[tid >> 5] = v;
            __syncthreads();
            v = 0.0;
#pragma unroll 2
            for (int w = 0; w < W; w++) v += g_red[w];
            __syncthreads();
        }
        return v;
    }
    __device__ __noinline__ double rmin(double v)
    {
#pragma unroll 2
        for (int m = 16; m > 0; m >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, m));
        if (W > 1)
        {
            if ((tid & 31) == 0) g_red[tid >> 5] = v;
            __syncthreads();
            v = g_red[0];
#pragma unroll 2
            for (int w = 1; w < W; w++) v = fmin(v, g_red[w]);
            __syncthreads();
        }
        return v;
    }
    // max of non-negative values; NaN is propagated (BLASFEO VECNRM_INF semantics, d_aux_lib4.c:4893-4995)
    __device__ __noinline__ double rmax_nan(double v, int isnan_)
    {
#pragma unroll 2
        for (int m = 16; m > 0; m >>= 1)
        {
            v = fmax(v, __shfl_xor_sync(0xffffffffu, v, m));
            isnan_ |= __shfl_xor_sync(0xffffffffu, isnan_, m);
        }
        if (W > 1)
        {
            if ((tid & 31) == 0) g_red[tid >> 5] = isnan_ ? NAN : v;
            __syncthreads();
            v = 0.0;
            isnan_ = 0;
#pragma unroll 2
            for (int w = 0; w < W; w++)
            {
                double x = g_red[w];
                if (x != x) isnan_ = 1;
                else v = fmax(v, x);
            }
            __syncthreads();
        }
        return isnan_ ? NAN : v;
    }
    // ---- addressing -------------------------------------------------------------------------------
    // vector sets: 0 = current iterate (solution record), 1 = step, 2 = iterative-refinement step
    __device__ __forceinline__ double *vux(int set, const StageDesc &s) const
    {
        return set == 0 ? CX.sol + s.sol.ux : CX.wk + (set == 1 ? s.step.ux : s.itref.ux);
    }
    __device__ __forceinline__ double *vpi(int set, const StageDesc &s) const
    {
        return set == 0 ? CX.sol + s.sol.pi : CX.wk + (set == 1 ? s.step.pi : s.itref.pi);
    }
    __device__ __forceinline__ double *vlam(int set, const StageDesc &s) const
    {
        return set == 0 ? CX.sol + s.sol.lam : CX.wk + (set == 1 ? s.step.lam : s.itref.lam);
    }
    __device__ __forceinline__ double *vt(int set, const StageDesc &s) const
    {
        return set == 0 ? CX.sol + s.sol.t : CX.wk + (set == 1 ? s.step.t : s.itref.t);
    }
    // residual sets: 0 = res, 1 = res_itref
    __device__ __forceinline__ double *rg(int set, const StageDesc &s) const { return CX.wk + (set == 0 ? s.res.g : s.ires.g); }
    __device__ __forceinline__ double *rb(int set, const StageDesc &s) const { return CX.wk + (set == 0 ? s.res.b : s.ires.b); }
    __device__ __forceinline__ double *rd(int set, const StageDesc &s) const { return CX.wk + (set == 0 ? s.res.d : s.ires.d); }
    __device__ __forceinline__ double *rm(int set, const StageDesc &s) const { return CX.wk + (set == 0 ? s.res.m : s.ires.m); }

    // ---- global-memory access ---------------------------------------------------------------------
    // QP records are read-only for the whole launch (ld.global.nc); work / solution records are written by this
    // CTA between passes and must be read with coherent loads.
    template <bool RO>
    __device__ __forceinline__ double ldv(const double *p) const
    {
        return RO ? __ldg(p) : __ldca(p);   // ld.global.nc / ld.global.ca: known address space, no generic-address path
    }
    // sum_j G[j*ld] * x[j]: G in global memory (row of a column-major matrix when ld = rows, column when ld = 1),
    // x in shared memory; 4 independent chains, 8 loads in flight
    template <bool RO>
    __device__ __forceinline__ double gdot(const double *G, int ld, const double *x, int len) const
    {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int j = 0;
#pragma unroll 2
        for (; j + 3 < len; j += 4)
        {
            const double a0 = ldv<RO>(G + ld * j), a1 = ldv<RO>(G + ld * (j + 1));
            const double a2 = ldv<RO>(G + ld * (j + 2)), a3 = ldv<RO>(G + ld * (j + 3));
            s0 += a0 * x[j]; s1 += a1 * x[j + 1]; s2 += a2 * x[j + 2]; s3 += a3 * x[j + 3];
        }
        for (; j < len; j++) s0 += ldv<RO>(G + ld * j) * x[j];
        return (s0 + s1) + (s2 + s3);
    }
    // row i of the symmetric n x n matrix H of which the lower triangle is stored (column-major, ld n), times x
    __device__ __forceinline__ double gdot_sym(const double *H, int n, int i, const double *x) const
    {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int j = 0;
#pragma unroll 2
        for (; j + 3 < n; j += 4)
        {
            const double a0 = __ldg(H + (j <= i ? i + n * j : j + n * i));
            const double a1 = __ldg(H + (j + 1 <= i ? i + n * (j + 1) : j + 1 + n * i));
            const double a2 = __ldg(H + (j + 2 <= i ? i + n * (j + 2) : j + 2 + n * i));
            const double a3 = __ldg(H + (j + 3 <= i ? i + n * (j + 3) : j + 3 + n * i));
            s0 += a0 * x[j]; s1 += a1 * x[j + 1]; s2 += a2 * x[j + 2]; s3 += a3 * x[j + 3];
        }
        for (; j < n; j++) s0 += __ldg(H + (j <= i ? i + n * j : j + n * i)) * x[j];
        return (s0 + s1) + (s2 + s3);
    }
    // 8-byte asynchronous global -> shared copy (LDGSTS): no register staging, completion via cp.async.wait_group
    __device__ __forceinline__ void cpa8(double *sdst, const double *gsrc) const
    {
        const unsigned sa = (unsigned) __cvta_generic_to_shared(sdst);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sa), "l"(gsrc));
    }
    // L2 prefetch of a 16-byte-multiple chunk (TMA bulk prefetch), issued by one thread
    __device__ __forceinline__ void prefetch_l2(const double *p, unsigned bytes)
    {
        if (tid == 0 && bytes)
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
    }
    // asynchronous copy of n doubles global -> shared (LDGSTS, no register staging: a register-staged copy loop stalls
    // at its first store until the load returns, one exposed round trip per loop); completion: desc_wait() + barrier
    __device__ __forceinline__ void cpv(double *sdst, const double *gsrc, int n) const
    {
        for (int i = tid; i < n; i += NT) cpa8(sdst + i, gsrc + i);
    }
    // the same two copies into the stage-block buffers (SM_, SAL_, SC_): asynchronous into shared memory, plain load and store
    // into the global scratch of the SPILL variant (RO: the source is a QP record, read-only for the whole launch)
    template <bool RO>
    __device__ __forceinline__ void cpb8(double *dst, const double *gsrc) const
    {
        if (SPILL) *dst = ldv<RO>(gsrc);
        else cpa8(dst, gsrc);
    }
    __device__ __forceinline__ void cpvb(double *dst, const double *gsrc, int n) const
    {
        if (SPILL)
            for (int i = tid; i < n; i += NT) dst[i] = ldv<false>(gsrc + i);
        else cpv(dst, gsrc, n);
    }
    // stage descriptor k -> ring slot k & 3, asynchronously (LDGSTS); desc_wait() + a barrier make it visible
    __device__ __forceinline__ void desc_fetch(int k)
    {
        constexpr int W8 = (int) (sizeof(StageDesc) / 8);
        if (tid < W8) cpa8(reinterpret_cast<double *>(&CX.ring[k & 3]) + tid, reinterpret_cast<const double *>(CX.SD + k) + tid);
    }
    __device__ __forceinline__ void desc_wait() { asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory"); }
    // descriptors for a sweep that starts at stage k0 and moves by dir (+1 / -1): k0 and its successor now, the rest one
    // stage ahead at the top of each stage (desc_next)
    __device__ __forceinline__ void desc_begin(int k0, int dir)
    {
        sync();
        desc_fetch(k0);
        if (k0 + dir >= 0 && k0 + dir <= CX.P.N) desc_fetch(k0 + dir);
        if (k0 - dir >= 0 && k0 - dir <= CX.P.N) desc_fetch(k0 - dir);
        desc_wait();
        sync();
    }
    __device__ __forceinline__ void desc_next(int k, int dir)
    {
        if (k + 2 * dir >= 0 && k + 2 * dir <= CX.P.N) desc_fetch(k + 2 * dir);
    }
    // L1 prefetch of n doubles starting at p (one 128-byte line per thread and round): issued at the top of a stage so
    // that the dependent phases below (each a short global-load -> shared -> barrier chain) hit L1 instead of paying an
    // L2 / HBM round trip each
    __device__ __forceinline__ void pf1(const double *p, int n) const
    {
#ifndef CUIPM_NO_PF1
        for (int i = tid * 16; i < n; i += NT * 16) asm volatile("prefetch.global.L1 [%0];" ::"l"(p + i));
#endif
    }
    // sum_c a[c*sa] * b[c*sb] on shared memory operands, 4 independent chains
    __device__ __forceinline__ double dot(const double *a, int sa, const double *b, int sb, int len)
    {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int c = 0;
        for (; c + 3 < len; c += 4)
        {
            s0 += a[c * sa] * b[c * sb];
            s1 += a[(c + 1) * sa] * b[(c + 1) * sb];
            s2 += a[(c + 2) * sa] * b[(c + 2) * sb];
            s3 += a[(c + 3) * sa] * b[(c + 3) * sb];
        }
        for (; c < len; c++) s0 += a[c * sa] * b[c * sb];
        return (s0 + s1) + (s2 + s3);
    }

    // ---------------------------------------------------------------------------------------------
    // residuals (restates OCP_QP_RES_COMPUTE / _LIN, external/hpipm/ocp_qp/x_ocp_qp_res.c:345-683)
    // lin==0: KKT residuals of the QP at the iterate -> residual set 0; returns mu, obj, gap, ||res_m - tau_min mask||.
    //         update!=0 first moves the iterate by alpha_u along the step (UPDATE_VAR_QP, x_core_qp_ipm_aux.c:472-582,
    //         with the step shortening and the t/lam clipping) -- the two sweeps are fused; and the complementarity
    //         residual is stored twice: res_m_bkp = lam*t and res_m = lam*t - tau_min (the affine right-hand side of the
    //         next iteration, BACKUP_RES_M / COMPUTE_TAU_MIN_QP :672-781).
    // lin==1: residual of the Newton system with rhs set `rhs` at step set `pset`, linearised at the iterate -> set `out`.
    // nrm[4] = inf-norms of (g, b, d, m).  Lane = row for H ux and A pi, lane = column for A' ux.
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void res_pass(int lin, int pset, int rhs, int out, int update, double alpha_u, double &mu, double &obj,
                                          double &gap, double nrm[4], double &res_m_tau)
    {
        const int N = CX.P.N;
        double a_mu = 0.0, a_obj = 0.0, a_gap = 0.0;
        double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
        int f0 = 0, f1 = 0, f2 = 0, f3 = 0, f4 = 0;
        double *ux = SV_, *x1 = ux + ev(CX.P.nvsmax), *pi = x1 + ev(CX.P.nxmax), *pim = pi + ev(CX.P.nxmax);
        double *lam = pim + ev(CX.P.nxmax), *lamr = lam + ev(CX.P.ncmax), *t = lamr + ev(CX.P.ncmax), *msk = t + ev(CX.P.ncmax);
        double *tmp0 = msk + ev(CX.P.ncmax), *tmp1 = tmp0 + ev(CX.P.nbgmax), *g_ = tmp1 + ev(CX.P.nbgmax);
        if (update && alpha_u < 1.0) alpha_u = alpha_u * ((1.0 - alpha_u) * 0.99 + alpha_u * 0.9999999);
        desc_begin(0, 1);
        for (int k = 0; k <= N; k++)
        {
            const StageDesc &s = CX.ring[k & 3];
            desc_next(k, 1);
            auto body = [&](auto dd) {
            const int n = dd.n(s), nu = dd.nu(s), nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc, nx1 = dd.nx1(s);
            const int *idxb = CX.ipool + s.idx_off, *rev = idxb + nb;
            const double *qk = CX.qp;
            pf1(qk + s.q_stage, (int) (s.q_stage_bytes >> 3));
            // ---- vectors of this stage (optionally moved along the step) to shared memory
            {
                double *gu = vux(pset, s);
                const double *du = CX.wk + s.step.ux;
                for (int i = tid; i < n + 2 * ns; i += NT)
                {
                    double v = gu[i];
                    if (update) { v += alpha_u * du[i]; gu[i] = v; }
                    ux[i] = v;
                }
            }
            if (k < N)
            {
                const StageDesc &s1 = CX.ring[(k + 1) & 3];
                const double *gu1 = vux(pset, s1) + s1.nu, *du1 = CX.wk + s1.step.ux + s1.nu, *dp = CX.wk + s.step.pi;
                double *gp = vpi(pset, s);
                for (int j = tid; j < nx1; j += NT)
                {
                    double v = gu1[j], p = gp[j];
                    if (update) { v += alpha_u * du1[j]; p += alpha_u * dp[j]; gp[j] = p; }
                    x1[j] = v;
                    pi[j] = p;
                }
                prefetch_l2(qk + s1.q_stage, s1.q_stage_bytes);
                if (update) prefetch_l2(CX.wk + s1.w_vec, s1.w_vec_bytes);
            }
            {
                double *gl = vlam(pset, s), *gt = vt(pset, s);
                const double *gm = qk + s.q_dmask, *dl = CX.wk + s.step.lam, *dtt = CX.wk + s.step.t;
                for (int i = tid; i < nc; i += NT)
                {
                    double l = gl[i], tt = gt[i];
                    const double mk = CX.mask_constr ? __ldg(gm + i) : 1.0;
                    if (update)
                    {
                        // iterate of the factorisation just used (UPDATE_VAR_QP backups, x_core_qp_ipm_aux.c:534-575): the point the
                        // sensitivities are evaluated at
                        (CX.wk + CX.P.w_bkp + s.sol.lam)[i] = l;
                        (CX.wk + CX.P.w_bkp + s.sol.t)[i] = tt;
                        l += alpha_u * dl[i];
                        tt += alpha_u * dtt[i];
                        if (CX.o.t_lam_min == 2)
                        {
                            l = l <= CX.o.lam_min ? CX.o.lam_min : l;
                            tt = tt <= CX.o.t_min ? CX.o.t_min : tt;
                        }
                        if (CX.mask_constr) l *= mk;
                        gl[i] = l;
                        gt[i] = tt;
                    }
                    lamr[i] = l;
                    lam[i] = CX.mask_constr ? l * mk : l;
                    t[i] = tt;
                    msk[i] = mk;
                }
            }
            sync();
            for (int i = tid; i < nbg; i += NT) tmp0[i] = lam[nbg + i] - lam[i];
            sync();
            // ---- rows of res_g (lane = row), res_b and C'ux (lane = column), matrices straight from global memory
            const double *gvec = rhs < 0 ? qk + s.q_rq : rg(rhs, s);
            const double *bvec = rhs < 0 ? qk + s.q_b : rb(rhs, s);
            const double *Hg = qk + s.q_RSQ, *Ag = qk + s.q_BAt, *Cg = qk + s.q_DCt;
            double *ob = rb(out, s);
            for (int oo = tid; oo < n + nx1 + ng; oo += NT)
            {
                if (oo < n)
                {
                    const int i = oo;
                    const double acc = gdot_sym(Hg, n, i, ux);
                    const double gv = gvec[i];
                    double r;
                    if (!lin)
                    {
                        r = acc + 2.0 * gv;
                        a_obj += 0.5 * r * ux[i];
                        r -= gv;
                        a_gap += r * ux[i];
                    }
                    else
                        r = acc + gv;
                    if (k > 0 && i >= nu) r -= pim[i - nu];
                    r += gdot<true>(Ag + i, n, pi, nx1);
                    for (int g = 0; g < ng; g++) r += __ldg(Cg + i + n * g) * tmp0[nb + g];
                    g_[i] = r;
                }
                else if (oo < n + nx1)
                {
                    const int j = oo - n;
                    const double acc = gdot<true>(Ag + n * j, 1, ux, n);
                    const double bv = bvec[j];
                    const double r = bv - x1[j] + acc;
                    ob[j] = r;
                    const double a = fabs(r);
                    m1 = fmax(m1, a);
                    f1 |= (a != a);
                    if (!lin) a_gap -= bv * pi[j];
                }
                else
                {
                    const int g = oo - n - nx1;
                    tmp1[nb + g] = gdot<true>(Cg + n * g, 1, ux, n);
                }
            }
            sync();
            // ---- box scatter, slack rows
            if (!s.dup_idxb)
                for (int i = tid; i < nb; i += NT)
                {
                    const int ix = idxb[i];
                    tmp1[i] = ux[ix];
                    g_[ix] += tmp0[i];
                }
            else if (tid == 0)
                for (int i = 0; i < nb; i++)
                {
                    const int ix = idxb[i];
                    tmp1[i] = ux[ix];
                    g_[ix] += tmp0[i];
                }
            if (ns > 0)
            {
                const double *Z = qk + s.q_Z, *zvec = rhs < 0 ? qk + s.q_z : rg(rhs, s) + n;
                for (int j = tid; j < 2 * ns; j += NT)
                {
                    const double sj = ux[n + j], zz = zvec[j];
                    double r;
                    if (!lin)
                    {
                        r = Z[j] * sj + 2.0 * zz;
                        a_obj += 0.5 * r * sj;
                        r -= zz;
                        a_gap += r * sj;
                    }
                    else
                        r = Z[j] * sj + zz;
                    r -= lam[2 * nbg + j];
                    const int jj = j < ns ? j : j - ns, offl = j < ns ? 0 : nbg;
                    for (int i = 0; i < nbg; i++)
                        if (rev[i] == jj) r -= lam[offl + i];
                    g_[n + j] = r;
                }
            }
            sync();
            // ---- res_d, res_m
            {
                const double *dvec = rhs < 0 ? qk + s.q_d : rd(rhs, s);
                double *od = rd(out, s), *om = rm(out, s), *obk = CX.wk + s.w_rmb;
                const double *mv = lin ? rm(rhs, s) : nullptr;
                const double *Lam = lin ? CX.sol + s.sol.lam : nullptr, *T = lin ? CX.sol + s.sol.t : nullptr;
                for (int i = tid; i < nc; i += NT)
                {
                    const double dv = dvec[i];
                    double r;
                    if (i < 2 * nbg)
                    {
                        const int up = i >= nbg, ii = up ? i - nbg : i;
                        const double v = tmp1[ii];
                        r = t[i] + dv + (up ? v : -v);
                        if (ns > 0 && rev[ii] >= 0) r -= ux[n + (up ? ns : 0) + rev[ii]];
                    }
                    else
                        r = t[i] - ux[n + (i - 2 * nbg)] + dv;
                    if (CX.mask_constr) r *= msk[i];
                    od[i] = r;
                    double a = fabs(r);
                    m2 = fmax(m2, a);
                    f2 |= (a != a);
                    double mm;
                    if (!lin)
                    {
                        a_gap -= dv * lam[i];
                        mm = lam[i] * t[i] - CX.o.m_relax;        // qp->m = m_relax everywhere (ocp_qp_hpipm.c:338-342, x_ocp_qp_res.c:513-514)
                        if (CX.mask_constr) mm *= msk[i];
                        a_mu += fabs(mm);
                        obk[i] = mm;
                        double ma = mm - CX.o.tau_min;
                        if (CX.mask_constr) ma *= msk[i];
                        om[i] = ma;                                  // affine rhs of the next iteration
                        const double a4 = fabs(mm - CX.o.tau_min * msk[i]);
                        m4 = fmax(m4, a4);
                        f4 |= (a4 != a4);
                    }
                    else
                    {
                        mm = mv[i] + Lam[i] * t[i] + lamr[i] * T[i];
                        if (CX.mask_constr) mm *= msk[i];
                        om[i] = mm;
                    }
                    a = fabs(mm);
                    m3 = fmax(m3, a);
                    f3 |= (a != a);
                }
                double *og = rg(out, s);
                for (int i = tid; i < n + 2 * ns; i += NT)
                {
                    const double r = g_[i];
                    og[i] = r;
                    const double a = fabs(r);
                    m0 = fmax(m0, a);
                    f0 |= (a != a);
                }
            }
            sync();
            for (int j = tid; j < nx1; j += NT) pim[j] = pi[j];      // pi_k is "pi_{k-1}" of the next stage
            sync();
            };
            if (SNX > 0 && k >= 1 && k <= N - 2) body(SMid{});
            else body(RDims{});
            desc_wait();
            sync();
        }
        nrm[0] = rmax_nan(m0, f0);
        nrm[1] = rmax_nan(m1, f1);
        nrm[2] = rmax_nan(m2, f2);
        nrm[3] = rmax_nan(m3, f3);
        if (!lin)
        {
            mu = rsum(a_mu) * CX.nc_mask_inv;
            obj = rsum(a_obj);
            gap = rsum(a_gap);
            res_m_tau = rmax_nan(m4, f4);
        }
    }

    // ---------------------------------------------------------------------------------------------
    // slack elimination (x_ocp_qp_kkt.c:220-335, 431-520): tmp0/tmp1 = effective Gamma / gamma of the
    // softened constraints; ds = slack part of the step rhs; Zi = inverse of the slack Hessian.
    // Parallel over slacks (a slack may soften several constraints).
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void cond_slacks(const StageDesc &s, int fact, const double *Gam, const double *gam, const double *rgs,
                                double *Zi, double *ds, double *tmp0, double *tmp1)
    {
        const int nb = s.nb, ns = s.ns, nbg = s.nbg;
        const int *rev = CX.ipool + s.idx_off + nb;
        const double *Z = CX.qp + s.q_Z;
        for (int j = tid; j < 2 * ns; j += NT)
        {
            const int jj = j < ns ? j : j - ns, offc = j < ns ? 0 : nbg;
            double zi = 0.0, d = rgs[j] + gam[2 * nbg + j];
            if (fact) zi = Z[j] + CX.o.reg_prim + Gam[2 * nbg + j];
            for (int i = 0; i < nbg; i++)
                if (rev[i] == jj)
                {
                    if (fact) zi += Gam[offc + i];
                    d += gam[offc + i];
                }
            if (fact) Zi[j] = 1.0 / zi;
            ds[j] = d;
        }
        sync();
        for (int i = tid; i < nbg; i += NT)
        {
            const int j = rev[i];
            double t0l, t0u, t1l, t1u;
            if (j != -1)
            {
                t0l = Gam[i] - Gam[i] * Zi[j] * Gam[i];
                t0u = Gam[nbg + i] - Gam[nbg + i] * Zi[ns + j] * Gam[nbg + i];
                t1l = gam[i] - Gam[i] * Zi[j] * ds[j];
                t1u = gam[nbg + i] - Gam[nbg + i] * Zi[ns + j] * ds[ns + j];
            }
            else
            {
                t0l = Gam[i]; t0u = Gam[nbg + i]; t1l = gam[i]; t1u = gam[nbg + i];
            }
            if (fact) tmp0[i] = t0l + t0u;
            tmp1[i] = t1l - t1u;
        }
    }

    // ---------------------------------------------------------------------------------------------
    // backward Riccati sweep with factorisation (OCP_QP_FACT_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:880-966)
    // rhs = residual set 0.  Writes L, Linv, lrow, Pb, Zs_inv (and the slack part of the step rhs).
    //
    // Thread r owns row r of the (n+1) x n stage block (row n carries the gradient).  Per stage:
    //   [A; b'] -> SAL_, then in place  AL = [A; b'] * Lxx_{k+1}         (TRMM_RLNN)
    //   column tiles of 4:  acc = H + diag + AL AL' - (already factored columns)   (SYRK + left-looking POTRF)
    //   the 4x4 diagonal block is factorised redundantly by every thread, the panel scaled, columns stored.
    // SM_ holds L_{k+1} (rows 0..n1, row n1 = its gradient row) when the stage starts and L_k when it ends.
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void fact_backward()
    {
        const int N = CX.P.N;
        double *Gam = SV_, *gam = Gam + ev(CX.P.ncmax), *tmp0 = gam + ev(CX.P.ncmax), *tmp1 = tmp0 + ev(CX.P.nbgmax);
        double *dadd = tmp1 + ev(CX.P.nbgmax), *rowv = dadd + ev(CX.P.nmax), *Linv = rowv + ev(CX.P.nmax);
        double *Zi = Linv + ev(CX.P.nmax), *ds = Zi + ev(2 * CX.P.nsmax), *D = ds + ev(2 * CX.P.nsmax);   // D: 4 x 4 diagonal block
        double *sCb = SC_ + ev((CX.P.nmax + 2) * CX.P.ngmax);
        int ldm_prev = 0;
        desc_begin(N, -1);
        for (int k = N; k >= 0; k--)
        {
            const StageDesc &s = CX.ring[k & 3];
            desc_next(k, -1);
            auto body = [&](auto dd) {
            const int n = dd.n(s), nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc, nx1 = dd.nx1(s), nu1 = dd.nu1(s), n1 = dd.n1(s);
            const int *idxb = CX.ipool + s.idx_off;
            const int ldal = ev(n + 1), ldm = ev(n + 1);
            const int kc = k < N ? nx1 : 0;
            pf1(CX.qp + s.q_RSQ, n * n);
            pf1(CX.wk + s.w_vec, (int) (s.w_vec_bytes >> 3) / 3);      // step / residual vectors (first third of the vector part)
            // ---- stage inputs: gradient into rowv, [A; b'] into SAL_ (both asynchronous, two groups), constraint quantities
            cpv(rowv, rg(0, s), n);
            asm volatile("cp.async.commit_group;" ::: "memory");
            if (k < N)
            {
                // [A; b'] into SAL_ with cp.async (LDGSTS): thread r copies row r (coalesced across threads); the copies are
                // all in flight while the constraint quantities below are computed and are waited for just before the TRMM
                const double *Ag = CX.qp + s.q_BAt, *b_ = rb(0, s);
                for (int r = tid; r <= n; r += NT)
                {
                    if (r < n)
                        for (int c = 0; c < nx1; c++) cpb8<true>(SAL_ + r + ldal * c, Ag + r + n * c);
                    else
                        for (int c = 0; c < nx1; c++) cpb8<false>(SAL_ + n + ldal * c, b_ + c);
                }
            }
            if (k > 0)
            {
                const StageDesc &sp = CX.ring[(k - 1) & 3];
                prefetch_l2(CX.qp + sp.q_stage, sp.q_stage_bytes);
                prefetch_l2(CX.wk + sp.w_vec, sp.w_vec_bytes);
            }
            {
                // Gamma, gamma (COMPUTE_GAMMA_GAMMA_QP, x_core_qp_ipm_aux.c:38-86)
                const double *gl = CX.sol + s.sol.lam, *gt = CX.sol + s.sol.t, *grd = rd(0, s), *grm = rm(0, s);
                const double t_min_inv = CX.o.t_min > 0 ? 1.0 / CX.o.t_min : 1e30;
                for (int i = tid; i < nc; i += NT)
                {
                    const double l = gl[i], tt = gt[i], ti = 1.0 / tt;
                    if (CX.o.t_lam_min == 1)
                        Gam[i] = (tt < CX.o.t_min ? t_min_inv : ti) * (l < CX.o.lam_min ? CX.o.lam_min : l);
                    else
                        Gam[i] = ti * l;
                    gam[i] = ti * (grm[i] - l * grd[i]);
                }
                for (int i = tid; i < n; i += NT) dadd[i] = CX.o.reg_prim;
                // the gradient copy (older group) must have landed; the [A; b'] copies may still be in flight
                asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 1;" ::: "memory");
            }
            sync();
            if (ns > 0)
            {
                cond_slacks(s, 1, Gam, gam, rg(0, s) + n, Zi, ds, tmp0, tmp1);
                sync();
                for (int j = tid; j < 2 * ns; j += NT)
                {
                    (CX.wk + s.w_Zsi)[j] = Zi[j];
                    (CX.wk + s.step.ux + n)[j] = ds[j];
                }
            }
            else
            {
                for (int i = tid; i < nbg; i += NT)
                {
                    tmp0[i] = Gam[i] + Gam[nbg + i];
                    tmp1[i] = gam[i] - gam[nbg + i];
                }
                sync();
            }
            if (!s.dup_idxb)
                for (int i = tid; i < nb; i += NT)
                {
                    const int ix = idxb[i];
                    dadd[ix] += tmp0[i];
                    rowv[ix] += tmp1[i];
                }
            else if (tid == 0)
                for (int i = 0; i < nb; i++)
                {
                    const int ix = idxb[i];
                    dadd[ix] += tmp0[i];
                    rowv[ix] += tmp1[i];
                }
            asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
            sync();
            if (k < N)
            {
                // ---- in place: AL = [A; b'] * Lxx   (row r, column tiles of 4; columns only read at c >= tile start)
                const double *Lx = SM_ + nu1 + ldm_prev * nu1;       // Lxx(c, j) = Lx[c + ldm_prev*j], zero above the diagonal
                for (int r = tid; r <= n; r += NT)
                {
                    double *arow = SAL_ + r;
                    for (int jt = 0; jt < nx1; jt += 4)
                    {
                        const int j1 = min(jt + 1, nx1 - 1), j2 = min(jt + 2, nx1 - 1), j3 = min(jt + 3, nx1 - 1);
                        double c0 = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0;
                        for (int c = jt; c < nx1; c++)
                        {
                            const double a = arow[ldal * c];
                            const double *Lc = Lx + c;
                            c0 += a * Lc[ldm_prev * jt];
                            c1 += a * Lc[ldm_prev * j1];
                            c2 += a * Lc[ldm_prev * j2];
                            c3 += a * Lc[ldm_prev * j3];
                        }
                        arow[ldal * jt] = c0;
                        if (jt + 1 < nx1) arow[ldal * (jt + 1)] = c1;
                        if (jt + 2 < nx1) arow[ldal * (jt + 2)] = c2;
                        if (jt + 3 < nx1) arow[ldal * (jt + 3)] = c3;
                    }
                }
                sync();
                // Pb = Lxx * (Lxx' b),  then the gradient row gets l_{k+1}
                {
                    double *Pb = CX.wk + s.w_Pb;
                    for (int i = tid; i < nx1; i += NT) Pb[i] = dot(Lx + i, ldm_prev, SAL_ + n, ldal, i + 1);
                }
                sync();
                for (int j = tid; j < nx1; j += NT) SAL_[n + ldal * j] += SM_[n1 + ldm_prev * (nu1 + j)];
            }
            if (ng > 0)
            {
                // general constraints enter the rank update as extra columns: own-row operand C diag(tmp0) (row n: tmp1),
                // broadcast operand C
                const double *Cg = CX.qp + s.q_DCt;
                for (int e = tid; e < (n + 1) * ng; e += NT)
                {
                    const int g = e / (n + 1), i = e - g * (n + 1);
                    SAL_[i + ldal * (kc + g)] = i < n ? Cg[i + n * g] * tmp0[nb + g] : tmp1[nb + g];
                    if (i < n) sCb[i + ldal * g] = Cg[i + n * g];
                }
            }
            sync();
            // ---- column tiles: SYRK + left-looking Cholesky, rows r >= jt (row n = gradient row)
            const double *Hg = CX.qp + s.q_RSQ;
            for (int jt = 0; jt < n; jt += 4)
            {
                const int w4 = min(4, n - jt);
                for (int r = jt + tid; r <= n; r += NT)
                {
                    // init: H (lower, from global; issued first so the loads overlap the products below)
                    double h0 = 0.0, h1 = 0.0, h2 = 0.0, h3 = 0.0;
                    if (r < n)
                    {
                        h0 = __ldg(Hg + r + n * jt);
                        if (w4 > 1 && r >= jt + 1) h1 = __ldg(Hg + r + n * (jt + 1));
                        if (w4 > 2 && r >= jt + 2) h2 = __ldg(Hg + r + n * (jt + 2));
                        if (w4 > 3 && r >= jt + 3) h3 = __ldg(Hg + r + n * (jt + 3));
                        if (r - jt < 4)
                        {
                            const double dd = dadd[r];
                            if (r == jt) h0 += dd;
                            else if (r == jt + 1) h1 += dd;
                            else if (r == jt + 2) h2 += dd;
                            else h3 += dd;
                        }
                    }
                    else
                    {
                        h0 = rowv[jt];
                        if (w4 > 1) h1 = rowv[jt + 1];
                        if (w4 > 2) h2 = rowv[jt + 2];
                        if (w4 > 3) h3 = rowv[jt + 3];
                    }
                    double c0 = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0;
                    {
                        const double *own = SAL_ + r, *bc = SAL_ + jt;
                        for (int c = 0; c < kc; c++)
                        {
                            const double a = own[ldal * c];
                            const double2 b01 = *reinterpret_cast<const double2 *>(bc + ldal * c);
                            const double2 b23 = *reinterpret_cast<const double2 *>(bc + ldal * c + 2);
                            c0 += a * b01.x; c1 += a * b01.y; c2 += a * b23.x; c3 += a * b23.y;
                        }
                        const double *bcg = sCb + jt;
                        for (int g = 0; g < ng; g++)
                        {
                            const double a = own[ldal * (kc + g)];
                            c0 += a * bcg[ldal * g]; c1 += a * bcg[ldal * g + 1]; c2 += a * bcg[ldal * g + 2]; c3 += a * bcg[ldal * g + 3];
                        }
                    }
                    {
                        const double *own = SM_ + r, *bc = SM_ + jt;
                        double e0 = 0.0, e1 = 0.0, e2 = 0.0, e3 = 0.0;
                        for (int c = 0; c < jt; c++)
                        {
                            const double a = own[ldm * c];
                            const double2 b01 = *reinterpret_cast<const double2 *>(bc + ldm * c);
                            const double2 b23 = *reinterpret_cast<const double2 *>(bc + ldm * c + 2);
                            e0 += a * b01.x; e1 += a * b01.y; e2 += a * b23.x; e3 += a * b23.y;
                        }
                        c0 -= e0; c1 -= e1; c2 -= e2; c3 -= e3;
                    }
                    c0 += h0; c1 += h1; c2 += h2; c3 += h3;
                    // park the raw panel row (rows of the diagonal block are read back by everybody)
                    double *mr = SM_ + r + ldm * jt;
                    mr[0] = c0;
                    if (w4 > 1) mr[ldm] = c1;
                    if (w4 > 2) mr[2 * ldm] = c2;
                    if (w4 > 3) mr[3 * ldm] = c3;
                }
                sync();
                // ---- 4x4 diagonal block (pivot rule blasfeo_ref/x_lapack_ref.c:84-91), redundantly per thread
                {
                    const double *dg = SM_ + jt + ldm * jt;
                    double d00 = dg[0], d10 = 0, d20 = 0, d30 = 0, d11 = 0, d21 = 0, d31 = 0, d22 = 0, d32 = 0, d33 = 0;
                    if (w4 > 1) { d10 = dg[1]; d11 = dg[1 + ldm]; }
                    if (w4 > 2) { d20 = dg[2]; d21 = dg[2 + ldm]; d22 = dg[2 + 2 * ldm]; }
                    if (w4 > 3) { d30 = dg[3]; d31 = dg[3 + ldm]; d32 = dg[3 + 2 * ldm]; d33 = dg[3 + 3 * ldm]; }
                    const double i0 = d00 > 0.0 ? rsqrt(d00) : 0.0;
                    const double l10 = d10 * i0, l20 = d20 * i0, l30 = d30 * i0;
                    d11 -= l10 * l10;
                    const double i1 = d11 > 0.0 ? rsqrt(d11) : 0.0;
                    const double l21 = (d21 - l20 * l10) * i1, l31 = (d31 - l30 * l10) * i1;
                    d22 -= l20 * l20 + l21 * l21;
                    const double i2 = d22 > 0.0 ? rsqrt(d22) : 0.0;
                    const double l32 = (d32 - l30 * l20 - l31 * l21) * i2;
                    d33 -= l30 * l30 + l31 * l31 + l32 * l32;
                    const double i3 = d33 > 0.0 ? rsqrt(d33) : 0.0;
                    sync();   // everybody has read the raw block before it is overwritten
                    for (int r = jt + tid; r <= n; r += NT)
                    {
                        double *mr = SM_ + r + ldm * jt;
                        const int rr = r - jt;     // position inside the panel: rows 0..3 form the diagonal block
                        double x0 = mr[0] * i0;
                        if (rr == 0) x0 = d00 * i0;
                        mr[0] = x0;
                        if (w4 > 1)
                        {
                            double x1 = rr == 0 ? 0.0 : (rr == 1 ? d11 * i1 : (mr[ldm] - x0 * l10) * i1);
                            mr[ldm] = x1;
                            if (w4 > 2)
                            {
                                double x2 = rr <= 1 ? 0.0 : (rr == 2 ? d22 * i2 : (mr[2 * ldm] - x0 * l20 - x1 * l21) * i2);
                                mr[2 * ldm] = x2;
                                if (w4 > 3)
                                {
                                    double x3 = rr <= 2 ? 0.0 : (rr == 3 ? d33 * i3 : (mr[3 * ldm] - x0 * l30 - x1 * l31 - x2 * l32) * i3);
                                    mr[3 * ldm] = x3;
                                }
                            }
                        }
                    }
                    if (tid == 0)
                    {
                        Linv[jt] = i0;
                        if (w4 > 1) Linv[jt + 1] = i1;
                        if (w4 > 2) Linv[jt + 2] = i2;
                        if (w4 > 3) Linv[jt + 3] = i3;
                    }
                }
                sync();
            }
            // ---- keep the factor (global: column-major n x n, ld n, zeros above the diagonal) and clear the strict upper
            // triangle on chip too (rows r < jt of later tiles were never written): the next stage uses Lxx as a full matrix
            {
                double *Lg = CX.wk + s.w_L;
                for (int r = tid; r < n; r += NT)
                    for (int j = 0; j < n; j++)
                    {
                        double v = 0.0;
                        if (r >= j) v = SM_[r + ldm * j];
                        else SM_[r + ldm * j] = 0.0;
                        Lg[r + n * j] = v;
                    }
                double *lr = CX.wk + s.w_lrow, *li = CX.wk + s.w_Linv;
                for (int j = tid; j < n; j += NT)
                {
                    lr[j] = SM_[n + ldm * j];
                    li[j] = Linv[j];
                }
            }
            ldm_prev = ldm;
            sync();
            };
            if (SNX > 0 && k >= 1 && k <= N - 2) body(SMid{});
            else body(RDims{});
            desc_wait();
            sync();
        }
    }

    // ---------------------------------------------------------------------------------------------
    // backward sweep of the LQ refactorisation (OCP_QP_FACT_LQ_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:1201-1475), the
    // fallback of lq_fact = 1 when a Cholesky step leaves a large linear-system residual, and the only
    // factorisation of lq_fact = 2:   L_k L_k' = Lh Lh' + W W',   Lh = chol(RSQ_k + reg I),
    //   W = [ sqrt(Gamma_b) on the idxb rows | DCt sqrt(Gamma_g) | BAt L_{k+1,xx} ]
    // computed with Householder reflectors from the right on [Lh | W] (non-negative diagonal, the formulas of BLASFEO's
    // GELQF_PD kernels) instead of a Cholesky factorisation of the accumulated sum.  The gradient is not carried as an
    // extra row: it goes through the substitutions of the solve-only sweep, whose results (backward quantities in step
    // set 1, Pb, Zs_inv) this sweep leaves behind, so that forward_pass(after_fact = 0) completes the step.
    // Cold path: generic dimensions only, Lh / L in SM_ (ld even(n+1)), W in a per-QP scratch of the work record
    // (column-major, ld n; thread r owns row r), reflector in SAL_.
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void fact_lq_backward()
    {
        const int N = CX.P.N;
        double *v = SV_, *gam = v + ev(CX.P.nvsmax), *Gam = gam + ev(CX.P.ncmax), *tmp0 = Gam + ev(CX.P.ncmax);
        double *tmp1 = tmp0 + ev(CX.P.nbgmax), *Zi = tmp1 + ev(CX.P.nbgmax), *ds = Zi + ev(2 * CX.P.nsmax);
        double *xprev = ds + ev(2 * CX.P.nsmax), *tmpx = xprev + ev(CX.P.nxmax), *tmpl = tmpx + ev(CX.P.nxmax);
        double *hv = SAL_, *Lis = SAL_ + ev(CX.P.nbgmax + CX.P.nxmax);
        double *Wg = CX.wk + CX.P.w_lq;
        desc_begin(N, -1);
        for (int k = N; k >= 0; k--)
        {
            const StageDesc &s = CX.ring[k & 3];
            desc_next(k, -1);
            const int n = s.n, nu = s.nu, nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc, nx1 = s.nx1, nu1 = s.nu1, n1 = s.n1;
            const int *idxb = CX.ipool + s.idx_off;
            const int ldm = ev(n + 1), mw = nb + ng + nx1, nsolve = k == 0 ? n : nu;
            const double *Ag = CX.qp + s.q_BAt, *Cg = CX.qp + s.q_DCt, *Hg = CX.qp + s.q_RSQ;
            // ---- Gamma, gamma, gradient, Lh <- tril(RSQ) + reg I
            {
                const double *gl = CX.sol + s.sol.lam, *gt = CX.sol + s.sol.t, *grd = rd(0, s), *grm = rm(0, s);
                const double t_min_inv = CX.o.t_min > 0 ? 1.0 / CX.o.t_min : 1e30;
                for (int i = tid; i < nc; i += NT)
                {
                    const double l = gl[i], tt = gt[i], ti = 1.0 / tt;
                    Gam[i] = CX.o.t_lam_min == 1 ? (tt < CX.o.t_min ? t_min_inv : ti) * (l < CX.o.lam_min ? CX.o.lam_min : l) : ti * l;
                    gam[i] = ti * (grm[i] - l * grd[i]);
                }
                const double *g_ = rg(0, s);
                for (int i = tid; i < n; i += NT) v[i] = g_[i];
                for (int r = tid; r < n; r += NT)
                    for (int j = 0; j < n; j++) SM_[r + ldm * j] = r >= j ? __ldg(Hg + r + n * j) + (r == j ? CX.o.reg_prim : 0.0) : 0.0;
                for (int r = tid; r < n; r += NT)
                    for (int j = 0; j < nb; j++) Wg[r + n * j] = 0.0;
            }
            sync();
            if (ns > 0)
            {
                cond_slacks(s, 1, Gam, gam, rg(0, s) + n, Zi, ds, tmp0, tmp1);
                sync();
                for (int j = tid; j < 2 * ns; j += NT)
                {
                    (CX.wk + s.w_Zsi)[j] = Zi[j];
                    (CX.wk + s.step.ux + n)[j] = ds[j];
                }
            }
            else
            {
                for (int i = tid; i < nbg; i += NT)
                {
                    tmp0[i] = Gam[i] + Gam[nbg + i];
                    tmp1[i] = gam[i] - gam[nbg + i];
                }
                sync();
            }
            // ---- W: box columns (one per bound; of bounds on the same variable the reference keeps the last one only,
            // it writes the entry instead of adding to it, :1281-1288), general-constraint columns, A Lxx columns
            if (!s.dup_idxb)
                for (int i = tid; i < nb; i += NT)
                {
                    const int ix = idxb[i];
                    const double g0 = tmp0[i] >= 0.0 ? tmp0[i] : 0.0;
                    Wg[ix + n * i] = sqrt(g0);
                    v[ix] += tmp1[i];
                }
            else if (tid == 0)
                for (int i = 0; i < nb; i++)
                {
                    const int ix = idxb[i];
                    int last = 1;
                    for (int j = i + 1; j < nb; j++) last &= idxb[j] != ix;
                    const double g0 = tmp0[i] >= 0.0 ? tmp0[i] : 0.0;
                    if (last) Wg[ix + n * i] = sqrt(g0);
                    v[ix] += tmp1[i];
                }
            for (int g = tid; g < ng; g += NT)
            {
                const double g0 = tmp0[nb + g] >= 0.0 ? tmp0[nb + g] : 0.0;
                hv[g] = sqrt(g0);
            }
            sync();
            for (int r = tid; r < n; r += NT)
            {
                double acc = 0.0;
                for (int g = 0; g < ng; g++)
                {
                    const double c = __ldg(Cg + r + n * g);
                    Wg[r + n * (nb + g)] = c * hv[g];
                    acc += c * tmp1[nb + g];
                }
                v[r] += acc;
            }
            if (k < N)
            {
                const double *L1 = CX.wk + CX.ring[(k + 1) & 3].w_L + nu1 + n1 * nu1, *b_ = rb(0, s);   // Lxx of stage k+1 (global)
                for (int r = tid; r < n; r += NT)
                    for (int j = 0; j < nx1; j++)
                    {
                        double acc = 0.0;
                        for (int c = j; c < nx1; c++) acc += __ldg(Ag + r + n * c) * L1[c + n1 * j];
                        Wg[r + n * (nbg + j)] = acc;
                    }
                // Pb = Lxx (Lxx' b)
                for (int j = tid; j < nx1; j += NT) tmpx[j] = b_[j];
                sync();
                for (int j = tid; j < nx1; j += NT) tmpl[j] = gdot<false>(L1 + j + n1 * j, 1, tmpx + j, nx1 - j);
                sync();
                double *Pb = CX.wk + s.w_Pb;
                for (int i = tid; i < nx1; i += NT)
                {
                    const double pb = gdot<false>(L1 + i, n1, tmpl, i + 1);
                    Pb[i] = pb;
                    tmpx[i] = pb + xprev[i];
                }
                sync();
                for (int i = tid; i < n; i += NT) v[i] += gdot<true>(Ag + i, n, tmpx, nx1);
            }
            sync();
            // ---- Lh = chol(SM_) in place (right-looking; pivot rule blasfeo_ref/x_lapack_ref.c:84-91)
            for (int j = 0; j < n; j++)
            {
                const double d = SM_[j + ldm * j];
                const double inv = d > 0.0 ? 1.0 / sqrt(d) : 0.0;
                sync();
                for (int r = j + tid; r < n; r += NT) SM_[r + ldm * j] = r == j ? d * inv : SM_[r + ldm * j] * inv;
                sync();
                for (int r = j + 1 + tid; r < n; r += NT)
                {
                    const double a = SM_[r + ldm * j];
                    for (int c = j + 1; c <= r; c++) SM_[r + ldm * c] -= a * SM_[c + ldm * j];
                }
                sync();
            }
            // ---- Householder reflectors from the right, row by row
            for (int i = 0; i < n; i++)
            {
                double part = 0.0;
                for (int j = tid; j < mw; j += NT)
                {
                    const double x = Wg[i + n * j];
                    hv[j] = x;
                    part += x * x;
                }
                const double sigma = rsum(part);
                sync();
                if (sigma == 0.0) continue;
                const double alpha = SM_[i + ldm * i];
                const double beta = sqrt(sigma + alpha * alpha);
                double tmp = alpha <= 0.0 ? alpha - beta : -sigma / (alpha + beta);
                const double tau = 2.0 * tmp * tmp / (sigma + tmp * tmp);
                tmp = 1.0 / tmp;
                for (int j = tid; j < mw; j += NT) hv[j] *= tmp;
                sync();
                if (tid == 0) SM_[i + ldm * i] = beta;
                for (int r = i + 1 + tid; r < n; r += NT)
                {
                    double ww = SM_[r + ldm * i];
                    for (int j = 0; j < mw; j++) ww += Wg[r + n * j] * hv[j];
                    ww = -ww * tau;
                    SM_[r + ldm * i] += ww;
                    for (int j = 0; j < mw; j++) Wg[r + n * j] += ww * hv[j];
                }
                sync();
            }
            // ---- keep the factor; Linv = 1 / diag
            {
                double *Lg = CX.wk + s.w_L, *li = CX.wk + s.w_Linv;
                for (int r = tid; r < n; r += NT)
                    for (int j = 0; j < n; j++) Lg[r + n * j] = r >= j ? SM_[r + ldm * j] : 0.0;
                for (int j = tid; j < n; j += NT)
                {
                    const double inv = 1.0 / SM_[j + ldm * j];
                    li[j] = inv;
                    Lis[j] = inv;
                }
            }
            sync();
            // ---- gradient: TRSV_LNN(_MN) on the first nsolve columns, as in the solve-only sweep
            if (tid < 32)
            {
                for (int j = 0; j < nsolve; j++)
                {
                    double part = 0.0;
                    for (int c = tid; c < j; c += 32) part += SM_[j + ldm * c] * v[c];
                    part = wsum(part);
                    if (tid == 0) v[j] = (v[j] - part) * Lis[j];
                    __syncwarp();
                }
            }
            sync();
            for (int i = nsolve + tid; i < n; i += NT) v[i] -= dot(SM_ + i, ldm, v, 1, nsolve);
            sync();
            {
                double *o_ = vux(1, s);
                for (int i = tid; i < n; i += NT) o_[i] = v[i];
                for (int j = tid; j < s.nx; j += NT) xprev[j] = v[nu + j];
            }
            // ---- gradient row of the factor for the Riccati getters (p_k = Lxx lrow_x): lrow_x = Lxx^{-1} v_x
            sync();
            if (tid < 32)
            {
                for (int j = nsolve; j < n; j++)
                {
                    double part = 0.0;
                    for (int c = nsolve + tid; c < j; c += 32) part += SM_[j + ldm * c] * v[c];
                    part = wsum(part);
                    if (tid == 0) v[j] = (v[j] - part) * Lis[j];
                    __syncwarp();
                }
            }
            sync();
            {
                double *lr = CX.wk + s.w_lrow;
                for (int j = tid; j < n; j += NT) lr[j] = v[j];
            }
            desc_wait();
            sync();
        }
    }

    // ---------------------------------------------------------------------------------------------
    // backward substitution with an existing factorisation (OCP_QP_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:1582-1680)
    // rhs residual set `rhs`, result (backward quantities) into step set `dst`.
    // rm_mode fuses the complementarity right-hand side update of the corrector into this sweep
    // (x_core_qp_ipm_aux.c:695-754): 0 keep res_m; 1 res_m = bkp + dt*dlam - sigma_mu; 2 res_m = bkp - sigma_mu.
    // Matrices are read straight from global memory (lane = row).
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void solve_backward(int rhs, int dst, int use_Pb, int rm_mode, double sigma_mu)
    {
        const int N = CX.P.N;
        double *v = SV_, *gam = v + ev(CX.P.nvsmax), *Gam = gam + ev(CX.P.ncmax), *tmp0 = Gam + ev(CX.P.ncmax);
        double *tmp1 = tmp0 + ev(CX.P.nbgmax), *Zi = tmp1 + ev(CX.P.nbgmax), *ds = Zi + ev(2 * CX.P.nsmax);
        double *xprev = ds + ev(2 * CX.P.nsmax), *tmpx = xprev + ev(CX.P.nxmax), *tmpl = tmpx + ev(CX.P.nxmax);
        double *Ls = SM_, *Lis = SAL_, *pbs = Lis + ev(CX.P.nmax);   // staged from global memory at the top of each stage
        desc_begin(N, -1);
        for (int k = N; k >= 0; k--)
        {
            const StageDesc &s = CX.ring[k & 3];
            desc_next(k, -1);
            auto body = [&](auto dd) {
            const int n = dd.n(s), nu = dd.nu(s), nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc, nx1 = dd.nx1(s), nu1 = dd.nu1(s), n1 = dd.n1(s);
            const int *idxb = CX.ipool + s.idx_off;
            const int nsolve = k == 0 ? n : nu;
            const double *Lg = CX.wk + s.w_L, *Li = CX.wk + s.w_Linv;
            pf1(CX.qp + s.q_BAt, n * nx1);
            pf1(Lg, n * nsolve);
            if (k > 0)
            {
                const StageDesc &sp = CX.ring[(k - 1) & 3];
                prefetch_l2(CX.qp + sp.q_BAt, (unsigned) (ev(sp.n * sp.nx1) * sizeof(double)));
                prefetch_l2(CX.wk + sp.w_fac, sp.w_fac_bytes);
            }
            {
                // pure copies first, as asynchronous global -> shared copies (all in flight at once) ...
                cpv(v, rg(rhs, s), n);
                if (ns > 0) cpv(Zi, CX.wk + s.w_Zsi, 2 * ns);
                cpvb(Ls, Lg, n * nsolve);
                cpvb(Lis, Li, nsolve);
                if (k < N && use_Pb) cpvb(pbs, CX.wk + s.w_Pb, nx1);
                // ... then the constraint quantities through registers while those are in flight
                const double *gl = CX.sol + s.sol.lam, *gt = CX.sol + s.sol.t, *grd = rd(rhs, s), *gm = CX.qp + s.q_dmask;
                double *grm = rm(rhs, s);
                const double *bk = CX.wk + s.w_rmb, *dl = CX.wk + s.step.lam, *dtt = CX.wk + s.step.t;
                const double t_min_inv = CX.o.t_min > 0 ? 1.0 / CX.o.t_min : 1e30;
                for (int i = tid; i < nc; i += NT)
                {
                    const double l = gl[i], tt = gt[i], ti = 1.0 / tt;
                    double m;
                    if (rm_mode == 0) m = grm[i];
                    else
                    {
                        m = rm_mode == 1 ? bk[i] + dtt[i] * dl[i] - sigma_mu : bk[i] - sigma_mu;
                        if (CX.mask_constr) m *= __ldg(gm + i);
                        grm[i] = m;
                    }
                    // the slack elimination needs the Gamma of the factorisation (clipped when t_lam_min==1)
                    Gam[i] = (ns > 0 && CX.o.t_lam_min == 1) ? (tt < CX.o.t_min ? t_min_inv : ti) * (l < CX.o.lam_min ? CX.o.lam_min : l) : ti * l;
                    gam[i] = ti * (m - l * grd[i]);
                }
                desc_wait();
            }
            sync();
            if (ns > 0)
            {
                cond_slacks(s, 0, Gam, gam, rg(rhs, s) + n, Zi, ds, tmp0, tmp1);
                sync();
                double *o_ = vux(dst, s) + n;
                for (int j = tid; j < 2 * ns; j += NT) o_[j] = ds[j];
            }
            else
            {
                for (int i = tid; i < nbg; i += NT) tmp1[i] = gam[i] - gam[nbg + i];
                sync();
            }
            if (!s.dup_idxb)
                for (int i = tid; i < nb; i += NT) v[idxb[i]] += tmp1[i];
            else if (tid == 0)
                for (int i = 0; i < nb; i++) v[idxb[i]] += tmp1[i];
            if (k < N)
            {
                if (use_Pb)
                {
                    for (int j = tid; j < nx1; j += NT) tmpx[j] = xprev[j] + pbs[j];
                }
                else
                {   // P b = Lxx (Lxx' b) from the factor of stage k+1 in global memory
                    const double *L1 = CX.wk + CX.ring[(k + 1) & 3].w_L + nu1 + n1 * nu1, *b_ = rb(rhs, s);
                    for (int j = tid; j < nx1; j += NT) tmpx[j] = b_[j];
                    sync();
                    for (int j = tid; j < nx1; j += NT) tmpl[j] = gdot<false>(L1 + j + n1 * j, 1, tmpx + j, nx1 - j);
                    sync();
                    for (int i = tid; i < nx1; i += NT) tmpx[i] = gdot<false>(L1 + i, n1, tmpl, i + 1) + xprev[i];
                }
            }
            sync();
            {
                const double *Ag = CX.qp + s.q_BAt, *Cg = CX.qp + s.q_DCt;
                for (int i = tid; i < n; i += NT)
                {
                    double acc = v[i] + gdot<true>(Ag + i, n, tmpx, nx1);
                    for (int g = 0; g < ng; g++) acc += __ldg(Cg + i + n * g) * tmp1[nb + g];
                    v[i] = acc;
                }
            }
            sync();
            // TRSV_LNN(_MN): forward substitution on the first nsolve columns
            if (tid < 32)
            {
                for (int j = 0; j < nsolve; j++)
                {
                    double part = 0.0;
                    for (int c = tid; c < j; c += 32) part += Ls[j + n * c] * v[c];
                    part = wsum(part);
                    if (tid == 0) v[j] = (v[j] - part) * Lis[j];
                    __syncwarp();
                }
            }
            sync();
            for (int i = nsolve + tid; i < n; i += NT) v[i] -= dot(Ls + i, n, v, 1, nsolve);
            sync();
            {
                double *o_ = vux(dst, s);
                for (int i = tid; i < n; i += NT) o_[i] = v[i];
                for (int j = tid; j < s.nx; j += NT) xprev[j] = v[nu + j];
            }
            sync();
            };
            if (SNX > 0 && k >= 1 && k <= N - 2) body(SMid{});
            else body(RDims{});
            desc_wait();
            sync();
        }
    }

    // ---------------------------------------------------------------------------------------------
    // forward sweep (x_ocp_qp_kkt.c:968-1006 / 1682-1722) + step of the constraint variables
    // (:1176-1193, EXPAND_SLACKS :524-598, COMPUTE_LAM_T_QP x_core_qp_ipm_aux.c:164-189) + the
    // ratio test (COMPUTE_ALPHA_QP :375-398).  after_fact: start from -lrow, pi = P x + p with p from lrow;
    // else: start from the backward quantities stored in the step set, pi = p_backward + P x.
    // do_lin: the residual of the linear system (OCP_QP_RES_COMPUTE_LIN) of this step is evaluated in the same
    // sweep -> residual set 1, norms in lin_nrm (only res_g needs matrix work: the other three parts vanish up to
    // round-off by construction of x_{k+1}, dt and dlam and are evaluated with the reference's formulas).
    // Returns the step length alpha of this step set.  Matrices straight from global memory.
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ double forward_pass(int rhs, int dst, int after_fact, int mask_out, int do_lin, double lin_nrm[4])
    {
        const int N = CX.P.N;
        double *v = SV_, *x1 = v + ev(CX.P.nvsmax), *tmp = x1 + ev(CX.P.nxmax), *p1 = tmp + ev(CX.P.nxmax), *pik = p1 + ev(CX.P.nxmax);
        double *pim = pik + ev(CX.P.nxmax), *Gam = pim + ev(CX.P.nxmax), *dt = Gam + ev(CX.P.ncmax), *lam = dt + ev(CX.P.ncmax);
        double *dlm = lam + ev(CX.P.ncmax), *Zi = dlm + ev(CX.P.ncmax), *ds = Zi + ev(2 * CX.P.nsmax), *g_ = ds + ev(2 * CX.P.nsmax);
        double *tmp0 = g_ + ev(CX.P.nvsmax);
        // staging areas borrowed from the factorisation buffers (idle during this sweep): the first nsolve columns of L_k
        // and the per-stage vectors, all fetched in ONE burst at the top of the stage instead of one exposed global
        // round trip per dependent phase
        double *Ls = SM_, *Lis = SAL_, *bs = Lis + ev(CX.P.nmax), *ts = bs + ev(CX.P.nxmax), *rds = ts + ev(CX.P.ncmax);
        double *rms = rds + ev(CX.P.ncmax), *mks = rms + ev(CX.P.ncmax);
        double alpha = 1.0;
        double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0;
        int f0 = 0, f1 = 0, f2 = 0, f3 = 0;
        desc_begin(0, 1);
        for (int k = 0; k <= N; k++)
        {
            const StageDesc &s = CX.ring[k & 3];
            desc_next(k, 1);
            auto body = [&](auto dd) {
            const int n = dd.n(s), nu = dd.nu(s), nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc, nx1 = dd.nx1(s), nu1 = dd.nu1(s), n1 = dd.n1(s);
            const int *idxb = CX.ipool + s.idx_off, *rev = idxb + nb;
            const int nsolve = k == 0 ? n : nu;
            const double *Lg = CX.wk + s.w_L, *Li = CX.wk + s.w_Linv;
            const double *Ag = CX.qp + s.q_BAt, *Cg = CX.qp + s.q_DCt;
            pf1(Lg, n * nsolve);
            pf1(Ag, n * nx1);
            if (k < N) pf1(CX.wk + CX.ring[(k + 1) & 3].w_L + n1 * nu1, n1 * nx1);
            if (do_lin) pf1(CX.qp + s.q_RSQ, n * n);
            {
                const double *src = after_fact ? CX.wk + s.w_lrow : vux(dst, s);
                for (int i = tid; i < nsolve; i += NT) v[i] = -src[i];
                // x part (k>0) was written into v by the previous stage
            }
            if (k < N)
            {
                const StageDesc &s1 = CX.ring[(k + 1) & 3];
                const double *ps = after_fact ? CX.wk + s1.w_lrow + nu1 : vux(dst, s1) + nu1;   // p part / backward value of x_{k+1}
                for (int j = tid; j < nx1; j += NT) p1[j] = ps[j];
                prefetch_l2(CX.qp + s1.q_stage, s1.q_stage_bytes);
            }
            if (ns > 0)
            {
                const double *z_ = CX.wk + s.w_Zsi, *d_ = vux(dst, s) + n;
                for (int j = tid; j < 2 * ns; j += NT) { Zi[j] = z_[j]; ds[j] = d_[j]; }
            }
            {
                for (int e = tid; e < n * nsolve; e += NT) Ls[e] = Lg[e];
                for (int j = tid; j < nsolve; j += NT) Lis[j] = Li[j];
                const double *b_ = rb(rhs, s);
                for (int j = tid; j < nx1; j += NT) bs[j] = b_[j];
                const double *gl = CX.sol + s.sol.lam, *gt = CX.sol + s.sol.t, *grd = rd(rhs, s), *grm = rm(rhs, s), *gm = CX.qp + s.q_dmask;
                for (int i = tid; i < nc; i += NT)
                {
                    lam[i] = gl[i];
                    ts[i] = gt[i];
                    rds[i] = grd[i];
                    rms[i] = grm[i];
                    mks[i] = CX.mask_constr ? __ldg(gm + i) : 1.0;
                }
            }
            sync();
            // TRSV_LTN(_MN): back substitution with the transposed factor on the first nsolve unknowns
            if (tid < 32)
            {
                for (int j = nsolve - 1; j >= 0; j--)
                {
                    double part = 0.0;
                    for (int i = j + 1 + tid; i < n; i += 32) part += Ls[i + n * j] * v[i];
                    part = wsum(part);
                    if (tid == 0) v[j] = (v[j] - part) * Lis[j];
                    __syncwarp();
                }
            }
            sync();
            {
                double *o_ = vux(dst, s);
                for (int i = tid; i < n; i += NT) o_[i] = v[i];
            }
            if (k < N)
            {
                const double *L1 = CX.wk + CX.ring[(k + 1) & 3].w_L + nu1 + n1 * nu1;      // Lxx of stage k+1: L1[i + n1*j]
                double *ob = rb(1, s);
                for (int j = tid; j < nx1; j += NT)
                {
                    const double acc = gdot<true>(Ag + n * j, 1, v, n), bv = bs[j];
                    const double xj = bv + acc;
                    x1[j] = xj;
                    if (do_lin)
                    {
                        const double r = bv - xj + acc;
                        ob[j] = r;
                        const double a = fabs(r);
                        m1 = fmax(m1, a);
                        f1 |= (a != a);
                    }
                }
                sync();
                for (int j = tid; j < nx1; j += NT)
                {
                    const double acc = gdot<false>(L1 + j + n1 * j, 1, x1 + j, nx1 - j);
                    tmp[j] = after_fact ? acc + p1[j] : acc;
                }
                sync();
                double *pi = vpi(dst, s);
                for (int i = tid; i < nx1; i += NT)
                {
                    const double acc = gdot<false>(L1 + i, n1, tmp, i + 1);
                    const double pv = after_fact ? acc : acc + p1[i];
                    pi[i] = pv;
                    pik[i] = pv;
                }
            }
            // ---- constraint part of the step at this stage
            {
                const double t_min_inv = CX.o.t_min > 0 ? 1.0 / CX.o.t_min : 1e30;
                for (int i = tid; i < nc; i += NT)
                {
                    const double l = lam[i], tt = ts[i];
                    Gam[i] = (ns > 0 && CX.o.t_lam_min == 1) ? (tt < CX.o.t_min ? t_min_inv : 1.0 / tt) * (l < CX.o.lam_min ? CX.o.lam_min : l)
                                                          : (1.0 / tt) * l;
                }
                for (int i = tid; i < nbg; i += NT)
                {
                    const double a = i < nb ? v[idxb[i]] : gdot<true>(Cg + n * (i - nb), 1, v, n);
                    dt[i] = a;
                    dt[nbg + i] = -a;
                }
                if (ns > 0)
                {
                    sync();
                    for (int j = tid; j < 2 * ns; j += NT)
                    {
                        const int jj = j < ns ? j : j - ns, offc = j < ns ? 0 : nbg;
                        double d = ds[j];
                        for (int i = 0; i < nbg; i++)
                            if (rev[i] == jj) d += Gam[offc + i] * dt[offc + i];
                        d = -Zi[j] * d;
                        ds[j] = d;
                        dt[2 * nbg + j] = d;
                    }
                    sync();
                    for (int i = tid; i < 2 * nbg; i += NT)
                    {
                        const int up = i >= nbg, ii = up ? i - nbg : i;
                        if (rev[ii] >= 0) dt[i] += ds[(up ? ns : 0) + rev[ii]];
                    }
                    double *o_ = vux(dst, s) + n;
                    for (int j = tid; j < 2 * ns; j += NT) o_[j] = ds[j];
                }
                sync();
                double *odl = vlam(dst, s), *odt = vt(dst, s), *ld_ = rd(1, s), *lm_ = rm(1, s);
                for (int i = tid; i < nc; i += NT)
                {
                    const double l = lam[i], tt = ts[i], ti = 1.0 / tt, rdi = rds[i], rmi = rms[i];
                    const double dtr = dt[i];
                    double dl = -ti * (rmi + (l * dtr) - (l * rdi));
                    double dti = dtr - rdi;
                    const double mk = mks[i];
                    if (CX.mask_constr && mask_out)
                    {
                        dl *= mk;
                        dti *= mk;
                    }
                    odl[i] = dl;
                    odt[i] = dti;
                    dlm[i] = CX.mask_constr ? dl * mk : dl;     // masked step multipliers (tmp_lam_mask of the linear residual)
                    if (dst == 1)
                    {   // ratio test on the main step (min over constraints, see COMPUTE_ALPHA_QP)
                        if (CX.o.m_relax == 0.0)
                        {
                            if (l + dl < 0.0) alpha = fmin(alpha, -l / dl);
                            if (tt + dti < 0.0) alpha = fmin(alpha, -tt / dti);
                        }
                        else
                            alpha = fmin(alpha, crit_step_m(l, tt, dl, dti, m_safe() * CX.o.m_relax * mk));
                    }
                    if (do_lin)
                    {
                        // res_d = rhs_d + dt -/+ (v[idxb] | C'v) [- ds] = rhs_d + dt - dtr ;  res_m = rhs_m + lam dt + dlam t
                        double r = (dti + rdi) - dtr;
                        if (CX.mask_constr) r *= mk;
                        ld_[i] = r;
                        double a = fabs(r);
                        m2 = fmax(m2, a);
                        f2 |= (a != a);
                        double mm = rmi + l * dti + dl * tt;
                        if (CX.mask_constr) mm *= mk;
                        lm_[i] = mm;
                        a = fabs(mm);
                        m3 = fmax(m3, a);
                        f3 |= (a != a);
                    }
                }
            }
            sync();
            if (do_lin)
            {
                // ---- res_g of the linear system (lane = row): H dux + rhs_g - dpi_{k-1} + A dpi_k + constraint multipliers
                const double *Hg = CX.qp + s.q_RSQ, *gv = rg(rhs, s);
                for (int i = tid; i < nbg; i += NT) tmp0[i] = dlm[nbg + i] - dlm[i];
                sync();
                for (int i = tid; i < n; i += NT)
                {
                    double r = gdot_sym(Hg, n, i, v) + gv[i];
                    if (k > 0 && i >= nu) r -= pim[i - nu];
                    r += gdot<true>(Ag + i, n, pik, nx1);
                    for (int g = 0; g < ng; g++) r += __ldg(Cg + i + n * g) * tmp0[nb + g];
                    g_[i] = r;
                }
                sync();
                if (!s.dup_idxb)
                    for (int i = tid; i < nb; i += NT) g_[idxb[i]] += tmp0[i];
                else if (tid == 0)
                    for (int i = 0; i < nb; i++) g_[idxb[i]] += tmp0[i];
                if (ns > 0)
                {
                    const double *Z = CX.qp + s.q_Z, *zv = rg(rhs, s) + n;
                    for (int j = tid; j < 2 * ns; j += NT)
                    {
                        double r = Z[j] * ds[j] + zv[j] - dlm[2 * nbg + j];
                        const int jj = j < ns ? j : j - ns, offl = j < ns ? 0 : nbg;
                        for (int i = 0; i < nbg; i++)
                            if (rev[i] == jj) r -= dlm[offl + i];
                        g_[n + j] = r;
                    }
                }
                sync();
                double *og = rg(1, s);
                for (int i = tid; i < n + 2 * ns; i += NT)
                {
                    const double r = g_[i];
                    og[i] = r;
                    const double a = fabs(r);
                    m0 = fmax(m0, a);
                    f0 |= (a != a);
                }
            }
            if (k < N)
            {
                for (int j = tid; j < nx1; j += NT)
                {
                    v[nu1 + j] = x1[j];
                    pim[j] = pik[j];
                }
            }
            sync();
            };
            if (SNX > 0 && k >= 1 && k <= N - 2) body(SMid{});
            else body(RDims{});
            desc_wait();
            sync();
            if (k + 2 <= N) prefetch_l2(CX.wk + CX.ring[(k + 2) & 3].w_fac, CX.ring[(k + 2) & 3].w_fac_bytes);   // factor needed by the next stage (its Lxx)
        }
        if (do_lin)
        {
            lin_nrm[0] = rmax_nan(m0, f0);
            lin_nrm[1] = rmax_nan(m1, f1);
            lin_nrm[2] = rmax_nan(m2, f2);
            lin_nrm[3] = rmax_nan(m3, f3);
        }
        return rmin(alpha);
    }

    // m != 0 (acados' tau_min option): largest step of one constraint that keeps lam, t >= 0 and lam*t >= m1 = m_safe*m, by
    // COMPUTE_ALPHA_QP's rule (x_core_qp_ipm_aux.c:398-440; evaluated from alpha = 1 per constraint, the minimum over the
    // constraints equals the reference's sequential pass because each test is monotone in the step length)
    __device__ __forceinline__ double m_safe() const { return (CX.o.mode == CUIPM_SPEED_ABS || CX.o.mode == CUIPM_SPEED) ? 0.3 : 0.5; }
    __device__ __noinline__ double crit_step_m(double l, double t, double dl, double dt, double m1) const
    {
        double a = 1.0, l1 = l + dl, t1 = t + dt;
        if (l1 < 0.0) { a = -l / dl; l1 = l + a * dl; }
        if (t1 < 0.0) { a = -t / dt; t1 = t + a * dt; }
        if (l1 * t1 - m1 < -1e-12)
        {
            const double c = l * t - m1;
            if (c > 0.0)
            {
                const double aa = dl * dt, b = dl * t + l * dt;
                const double d = b * b - 4.0 * aa * c, sd = sqrt(d), tmp = 0.5 / aa;
                a = (-b - sd) * tmp;
            }
            else
                a = 0.0;
        }
        return a;
    }

    // step length of the main step from global memory (after iterative refinement changed it)
    __device__ __noinline__ double alpha_pass()
    {
        double alpha = 1.0;
        for (int k = 0; k <= CX.P.N; k++)
        {
            const StageDesc s = CX.SD[k];
            const double *l = CX.sol + s.sol.lam, *t = CX.sol + s.sol.t, *dl = CX.wk + s.step.lam, *dt = CX.wk + s.step.t;
            for (int i = tid; i < s.nc; i += NT)
            {
                if (CX.o.m_relax == 0.0)
                {
                    if (l[i] + dl[i] < 0.0) alpha = fmin(alpha, -l[i] / dl[i]);
                    if (t[i] + dt[i] < 0.0) alpha = fmin(alpha, -t[i] / dt[i]);
                }
                else
                    alpha = fmin(alpha, crit_step_m(l[i], t[i], dl[i], dt[i], m_safe() * CX.o.m_relax * __ldg(CX.qp + s.q_dmask + i)));
            }
        }
        return rmin(alpha);
    }

    // COMPUTE_MU_AFF_QP (x_core_qp_ipm_aux.c:636-668)
    __device__ __noinline__ double mu_aff_pass(double alpha)
    {
        double acc = 0.0;
        for (int k = 0; k <= CX.P.N; k++)
        {
            const StageDesc s = CX.SD[k];
            const double *l = CX.sol + s.sol.lam, *t = CX.sol + s.sol.t, *dl = CX.wk + s.step.lam, *dt = CX.wk + s.step.t;
            if (CX.o.m_relax == 0.0)
                for (int i = tid; i < s.nc; i += NT) acc += fabs((l[i] + alpha * dl[i]) * (t[i] + alpha * dt[i]));
            else        // m != 0 (tau_min option): |(lam + alpha dlam)(t + alpha dt) - m|, m = qp->m * d_mask
                for (int i = tid; i < s.nc; i += NT)
                    acc += fabs(-CX.o.m_relax * __ldg(CX.qp + s.q_dmask + i) + (l[i] + alpha * dl[i]) * (t[i] + alpha * dt[i]));
        }
        return rsum(acc) * CX.nc_mask_inv;
    }

    // step <- step + itref
    __device__ __noinline__ void add_itref()
    {
        for (int k = 0; k <= CX.P.N; k++)
        {
            const StageDesc s = CX.SD[k];
            double *a = CX.wk + s.step.ux;
            const double *b = CX.wk + s.itref.ux;
            for (int i = tid; i < s.n + 2 * s.ns; i += NT) a[i] += b[i];
            a = CX.wk + s.step.pi; b = CX.wk + s.itref.pi;
            for (int i = tid; i < s.nx1; i += NT) a[i] += b[i];
            a = CX.wk + s.step.lam; b = CX.wk + s.itref.lam;
            for (int i = tid; i < s.nc; i += NT) a[i] += b[i];
            a = CX.wk + s.step.t; b = CX.wk + s.itref.t;
            for (int i = tid; i < s.nc; i += NT) a[i] += b[i];
        }
        sync();
    }

    // the throughput kernel keeps the caller's pi, lam, t of a warm start in the refinement vectors before it touches them
    __device__ __noinline__ void restore_warm_start()
    {
        for (int k = 0; k <= CX.P.N; k++)
        {
            const StageDesc s = CX.SD[k];
            for (int i = tid; i < s.nx1; i += NT) (CX.sol + s.sol.pi)[i] = (CX.wk + s.itref.pi)[i];
            for (int i = tid; i < s.nc; i += NT)
            {
                (CX.sol + s.sol.lam)[i] = (CX.wk + s.itref.lam)[i];
                (CX.sol + s.sol.t)[i] = (CX.wk + s.itref.t)[i];
            }
        }
        sync();
    }

    // OCP_QP_INIT_VAR, var_init_scheme 1 (x_ocp_qp_ipm.c:1611-1760,1884-2022)
    __device__ __noinline__ void init_var()
    {
        const double thr0 = 0.1;
        const int N = CX.P.N;
        // the reference's plugin zeroes the primal iterate before every solve, whatever warm_start says
        // (acados/ocp_qp/ocp_qp_hpipm.c:333-336): warm starts carry over pi, lam and t only
        if (CX.o.warm_start >= 2)
        {
            const double lmin = CX.o.warm_start >= 3 ? CX.o.lam0_min : thr0, tmin = CX.o.warm_start >= 3 ? CX.o.t0_min : thr0;
            for (int k = 0; k <= N; k++)
            {
                const StageDesc s = CX.SD[k];
                double *l = CX.sol + s.sol.lam, *t = CX.sol + s.sol.t, *gux = CX.sol + s.sol.ux;
                for (int i = tid; i < s.n + 2 * s.ns; i += NT) gux[i] = 0.0;
                for (int i = tid; i < s.nc; i += NT)
                {
                    if (l[i] < lmin) l[i] = lmin;
                    if (t[i] < tmin) t[i] = tmin;
                }
            }
            sync();
            return;
        }
        double *ux = SV_, *tt = ux + ev(CX.P.nvsmax), *cg = tt + ev(CX.P.ncmax);
        for (int k = 0; k <= N; k++)
        {
            const StageDesc s = CX.SD[k];
            const int n = s.n, nb = s.nb, ng = s.ng, ns = s.ns, nbg = s.nbg, nc = s.nc;
            const int *idxb = CX.ipool + s.idx_off, *rev = idxb + nb;
            const double *d = CX.qp + s.q_d;
            double *gux = CX.sol + s.sol.ux, *gpi = CX.sol + s.sol.pi, *gl = CX.sol + s.sol.lam, *gt = CX.sol + s.sol.t;
            for (int i = tid; i < s.nx1; i += NT) gpi[i] = 0.0;
            if (CX.o.t0_init == 0 || CX.o.t0_init == 1)
            {
                const double l0 = CX.o.t0_init == 0 ? sqrt(CX.o.mu0) : CX.o.mu0, t0 = CX.o.t0_init == 0 ? sqrt(CX.o.mu0) : 1.0;
                for (int i = tid; i < n + 2 * ns; i += NT) gux[i] = 0.0;
                for (int i = tid; i < nc; i += NT) { gl[i] = l0; gt[i] = t0; }
                continue;
            }
            for (int i = tid; i < n + 2 * ns; i += NT) ux[i] = 0.0;
            sync();
            for (int j = tid; j < 2 * ns; j += NT)
            {
                double tj = ux[n + j] - d[2 * nbg + j];
                if (tj < thr0)
                {
                    tj = thr0;
                    ux[n + j] = d[2 * nbg + j] + tj;
                }
                tt[2 * nbg + j] = tj;
            }
            sync();
            // boxes: serial over constraints if an index repeats, else parallel
            for (int j = (s.dup_idxb ? 0 : tid); j < nb && (!s.dup_idxb || tid == 0); j += (s.dup_idxb ? 1 : NT))
            {
                const int ix = idxb[j];
                double tl = ux[ix], tu = -ux[ix];
                if (ns > 0 && rev[j] != -1) { tl += ux[n + rev[j]]; tu += ux[n + ns + rev[j]]; }
                tl -= d[j];
                tu -= d[nbg + j];
                if (tl < thr0)
                {
                    if (tu < thr0)
                    {
                        ux[ix] = 0.5 * (d[j] - d[nbg + j]);
                        tl = thr0; tu = thr0;
                    }
                    else
                    {
                        tl = thr0;
                        ux[ix] = d[j] + thr0;
                    }
                }
                else if (tu < thr0)
                {
                    tu = thr0;
                    ux[ix] = -d[nbg + j] - thr0;
                }
                tt[j] = tl;
                tt[nbg + j] = tu;
            }
            sync();
            if (ng > 0)
            {
                const double *Cm = CX.qp + s.q_DCt;
                for (int g = tid; g < ng; g += NT)
                {
                    double acc = 0.0;
                    for (int i = 0; i < n; i++) acc += Cm[i + n * g] * ux[i];
                    cg[g] = acc;
                }
                sync();
                for (int g = tid; g < ng; g += NT)
                {
                    double tl = cg[g], tu = -cg[g];
                    if (ns > 0 && rev[nb + g] != -1) { tl += ux[n + rev[nb + g]]; tu += ux[n + ns + rev[nb + g]]; }
                    tl -= d[nb + g];
                    tu -= d[nbg + nb + g];
                    tt[nb + g] = thr0 > tl ? thr0 : tl;
                    tt[nbg + nb + g] = thr0 > tu ? thr0 : tu;
                }
                sync();
            }
            for (int i = tid; i < n + 2 * ns; i += NT) gux[i] = ux[i];
            for (int i = tid; i < nc; i += NT)
            {
                gt[i] = tt[i];
                gl[i] = CX.o.mu0 / tt[i];
            }
            sync();
        }
        sync();
    }

    // ---------------------------------------------------------------------------------------------
    // solution sensitivities (OCP_QP_IPM_SENS_FRW / _ADJ, x_ocp_qp_ipm.c:3285-3444): OCP_QP_SOLVE_KKT_STEP with the seed as
    // right-hand side, at the iterate of the last factorisation (CX.sol points at the backup record), Pb recomputed.
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void sens(const double *seed, double *out, int adjoint)
    {
        const int N = CX.P.N;
        for (int k = 0; k <= N; k++)
        {
            const StageDesc s = CX.SD[k];
            double *g_ = rg(0, s), *b_ = rb(0, s), *d_ = rd(0, s), *m_ = rm(0, s);
            const double *tb = CX.sol + s.sol.t;
            for (int i = tid; i < s.n + 2 * s.ns; i += NT) g_[i] = seed[s.sol.ux + i];
            for (int i = tid; i < s.nx1; i += NT) b_[i] = seed[s.sol.pi + i];
            for (int i = tid; i < s.nc; i += NT)
            {
                d_[i] = seed[s.sol.lam + i];
                m_[i] = adjoint ? seed[s.sol.t + i] * tb[i] : seed[s.sol.t + i];
            }
        }
        sync();
        double dmy4[4];
        solve_backward(0, 1, 0, 0, 0.0);
        forward_pass(0, 1, 0, 0, 0, dmy4);
        for (int k = 0; k <= N; k++)
        {
            const StageDesc s = CX.SD[k];
            const double *tb = CX.sol + s.sol.t;
            for (int i = tid; i < s.n + 2 * s.ns; i += NT) out[s.sol.ux + i] = (CX.wk + s.step.ux)[i];
            for (int i = tid; i < s.nx1; i += NT) out[s.sol.pi + i] = (CX.wk + s.step.pi)[i];
            for (int i = tid; i < s.nc; i += NT)
            {
                out[s.sol.lam + i] = (CX.wk + s.step.lam)[i];
                const double dt = (CX.wk + s.step.t)[i];
                out[s.sol.t + i] = adjoint ? dt * (1.0 / tb[i]) : dt;
            }
        }
        sync();
    }

    // ---------------------------------------------------------------------------------------------
    // driver (OCP_QP_IPM_SOLVE x_ocp_qp_ipm.c:2684-3120 + OCP_QP_IPM_DELTA_STEP :2208-2682)
    // ---------------------------------------------------------------------------------------------
    __device__ __noinline__ void solve(cuipm_info *info, double *stat)
    {
        const int N = CX.P.N;
        const int SM = CUIPM_STAT_M;
        double res_max[4] = {0, 0, 0, 0}, mu = 0.0, obj = 0.0, gap = 0.0;
        int lq_count = 0, force_lq = 0, status, iter = 0;
        if (stat)
            for (int i = tid; i < SM * (CX.o.stat_max + 1); i += NT) stat[i] = 0.0;
#ifdef CUIPM_PROFILE
        if (tid == 0)
            for (int i = 0; i < 16; i++) CX.prof[i] = 0;
#endif

        // constraint mask census (x_ocp_qp_ipm.c:2774-2806)
        int cnt = 0;
        for (int k = 0; k <= N; k++)
        {
            const StageDesc s = CX.SD[k];
            const double *gm = CX.qp + s.q_dmask;
            for (int i = tid; i < s.nc; i += NT) cnt += gm[i] != 0.0;
        }
        const int nc_mask = (int) (rsum((double) cnt) + 0.5);
        CX.mask_constr = nc_mask < CX.P.nct;
        CX.nc_mask_inv = nc_mask > 0 ? 1.0 / nc_mask : 0.0;

        if (CX.P.nct == 0 || nc_mask == 0)
        {
            // no (active) constraints: one Riccati pass on the QP data (OCP_QP_FACT_SOLVE_KKT_UNCONSTR, x_ocp_qp_kkt.c:39-137)
            for (int k = 0; k <= N; k++)
            {
                const StageDesc s = CX.SD[k];
                double *l = CX.sol + s.sol.lam, *t = CX.sol + s.sol.t, *d_ = rd(0, s), *m_ = rm(0, s), *g_ = rg(0, s), *b_ = rb(0, s);
                for (int i = tid; i < s.nc; i += NT) { l[i] = 0.0; t[i] = 1.0; d_[i] = 0.0; m_[i] = 0.0; }
                for (int i = tid; i < s.n; i += NT) g_[i] = (CX.qp + s.q_rq)[i];
                for (int i = tid; i < 2 * s.ns; i += NT) g_[s.n + i] = (CX.qp + s.q_z)[i];
                for (int i = tid; i < s.nx1; i += NT) b_[i] = (CX.qp + s.q_b)[i];
            }
            sync();
            fact_backward();
            double dmy4[4], dmy;
            forward_pass(0, 1, 1, 1, 0, dmy4);
            for (int k = 0; k <= N; k++)
            {
                const StageDesc s = CX.SD[k];
                for (int i = tid; i < s.n + 2 * s.ns; i += NT) (CX.sol + s.sol.ux)[i] = (CX.wk + s.step.ux)[i];
                for (int i = tid; i < s.nx1; i += NT) (CX.sol + s.sol.pi)[i] = (CX.wk + s.step.pi)[i];
            }
            sync();
            res_pass(0, 0, -1, 0, 0, 0.0, mu, obj, gap, res_max, dmy);
            if (stat && 0 < CX.o.stat_max && tid == 0)
            {   // column quirk of the reference's unconstrained branch (x_ocp_qp_ipm.c:2822-2829)
                stat[6] = res_max[0]; stat[7] = res_max[1]; stat[8] = res_max[2]; stat[9] = res_max[3];
                stat[10] = gap; stat[11] = obj;
            }
            const double u0 = CX.sol[CX.SD[0].sol.ux];
            status = (u0 != u0) ? CUIPM_NAN_SOL : CUIPM_SUCCESS;
        }
        else
        {
            init_var();
            if (CX.mask_constr)
            {
                for (int k = 0; k <= N; k++)
                {
                    const StageDesc s = CX.SD[k];
                    double *l = CX.sol + s.sol.lam;
                    const double *gm = CX.qp + s.q_dmask;
                    for (int i = tid; i < s.nc; i += NT) l[i] *= gm[i];
                }
                sync();
            }
            double alpha = 1.0, res_m_tau = 0.0;
            res_pass(0, 0, -1, 0, 0, 0.0, mu, obj, gap, res_max, res_m_tau);
            if (stat && 0 < CX.o.stat_max && tid == 0)
            {
                stat[7] = res_max[0]; stat[8] = res_max[1]; stat[9] = res_max[2]; stat[10] = res_max[3];
                stat[11] = gap; stat[12] = obj;
            }
            int kk;
            for (kk = 0; kk < CX.o.iter_max && alpha > CX.o.alpha_min
                         && (res_max[0] > CX.o.res_g_max || res_max[1] > CX.o.res_b_max || res_max[2] > CX.o.res_d_max
                             || res_m_tau > CX.o.res_m_max || gap > CX.o.dual_gap_max);
                 kk++)
            {
                double *st = (stat && kk + 1 < CX.o.stat_max) ? stat + SM * (size_t) (kk + 1) : nullptr;
                double nrm[4] = {0, 0, 0, 0}, dmy;
                PROF_T0();
                // affine direction: res_m already holds lam*t - tau_min (written by the residual sweep)
                // Cholesky, with a switch to LQ for the rest of the solve once a Cholesky step leaves a large residual in the
                // linear system (x_ocp_qp_ipm.c:2246-2346)
                int used_lq = 0;
                if (CX.o.lq_fact == 0 || (CX.o.lq_fact == 1 && !force_lq))
                {
                    fact_backward();
                    PROF_ADD(2);
                    alpha = forward_pass(0, 1, 1, 1, CX.o.lq_fact == 1, nrm);
                    PROF_ADD(3);
                    if (CX.o.lq_fact == 1)
                    {
                        const double g00 = (CX.wk + CX.SD[0].ires.g)[0];
                        if ((nrm[0] == 0.0 && g00 != g00) || nrm[0] > 1e-5 || nrm[1] > 1e-5 || nrm[2] > 1e-5 || nrm[3] > 1e-5)
                            force_lq = used_lq = 1;
                    }
                }
                else
                    used_lq = 1;
                if (used_lq)
                {
                    fact_lq_backward();
                    alpha = forward_pass(0, 1, 0, 1, 0, nrm);
                    lq_count++;
                }
                if (st && tid == 0) st[13] = used_lq;
                if (st && tid == 0) { st[0] = alpha; st[1] = alpha; }
                int itref1 = 0;
                if (CX.o.pred_corr == 1)
                {
                    double mu_aff = mu_aff_pass(alpha);
                    const double tmp = mu_aff / mu;
                    const double sigma = tmp * tmp * tmp;
                    double sigma_mu = sigma * mu;
                    sigma_mu = sigma_mu > CX.o.tau_min ? sigma_mu : CX.o.tau_min;
                    if (st && tid == 0) { st[2] = mu_aff; st[3] = sigma; }
                    PROF_ADD(5);
                    solve_backward(0, 1, 1, 1, sigma_mu);
                    PROF_ADD(4);
                    const int want_lin = CX.o.itref_corr_max > 0;
                    alpha = forward_pass(0, 1, 0, 1, want_lin, nrm);
                    PROF_ADD(3);
                    if (CX.o.cond_pred_corr == 1)
                    {
                        const double mu_aff0 = mu_aff;
                        mu_aff = mu_aff_pass(alpha);
                        if (mu_aff > 2.0 * mu_aff0)
                        {
                            solve_backward(0, 1, 1, 2, sigma_mu);
                            alpha = forward_pass(0, 1, 0, 1, want_lin, nrm);
                        }
                    }
                    int iter_ref_step = 0;
                    if (CX.o.itref_corr_max > 0)
                    {
                        for (itref1 = 0; itref1 < CX.o.itref_corr_max; itref1++)
                        {
                            PROF_ADD(5);
                            // nrm = norms of the linear residual of the current step (from the fused sweep, or recomputed below)
                            if ((nrm[0] < CX.o.res_g_max || nrm[0] < 1e-3 * res_max[0]) && (nrm[1] < CX.o.res_b_max || nrm[1] < 1e-3 * res_max[1])
                                && (nrm[2] < CX.o.res_d_max || nrm[2] < 1e-3 * res_max[2]) && (nrm[3] < CX.o.res_m_max || nrm[3] < 1e-3 * res_max[3]))
                                break;
                            solve_backward(1, 2, 0, 0, 0.0);
                            forward_pass(1, 2, 0, 0, 0, nrm);
                            iter_ref_step = 1;
                            add_itref();
                            res_pass(1, 1, 0, 1, 0, 0.0, dmy, dmy, dmy, nrm, dmy);
                            PROF_ADD(1);
                        }
                        if (st && tid == 0) { st[16] = nrm[0]; st[17] = nrm[1]; st[18] = nrm[2]; st[19] = nrm[3]; }
                    }
                    if (iter_ref_step) alpha = alpha_pass();
                    if (st && tid == 0) { st[4] = alpha; st[5] = alpha; }
                }
                if (st && tid == 0) st[15] = itref1;
                PROF_ADD(5);
                // move along the step and evaluate the residuals of the new iterate in one sweep
                res_pass(0, 0, -1, 0, 1, alpha, mu, obj, gap, res_max, res_m_tau);
                PROF_ADD(0);
                if (st && tid == 0)
                {
                    st[6] = mu; st[7] = res_max[0]; st[8] = res_max[1]; st[9] = res_max[2]; st[10] = res_max[3];
                    st[11] = gap; st[12] = obj;
                }
            }
            iter = kk;
            if (kk == CX.o.iter_max) status = CUIPM_MAX_ITER;
            else if (alpha <= CX.o.alpha_min) status = CUIPM_MIN_STEP;
            else if (mu != mu) status = CUIPM_NAN_SOL;
            else status = CUIPM_SUCCESS;
        }
#ifdef CUIPM_PROFILE
        if (stat && tid == 0)
            for (int i = 0; i < 16; i++) stat[SM * (size_t) CX.o.stat_max + i] = (double) CX.prof[i];
#endif
        if (tid == 0)
        {
            info->status = status;
            info->iter = iter;
            for (int i = 0; i < 4; i++) info->res_max[i] = res_max[i];
            info->mu = mu;
            info->obj = obj;
            info->dual_gap = gap;
            info->lq_count = lq_count;
            info->reserved = 0;
        }
    }

};

// MINB: resident CTAs per SM the register allocation is bounded for (CUIPM_GENERIC_INSTANCES below)
template <int W, int SNX, int SNU, bool SPILL, int MINB>
__global__ void __launch_bounds__(32 * W, MINB) cuipm_solve_kernel(const LaunchArgs a)
{
    if (threadIdx.x == 0)
    {
        CX.P = a.P;
        CX.SD = a.sd;
        CX.ipool = a.ipool;
        CX.o = a.o;
    }
    Ker<W, SNX, SNU, SPILL> K;
    // second pass behind the throughput kernel: only the QPs it handed back
    const int nq = a.redo_count ? *a.redo_count : a.nbatch;
    for (int i = blockIdx.x; i < nq; i += gridDim.x)
    {
        const int q = a.redo_list ? a.redo_list[i] : i;
        if (threadIdx.x == 0)
        {
            CX.qp = a.qp + (size_t) q * a.P.qp_stride;
            CX.sol = a.sol + (size_t) q * a.P.sol_stride;
            CX.wk = a.work + (size_t) q * a.P.work_stride;
            // by QP, not by CTA: the chunks of a host solve run concurrently, each with its own part of the scratch
            if (SPILL) CX.spx = a.spill + (size_t) q * spill_doubles(a.P);
        }
        K.sync();
        if (a.redo_list && a.o.warm_start >= 2) K.restore_warm_start();
        K.solve(a.info + q, a.stat ? a.stat + (size_t) q * CUIPM_STAT_M * (a.o.stat_max + 1) : nullptr);
        K.sync();
    }
}

template <int W, bool SPILL, int MINB>
__global__ void __launch_bounds__(32 * W, MINB) cuipm_sens_kernel(const LaunchArgs a)
{
    if (threadIdx.x == 0)
    {
        CX.P = a.P;
        CX.SD = a.sd;
        CX.ipool = a.ipool;
        CX.o = a.o;
        CX.mask_constr = 0;      // the reference's sensitivity substitution does not mask
        CX.nc_mask_inv = 0.0;
    }
    Ker<W, 0, 0, SPILL> K;
    for (int q = blockIdx.x; q < a.nbatch; q += gridDim.x)
    {
        if (threadIdx.x == 0)
        {
            CX.qp = a.qp + (size_t) q * a.P.qp_stride;
            CX.wk = a.work + (size_t) q * a.P.work_stride;
            CX.sol = CX.wk + a.P.w_bkp;      // lam, t of the iterate the factorisation belongs to
            if (SPILL) CX.spx = a.spill + (size_t) q * spill_doubles(a.P);
        }
        K.sync();
        K.sens(a.seed + (size_t) q * a.P.sol_stride, a.sens + (size_t) q * a.P.sol_stride, a.adjoint);
        K.sync();
    }
}

}  // namespace

// ---- host side of the generic path (GenericPath, cuipm_device.h) -------------------------------------------------------

// the compiled instances: warps per QP, interior (nx, nu) of the specialised sweeps (0, 0: any shape, these have a sensitivity kernel
// too), global-scratch variant, and the resident CTAs per SM the registers are bounded for: 1 in the global-scratch variant, so that
// it does not spill (its shapes gain nothing from more CTAs per SM, and they run from L2 anyway)
#define CUIPM_GENERIC_INSTANCES(X)                                                              \
    X(1, 21, 3, false, 16) X(1, 8, 3, false, 16) X(1, 4, 1, false, 16) X(1, 12, 4, false, 16) \
    X(1, 0, 0, false, 16) X(2, 0, 0, false, 8) X(4, 0, 0, false, 4)                           \
    X(1, 0, 0, true, 1) X(2, 0, 0, true, 1) X(4, 0, 0, true, 1)

typedef void (*GenericKernel)(LaunchArgs);

struct GenericInstance
{
    int warps, snx, snu, spill;
    GenericKernel solve, sens;   // sens: null for a specialisation
};

template <int W, int SNX, bool SPILL, int MINB>
static GenericKernel sens_kernel() { if constexpr (SNX == 0) return cuipm_sens_kernel<W, SPILL, MINB>; else return nullptr; }

static const GenericInstance kGeneric[] = {
#define X(W_, SNX_, SNU_, SPILL_, MB_) {W_, SNX_, SNU_, SPILL_, cuipm_solve_kernel<W_, SNX_, SNU_, SPILL_, MB_>, sens_kernel<W_, SNX_, SPILL_, MB_>()},
    CUIPM_GENERIC_INSTANCES(X)
#undef X
};

// the instance for `warps` and the variant: the specialisation for interior stages (nx, nu) if there is one, else the one for any shape
static const GenericInstance &instance_for(int warps, int spill, int nx, int nu)
{
    const GenericInstance *any = &kGeneric[0];
    for (const GenericInstance &i : kGeneric)
        if (i.warps == warps && i.spill == spill)
        {
            if (i.snx == nx && i.snu == nu) return i;
            if (i.snx == 0) any = &i;
        }
    return *any;
}

// dynamic shared memory (bytes) of a launch for P: every buffer on chip, or the vector area alone in the global-scratch variant
static size_t smem_bytes(const ProbDesc &P, bool spill) { return sizeof(double) * (size_t) (spill ? P.sm_V : P.sm_total); }

static int launch(GenericKernel k, const LaunchArgs &a, int grid, int warps, void *stream)
{
    const size_t smem = smem_bytes(a.P, a.spill != nullptr);
    const int rc = set_dynamic_smem((const void *) k, smem);
    if (rc != CUIPM_OK) return rc;
    k<<<grid, 32 * warps, smem, (cudaStream_t) stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CUIPM_OK : cuda_error("kernel launch", e);
}

int GenericPath::create(const ProbDesc &P, int max_batch, int device)
{
    warps = P.nmax > 40 ? 4 : 1;   // one warp owns one QP unless the stage block is large
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    // the dynamic shared memory every instance of a variant (0 on chip, 1 global scratch) may request: the choice holds for any "warps"
    size_t lim[2] = {SIZE_MAX, SIZE_MAX};
    for (const GenericInstance &i : kGeneric)
        for (GenericKernel k : {i.solve, i.sens})
        {
            size_t l = 0;
            if (!k) continue;   // the specialisations have no sensitivity kernel
            if (smem_limit((const void *) k, &l) != CUIPM_OK) return CUIPM_ERR_CUDA;
            lim[i.spill] = std::min(lim[i.spill], l);
        }
    // shapes whose buffers do not fit keep the stage-block buffers in a device scratch buffer, the vector area on chip
    spill_needed = spill = smem_bytes(P, false) > lim[0];
    if (spill && smem_bytes(P, true) > lim[1])
    {
        set_error("stage dimensions need more than the " + std::to_string(lim[1]) + " bytes of shared memory a block may have for the "
                  "solver's vectors alone");
        return CUIPM_ERR_TOO_LARGE;
    }
    // a separate buffer, not part of the work record: the getters, the sensitivities and the hand-back path read that layout
    scratch_bytes = sizeof(double) * spill_doubles(P) * (size_t) max_batch;
    if (spill) CK(cudaMalloc(&d_spill, scratch_bytes));
    return CUIPM_OK;
}

int GenericPath::solve(LaunchArgs a, size_t lo, void *stream) const
{
    // by QP, not by CTA: the chunks of a host solve run concurrently, each with its own part of the scratch
    a.spill = spill ? d_spill + spill_doubles(a.P) * lo : nullptr;
    // behind the throughput kernel only a few QPs are left: a small grid (eight CTAs per SM) whose blocks walk the hand-back list
    const int grid = a.redo_list ? std::min(a.nbatch, 8 * sms) : a.nbatch;
    return launch(instance_for(warps, spill, a.P.mid_nx, a.P.mid_nu).solve, a, grid, warps, stream);
}

int GenericPath::sens(LaunchArgs a, void *stream) const
{
    a.spill = spill ? d_spill : nullptr;
    return launch(instance_for(warps, spill, 0, 0).sens, a, a.nbatch, warps, stream);
}

int GenericPath::set_warps(int value)
{
    if (value != 1 && value != 2 && value != 4) { set_error("warps must be 1, 2 or 4"); return CUIPM_ERR_INVALID; }
    warps = value;
    return CUIPM_OK;
}

int GenericPath::set_spill(int value)
{
    if (value != 0 && !d_spill) CK(cudaMalloc(&d_spill, scratch_bytes));
    spill = spill_needed || value != 0;
    return CUIPM_OK;
}

void GenericPath::destroy() { cudaFree(d_spill); }

}  // namespace cuipm
