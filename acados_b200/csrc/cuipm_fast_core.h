// cuipm_fast_core.h -- body of the throughput kernel of the batched OCP-QP interior-point solver.
//
// Mapping: a GROUP of G lanes owns one QP for the whole solve and a warp carries 32/G QPs in lock step, so that every
// serial piece of the algorithm (pivots, reciprocal square roots, the scalar logic of the IPM) is one instruction stream
// for 32/G QPs.  Lane l of a group owns rows l, l+G, l+2G, ... of the stage block; the rank-k updates are register tiles
// of (row slots) x 8 columns fed by one LDS per own row and 128-bit broadcast loads of the other operand; the gradient
// travels as a vector next to the factorisation (a fused right-looking substitution), so the row slots hold matrix rows only.
//
// Data movement: every input of a stage is brought into shared memory by asynchronous copies: the matrices (dynamics block,
// Hessian block, the factor of the next stage) by one bulk copy per QP (TMA, cp.async.bulk), issued by lane 0 of the group
// and completed on the warp's mbarrier; the "images" of the contiguous vector ranges of the three records by 16-byte copies
// (cp.async) by the lanes of the group, completed by a wait on the lane's copies and a warp barrier.  The arithmetic then runs
// on shared memory and registers only, results leave through plain stores.  The matrices come from the
// kernel-side QP record (FastArgs::qpk, written by the repack pass): odd leading dimension (row and column accesses of a
// group both bank-conflict free), Hessian stored as a full symmetric matrix; the factorisation takes the dynamics block
// from the caller's record (even leading dimension n: its broadcast operand is read with 128-bit loads).
//
// Algorithm and work-record layout are those of the generic kernel (cuipm_kernel.cu), which restates HPIPM's
// d_ocp_qp_ipm_solve (external/hpipm/ocp_qp/x_ocp_qp_ipm.c:2684-3120): the sensitivity kernel and the Riccati getters
// read what this kernel leaves behind.  Restrictions (checked on the host, cuipm_plan.h fast_plan): x0 eliminated,
// uniform interior stages, no general constraints.  Cold paths -- the LQ refactorisation, iterative refinement steps, a QP
// without active constraints -- are not here: a QP that needs one is handed back (status CUIPM_FAST_REDO, index appended to
// redo_list) and solved from scratch by the generic kernel.
//
// Scheduling: either a group keeps its QP for the whole solve (run / solve), or -- batches larger than the QPs the device holds
// at once -- for one iteration at a time, the unfinished QPs circulating through rings ordered by their duality measure
// (rr_first / rr_loop below: same arithmetic, bit-identical results, fewer idle slots at the end of the headline batch).  For one QP per
// warp and contraction lengths that are multiples of four the level-3 parts of the factorisation run on the FP64 tensor cores
// (fk_dmma: mma.m8n8k4), otherwise on register tiles.
//
// The file is written against a few warp primitives supplied by the including translation unit (FK_DEV, fk_lane, fk_sync,
// fk_shfl_xor / _i, fk_any, fk_cp16, fk_cp_wait, fk_bulk, fk_mbar_t, fk_mbar_init / _arrive_tx / _wait, fk_fence_async /
// _global, fk_ldg, fk_double2, fk_ld2, fk_dmma, fk_rsqrt, fk_atomic_inc / _add / _cas, fk_ld_volatile, fk_st_volatile,
// fk_threadfence, fk_nanosleep): the CUDA instantiation is cuipm_fast.cu; oracle/fast_emul.cpp instantiates the same body on a
// host emulation of a warp for the CPU test-suite.
#ifndef CUIPM_FAST_CORE_H_
#define CUIPM_FAST_CORE_H_

#include "cuipm_device.h"

// bytes brought into shared memory by one bulk or 16-byte asynchronous copy: a host build can count them (the staged bytes per
// QP-iteration are what the sweeps of this kernel cost on the H100, tests/test_fast_staged_bytes.py)
#ifndef FK_COUNT_STAGED
#define FK_COUNT_STAGED(bytes) do {} while (0)
#endif

#ifndef FK_PROF_T0
#define FK_PROF_T0() do {} while (0)
#define FK_PROF_ADD(slot) do {} while (0)
#define FK_PROF_T2() do {} while (0)
#define FK_PROF_ADD2(slot) do {} while (0)
#endif

// the constraints i softened by slack jj, in increasing order (inv: inverse of idxs_rev, see Ker::Ker)
#define FK_FOR_SLACK(i, jj) \
    _Pragma("unroll 1") for (int i_ = inv[jj], i = i_ >= 0 ? i_ : 0, e_ = i_ >= 0 ? i_ + 1 : (i_ == -2 ? nb : 0); i < e_; i++) \
        if (i_ >= 0 || rev[i] == (jj))

// Unrolling: the short loops of a lane over its elements of a vector (run-time trip counts of 1..4) are kept as loops
// ("unroll 1"): the compiler's unroll-by-four with a remainder chain executes more instructions than the loop it replaces at
// these trip counts, and multiplies the instruction footprint of the sweeps (on the headline shape the SASS shrinks from 574
// to 337 KB).  The loops over the 8-column tiles of a stage are unrolled in full (row slots above a tile vanish at compile
// time); the inner loops of the dot products, TRMM, SYRK and the left-looking update are unrolled by 4, 4, 3 and 2.

namespace cuipm {
namespace fastk {

FK_DEV int evn(int n) { return (n + 1) & ~1; }

// a product rounded before it is used: never contracted into an FMA with the sum it enters (the host build of the emulation
// has no FMA to contract into)
FK_DEV double mul_rn(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// per-QP scalars of the IPM loop
struct QpState
{
    double mu, obj, gap, alpha, res_m_tau;
    double res_max[4];
};

// the residual of the linear system of the iteration just run: inf-norms of its stationarity rows for the affine and the final
// step (from the residual sweep that applies the step), the tests on its other rows (from the forward sweeps), res_max[0] of
// the iterate the steps were computed at
struct LinNrm
{
    double aff_g, fin_g, res0_g;
    bool aff_bdm_large, fin_bdm_small;
};

template <int NX, int NU, int G>
struct Ker
{
    static constexpr int NM = NX + NU;                    // rows of an interior stage block
    static constexpr int QPW = 32 / G;                    // QPs per warp
    static constexpr int LDK = NM | 1;                     // leading dimension of the kernel-side record (odd: row and column accesses
                                                          // of a group in shared memory are both bank-conflict free)
    static constexpr int LDW = ((NM + 1) / 4) * 4 + 2;    // leading dimension of the factor being built (>= NM, = 2 mod 4: 16-byte aligned columns)
    static constexpr int RPM = (NM + G - 1) / G;          // row slots per lane
    static constexpr int NXe = (NX + 1) & ~1, NMe = (NM + 2) & ~1;
    static constexpr int SZA = (LDK * NX + 1) & ~1;       // dynamics block [B'; A'] (-> A Lxx in place in the factorisation, leading dimension n there)
    static constexpr int SZL = LDW * NM;                  // L_{k+1} -> L_k (factorisation); Hessian / L_{k+1} (other sweeps)
    static constexpr int SZU = (NM * NU + 1) & ~1;        // first nu columns of L_k (substitutions), leading dimension n
    static constexpr int MATS = SZA + SZL + SZU;

    // FP64 tensor-core tiles (mma.m8n8k4) for the level-3 parts of the factorisation: one QP per warp only (the fragments span
    // the 32 lanes), contraction lengths that are multiples of four
    template <int NX1>
    struct MMA
    {
#ifdef FK_NO_MMA
        static constexpr bool on = false;
#else
        static constexpr bool on = G == 32 && NX1 % 4 == 0 && NM >= 16 && (NM * NU + 1) / 2 * 2 >= 66 * 8;   // (the fragments are transposed through LU)
#endif
    };
    // stage kinds: 0 = first (nx = 0), 1 = interior, 2 = last (nu = 0)
    template <int KIND>
    struct KD
    {
        static constexpr int nx = KIND == 0 ? 0 : NX, nu = KIND == 2 ? 0 : NU, nx1 = KIND == 2 ? 0 : NX;
    };

    const FastArgs &A;
    double *smem0;             // shared memory of the groups of the warp (after the index maps)
    const int *IDX;            // index maps (idxb, idxs_rev), shared by the groups: entry e = (idxb | idxs_rev | its inverse) at IDX + 4*e*nbe (FastArgs::nmaps entries)
    fk_mbar_t *bar;            // completes the bulk copies of the matrices (the vector images complete through wait_vec)
    int li, gq;                // lane within the group, group within the warp
    double *MA, *ML, *LU, *V;
    const double *qp, *qk;     // this group's QP record: the caller's, the kernel-side one
    double *sol, *wk;
    bool act;                  // this group's QP is being solved: global stores enabled
    unsigned ph;               // phase parity of the barrier; it lives as long as the barrier
    unsigned tx;               // bytes of matrix copies issued and not yet announced to the barrier
    double nc_mask_inv;

    struct View { const double *q; const double *k; double *s; double *w; const int *ip; unsigned kk; };

    FK_DEV Ker(const FastArgs &a, double *smem, fk_mbar_t *b) : A(a)
    {
        const int lane = fk_lane();
        li = lane % G;
        gq = lane / G;
        // the index maps are the same for every QP (and, checked on the host, for every interior stage): one copy per warp
        int *idx = reinterpret_cast<int *>(smem);
        for (int e = 0; e < a.nmaps; e++)
        {
            // maps of entry e: stage 0 / 1 / N when the interior stages share their maps (nmaps = 3), else of stage e
            const int k = a.nmaps == 3 ? (e == 0 ? 0 : (e == 1 ? 1 : a.N)) : e;
            const StageDesc &sdk_ = k == 0 ? a.s0 : (k == a.N ? a.sN : a.s1);
            const int off = sdk_.idx_off + ((k >= 1 && k < a.N) ? (k - 1) * a.is : 0);
            for (int i = lane; i < 2 * sdk_.nb; i += 32) idx[4 * e * a.nbe + i] = a.ipool[off + i];
        }
        fk_sync();
        // inverse of idxs_rev: the constraint softened by slack j (-1: none, -2: several -- the loops then scan idxs_rev)
        for (int e = 0; e < a.nmaps; e++)
        {
            const int k = a.nmaps == 3 ? (e == 0 ? 0 : (e == 1 ? 1 : a.N)) : e;
            const StageDesc &sdk_ = k == 0 ? a.s0 : (k == a.N ? a.sN : a.s1);
            const int *rev_ = idx + 4 * e * a.nbe + sdk_.nb;
            for (int j = lane; j < sdk_.ns; j += 32)
            {
                int f = -1;
                for (int i = 0; i < sdk_.nb; i++)
                    if (rev_[i] == j) f = f == -1 ? i : -2;
                idx[4 * e * a.nbe + 2 * sdk_.nb + j] = f;
            }
        }
        IDX = idx;
        smem += 2 * a.nmaps * a.nbe;
        smem0 = smem;
        bar = b;
        double *S = smem + (size_t) gq * a.gstride;
        MA = S; ML = MA + SZA; LU = ML + SZL; V = LU + SZU;
        qp = nullptr; qk = nullptr; sol = nullptr; wk = nullptr; act = false;
        ph = 0; tx = 0;
        nc_mask_inv = 0.0;
        if (lane == 0) fk_mbar_init(bar, 1);
        fk_fence_async();
        fk_sync();
    }

    // solves QPs first_qp .. first_qp + QPW - 1 (those that exist), one per group
    FK_DEV void run(int first_qp)
    {
        int q = first_qp + gq;
        const bool valid = q < A.nbatch;
        if (!valid) q = A.nbatch - 1;
        solve(q, valid);
        fk_sync();
    }

    template <int KIND>
    FK_DEV const StageDesc &sdk() const { return KIND == 0 ? A.s0 : (KIND == 1 ? A.s1 : A.sN); }
    template <int KIND>
    FK_DEV View view(int k) const
    {
        const unsigned kk = KIND == 1 ? (unsigned) (k - 1) : 0u;
        return View{qp + kk * A.qs, qk + A.kq[KIND] + kk * A.kqs, sol + kk * A.ss, wk + kk * A.ws, A.ipool + (int) kk * A.is, kk};
    }
    FK_DEV const StageDesc &sdr(int k) const { return k == 0 ? A.s0 : (k == A.N ? A.sN : A.s1); }
    FK_DEV View viewr(int k) const
    {
        const unsigned kk = (k >= 1 && k < A.N) ? (unsigned) (k - 1) : 0u;
        const int kind = k == 0 ? 0 : (k == A.N ? 2 : 1);
        return View{qp + kk * A.qs, qk + A.kq[kind] + kk * A.kqs, sol + kk * A.ss, wk + kk * A.ws, A.ipool + (int) kk * A.is, kk};
    }

    // ---- group reductions ---------------------------------------------------------------------------
    FK_DEV double gsum(double v) const
    {
#pragma unroll
        for (int m = G / 2; m > 0; m >>= 1) v += fk_shfl_xor(v, m);
        return v;
    }
    FK_DEV double gmin(double v) const
    {
#pragma unroll
        for (int m = G / 2; m > 0; m >>= 1) v = fmin(v, fk_shfl_xor(v, m));
        return v;
    }
    // max of non-negative values; NaN is propagated (BLASFEO VECNRM_INF semantics, d_aux_lib4.c:4893-4995)
    FK_DEV double gmax_nan(double v, int isnan_) const
    {
#pragma unroll
        for (int m = G / 2; m > 0; m >>= 1)
        {
            v = fmax(v, fk_shfl_xor(v, m));
            isnan_ |= fk_shfl_xor_i(isnan_, m);
        }
        return isnan_ ? NAN : v;
    }
    FK_DEV void st(double *p, double v) const { if (act) *p = v; }
    // two consecutive doubles of shared memory: one 128-bit load where the address is known to be 16-byte aligned
    template <bool ALIGNED>
    FK_DEV fk_double2 ld_pair(const double *p) const
    {
        if (ALIGNED) return fk_ld2(p);
        fk_double2 r;
        r.x = p[0]; r.y = p[1];
        return r;
    }

    // ---- staging ---------------------------------------------------------------------------------------------------------
    // Matrices: one contiguous range of `nd` doubles (even) of this group's record REC (0 kernel-side QP record, 1 solution,
    // 2 work, 3 the caller's QP record) at record offset `off`, to offset `soff` of the group's shared memory, as one bulk
    // asynchronous copy completed on the barrier.  Lane 0 of every group issues the copy of its QP (the compiler serialises the
    // 32/G different operand sets); every lane keeps the byte count of the warp.
    template <int REC>
    FK_DEV void bulk(int soff, size_t off, int nd)
    {
        if (li == 0)
        {
            fk_bulk(smem0 + (size_t) gq * A.gstride + soff, (REC == 0 ? qk : (REC == 1 ? sol : (REC == 2 ? wk : qp))) + off, (unsigned) nd * 8u, bar);
            FK_COUNT_STAGED((unsigned) nd * 8u);
        }
        tx += (unsigned) (QPW * nd) * 8u;
    }
    // Vector images: contiguous range of `nd` doubles (even) of this group's record REC at record offset `off` -> dst (shared
    // memory of the group), as 16-byte asynchronous copies by the lanes of the group (LDGSTS: all groups of the warp copy at
    // once, a handful of instructions per range; a bulk copy per group costs ~25 issue slots of operand marshalling each).
    // Completed by wait_vec().
    template <int REC>
    FK_DEV void vcopy(double *dst, size_t off, int nd)
    {
        const double *src = (REC == 0 ? qk : (REC == 1 ? sol : (REC == 2 ? wk : qp))) + off;
#pragma unroll 1
        for (int e = 2 * li; e < nd; e += 2 * G)
        {
            fk_cp16(dst + e, src + e);
            FK_COUNT_STAGED(16u);
        }
    }
    // all lanes are done with the buffers the next copies overwrite
    FK_DEV void stage_begin() { fk_fence_async(); fk_sync(); }
    // the copies of this stage have been issued: announce their bytes
    FK_DEV void stage_arm()
    {
        if (fk_lane() == 0) fk_mbar_arrive_tx(bar, tx);
        tx = 0;
    }
    // matrix copies announced separately (a second batch inside a stage, requests for the next stage)
    FK_DEV void stage_arm_mat()
    {
        if (fk_lane() == 0) fk_mbar_arrive_tx(bar, tx);
        tx = 0;
    }
    FK_DEV void wait_vec() { FK_PROF_T0(); fk_cp_wait(); fk_sync(); FK_PROF_ADD(5); }      // own copies landed, then everybody's
    FK_DEV void wait_mat() { FK_PROF_T0(); fk_mbar_wait(bar, ph); ph ^= 1u; FK_PROF_ADD(6); }
    FK_DEV int voff(const double *p) const { return (int) (p - (smem0 + (size_t) gq * A.gstride)); }

    // out[i] = 1 / t[i], i < nc, over the lanes of the group; four reciprocals per lane are in flight at once (a double
    // precision division is a dependent chain of ~10 instructions: one after the other they dominated the vector phases)
    FK_DEV void recip_vec(const double *t, double *out, int nc) const
    {
        for (int i0 = li; i0 < nc; i0 += 4 * G)
        {
            double v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = t[i0 + G * u < nc ? i0 + G * u : i0];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = 1.0 / v[u];
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (i0 + G * u < nc) out[i0 + G * u] = v[u];
        }
    }

    // ---- small dense helpers on shared memory -----------------------------------------------------------------------
    // y[i] (+)= sum_j M[i + ld*j] * x[j], j < nc, for the rows i = li, li+G, ... < nr of this lane (row access), x broadcast
    template <int nr, int nc>
    FK_DEV void rows_dot(const double *M, int ld, const double *x, double (&out)[RPM > 0 ? RPM : 1]) const
    {
        constexpr int RP = (nr + G - 1) / G;
#pragma unroll
        for (int m = 0; m < RP; m++) out[m] = 0.0;
        double o2[RPM > 0 ? RPM : 1];
#pragma unroll
        for (int m = 0; m < RP; m++) o2[m] = 0.0;
        int j = 0;
#pragma unroll 4
        for (; j + 1 < nc; j += 2)
        {
            const fk_double2 xx = fk_ld2(x + j);
            const double x0 = xx.x, x1 = xx.y;
#pragma unroll
            for (int m = 0; m < RP; m++)
            {
                const int r = li + G * m;
                const int rr = r < nr ? r : 0;
                out[m] += M[rr + ld * j] * x0;
                o2[m] += M[rr + ld * (j + 1)] * x1;
            }
        }
        if (j < nc)
        {
            const double x0 = x[j];
#pragma unroll
            for (int m = 0; m < RP; m++)
            {
                const int r = li + G * m;
                const int rr = r < nr ? r : 0;
                out[m] += M[rr + ld * j] * x0;
            }
        }
#pragma unroll
        for (int m = 0; m < RP; m++) out[m] += o2[m];
    }
    // z[j] = sum_i M[i + ld*j] * w[i], i < nr, for the columns j = li, li+G, ... < nc of this lane (column access), w broadcast
    template <int nr, int nc>
    FK_DEV void cols_dot(const double *M, int ld, const double *w, double (&out)[RPM > 0 ? RPM : 1]) const
    {
        constexpr int CP = (nc + G - 1) / G;
        double o2[RPM > 0 ? RPM : 1];
#pragma unroll
        for (int m = 0; m < CP; m++) { out[m] = 0.0; o2[m] = 0.0; }
        int i = 0;
#pragma unroll 4
        for (; i + 1 < nr; i += 2)
        {
            const fk_double2 ww = fk_ld2(w + i);
            const double w0 = ww.x, w1 = ww.y;
#pragma unroll
            for (int m = 0; m < CP; m++)
            {
                const int c = li + G * m;
                const int cc = c < nc ? c : 0;
                out[m] += M[i + ld * cc] * w0;
                o2[m] += M[i + 1 + ld * cc] * w1;
            }
        }
        if (i < nr)
        {
            const double w0 = w[i];
#pragma unroll
            for (int m = 0; m < CP; m++)
            {
                const int c = li + G * m;
                const int cc = c < nc ? c : 0;
                out[m] += M[i + ld * cc] * w0;
            }
        }
#pragma unroll
        for (int m = 0; m < CP; m++) out[m] += o2[m];
    }

    // matrices of stage k of the residual sweep: dynamics block and symmetric Hessian of the kernel-side record
    FK_DEV void res_issue_mat(int k)
    {
        const StageDesc &s = sdr(k);
        const unsigned kk = (k >= 1 && k < A.N) ? (unsigned) (k - 1) : 0u;
        const int kind = k == 0 ? 0 : (k == A.N ? 2 : 1);
        if (s.nx1 > 0) bulk<0>(voff(MA), (size_t) A.kq[kind] + (size_t) kk * A.kqs, evn(LDK * s.nx1));
        bulk<0>(voff(ML), (size_t) A.kq[kind] + (size_t) kk * A.kqs + A.kH[kind], evn(LDK * s.n));
        stage_arm_mat();
    }

    // ---------------------------------------------------------------------------------------------
    // residuals of the QP at the iterate (OCP_QP_RES_COMPUTE, x_ocp_qp_res.c:345-531) -> residual set 0, with
    // UPDATE_VAR_QP fused (x_core_qp_ipm_aux.c:472-582: the iterate first moves by alpha_u along the step, with the
    // step shortening and the t/lam clipping) and the affine complementarity right-hand side of the next
    // iteration (res_m = lam*t - tau_min, backup lam*t; BACKUP_RES_M / COMPUTE_TAU_MIN_QP :672-781).
    // Staged: dynamics block, symmetric Hessian, the solution and step records of the stage, ux of the next stage, the
    // vector part of the QP record.
    // ---------------------------------------------------------------------------------------------
    struct ResAcc
    {
        double a_mu, a_obj, a_gap, m0, m1, m2, m3, m4;
        int f0, f1, f2, f3, f4;
        // stationarity rows of the residual of the linear system: inf-norms for the affine (a) and the final (f) step, and
        // dpi of the stage before for the rows of this lane (entry m: row li + G m)
        double ma, mf, pa[RPM > 0 ? RPM : 1], pf[RPM > 0 ? RPM : 1];
        int fa, ff;
    };

    // stationarity rows of the residual of the linear system of one step (dux, dpi_k, dlam: du, dp, dl; dl is masked unless mask_dl;
    // dpi_{k-1}: pm) -> inf-norm mx / NaN flag fl:  ((H dux + rhs_g) - dpi_{k-1} + A dpi_k) + bound multipliers, slack rows
    // Z ds + rhs_g - multipliers; a masked multiplier step is rounded before it is summed (OCP_QP_RES_COMPUTE_LIN).  ML, MA:
    // Hessian and dynamics block; rg: rhs_g (residual set 0 of the iterate the step was computed at).
    template <int KIND>
    FK_DEV void lin_rows(const double *du, const double *dp, const double *dl, bool mask_dl, const double *msk, const double *rg,
                         const double *qZ, const int *idxb, const int *rev, const int *inv, int nb, int ns, const double (&pm)[RPM > 0 ? RPM : 1],
                         double &mx, int &fl) const
    {
        constexpr int nx = KD<KIND>::nx, nu = KD<KIND>::nu, n = nx + nu, nx1 = KD<KIND>::nx1;
        constexpr int RP = (n + G - 1) / G;
        double hx[RPM > 0 ? RPM : 1], ap[RPM > 0 ? RPM : 1];
        rows_dot<n, n>(ML, LDK, du, hx);
        if (nx1 > 0) rows_dot<n, nx1>(MA, LDK, dp, ap);
#pragma unroll
        for (int m = 0; m < RP; m++)
        {
            const int i = li + G * m;
            if (i < n)
            {
                double r = hx[m] + rg[i];
                if (nx > 0 && i >= nu) r -= pm[m];
                if (nx1 > 0) r += ap[m];
                // the bound on row i (at most one: the throughput kernel takes no repeated index in idxb)
                for (int b = 0; b < nb; b++)
                    if (idxb[b] == i)
                        r += (mask_dl ? mul_rn(dl[nb + b], msk[nb + b]) : dl[nb + b]) - (mask_dl ? mul_rn(dl[b], msk[b]) : dl[b]);
                const double a = fabs(r);
                mx = fmax(mx, a);
                fl |= (a != a);
            }
        }
#pragma unroll 1
        for (int j = li; j < 2 * ns; j += G)
        {
            double r = qZ[j] * du[n + j] + rg[n + j] - (mask_dl ? mul_rn(dl[2 * nb + j], msk[2 * nb + j]) : dl[2 * nb + j]);
            const int jj = j < ns ? j : j - ns, offl = j < ns ? 0 : nb;
            FK_FOR_SLACK(i, jj) r -= mask_dl ? mul_rn(dl[offl + i], msk[offl + i]) : dl[offl + i];
            const double a = fabs(r);
            mx = fmax(mx, a);
            fl |= (a != a);
        }
    }

    // lin_a / lin_f: also the stationarity rows of the residual of the linear system for the affine step (kept by the forward
    // sweep in ires) / for the step applied (update only)
    template <int KIND>
    FK_DEV void res_stage(int k, int update, bool lin_a, bool lin_f, double alpha_u, ResAcc &R)
    {
        constexpr int nx = KD<KIND>::nx, nu = KD<KIND>::nu, n = nx + nu, nx1 = KD<KIND>::nx1;
        constexpr int RP = (n + G - 1) / G, CP = (nx1 + G - 1) / G;
        const StageDesc &sd = sdk<KIND>();
        const View v = view<KIND>(k);
        const int nb = sd.nb, ns = sd.ns, nc = sd.nc;
        const int *idxb = IDX + 4 * (A.nmaps == 3 ? KIND : k) * A.nbe, *rev = idxb + nb, *inv = rev + nb;
        const int nu1 = (nx1 > 0 && k + 1 < A.N) ? NU : 0, n1e = (nx1 + nu1 + 1) & ~1;
        // images
        const int solN = (int) (sd.sol.t - sd.sol.ux) + evn(nc), stpN = (int) (sd.step.t - sd.step.ux) + evn(nc);
        const int qvN = (int) ((sd.q_stage + sd.q_stage_bytes / 8u) - sd.q_b);
        double *SOL = V, *STP = SOL + (A.nve + NXe + 2 * A.nce), *SOLN = STP + (A.nve + NXe + 2 * A.nce), *STPN = SOLN + NMe;
        double *QV = STPN + NMe, *tmp0 = QV + (NXe + NMe + 2 * A.nce + 2 * A.ns2e), *tmp1 = tmp0 + A.nbe, *g_ = tmp1 + A.nbe, *pim = g_ + A.nve;
        double *x1 = pim + NXe, *AF = x1 + NXe;
        stage_begin();
        vcopy<1>(SOL, (size_t) v.kk * A.ss + sd.sol.ux, solN);
        if (update) vcopy<2>(STP, (size_t) v.kk * A.ws + sd.step.ux, stpN);
        vcopy<0>(QV, (size_t) A.kq[KIND] + (size_t) v.kk * A.kqs + A.kV[KIND], evn(qvN));
        // rhs_g of the linear system = the residual set 0 this stage overwrites: staged in g_, every row is read (lin_rows) by
        // the lane that later writes it, before it does
        if (lin_a || lin_f) vcopy<2>(g_, (size_t) v.kk * A.ws + sd.res.g, evn(n + 2 * ns));
        if (lin_a) vcopy<2>(AF, (size_t) v.kk * A.ws + sd.ires.g, (int) (sd.ires.d - sd.ires.g) + evn(nc));
        if (nx1 > 0)
        {
            const StageDesc &s1 = sdr(k + 1);
            const View v1 = viewr(k + 1);
            vcopy<1>(SOLN, (size_t) v1.kk * A.ss + s1.sol.ux, n1e);
            if (update) vcopy<2>(STPN, (size_t) v1.kk * A.ws + s1.step.ux, n1e);
        }
        if (KIND == 0) res_issue_mat(k);        // the matrices of every later stage were requested by the stage before it
        wait_vec();
        double *ux = SOL, *pi = SOL + (sd.sol.pi - sd.sol.ux), *lam = SOL + (sd.sol.lam - sd.sol.ux), *t = SOL + (sd.sol.t - sd.sol.ux);
        const double *du = STP, *dp = STP + (sd.step.pi - sd.step.ux), *dl = STP + (sd.step.lam - sd.step.ux), *dtt = STP + (sd.step.t - sd.step.ux);
        const double *qb = QV, *qrq = QV + (sd.q_rq - sd.q_b), *qd = QV + (sd.q_d - sd.q_b), *msk = QV + (sd.q_dmask - sd.q_b);
        const double *qZ = QV + (sd.q_Z - sd.q_b), *qz = QV + (sd.q_z - sd.q_b);
        // ---- move along the step (in the images; the new iterate goes back to the solution record)
        if (update)
        {
            double *gu = v.s + sd.sol.ux, *gp = v.s + sd.sol.pi;
#pragma unroll 1
            for (int i = li; i < n + 2 * ns; i += G)
            {
                const double x = ux[i] + alpha_u * du[i];
                ux[i] = x;
                st(gu + i, x);
            }
#pragma unroll 1
            for (int j = li; j < nx1; j += G)
            {
                const double p = pi[j] + alpha_u * dp[j];
                pi[j] = p;
                st(gp + j, p);
            }
        }
#pragma unroll 1
        for (int j = li; j < nx1; j += G) x1[j] = update ? SOLN[nu1 + j] + alpha_u * STPN[nu1 + j] : SOLN[nu1 + j];
        {
            double *gl = v.s + sd.sol.lam, *gt = v.s + sd.sol.t;
            double *bl = wk + A.w_bkp + (sd.sol.lam + v.kk * A.ss), *bt = wk + A.w_bkp + (sd.sol.t + v.kk * A.ss);
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                double l = lam[i], tt = t[i];
                const double mk = msk[i];
                if (update)
                {
                    // iterate of the factorisation just used (UPDATE_VAR_QP backups, x_core_qp_ipm_aux.c:534-575): the point the
                    // sensitivities are evaluated at
                    st(bl + i, l);
                    st(bt + i, tt);
                    l += alpha_u * dl[i];
                    tt += alpha_u * dtt[i];
                    if (A.o.t_lam_min == 2)
                    {
                        l = l <= A.o.lam_min ? A.o.lam_min : l;
                        tt = tt <= A.o.t_min ? A.o.t_min : tt;
                    }
                    l *= mk;
                    st(gl + i, l);
                    st(gt + i, tt);
                }
                lam[i] = l * mk;
                t[i] = tt;
            }
        }
        fk_sync();
#pragma unroll 1
        for (int i = li; i < nb; i += G) tmp0[i] = lam[nb + i] - lam[i];
        wait_mat();
        fk_sync();
        if (lin_a) lin_rows<KIND>(AF, AF + (sd.ires.b - sd.ires.g), AF + (sd.ires.d - sd.ires.g), false, msk, g_, qZ, idxb, rev, inv, nb, ns, R.pa, R.ma, R.fa);
        if (lin_f) lin_rows<KIND>(du, dp, dl, true, msk, g_, qZ, idxb, rev, inv, nb, ns, R.pf, R.mf, R.ff);
        // ---- rows of res_g (lane = row), res_b (lane = column)
        {
            double hx[RPM > 0 ? RPM : 1], ap[RPM > 0 ? RPM : 1];
            rows_dot<n, n>(ML, LDK, ux, hx);
            if (nx1 > 0) rows_dot<n, nx1>(MA, LDK, pi, ap);
#pragma unroll
            for (int m = 0; m < RP; m++)
            {
                const int i = li + G * m;
                if (i < n)
                {
                    const double gv = qrq[i];
                    double r = hx[m] + 2.0 * gv;
                    R.a_obj += 0.5 * r * ux[i];
                    r -= gv;
                    R.a_gap += r * ux[i];
                    if (nx > 0 && i >= nu) r -= pim[i - nu];
                    if (nx1 > 0) r += ap[m];
                    g_[i] = r;
                }
            }
            if (nx1 > 0)
            {
                double au[RPM > 0 ? RPM : 1];
                cols_dot<n, nx1>(MA, LDK, ux, au);
                double *ob = v.w + sd.res.b;
#pragma unroll
                for (int m = 0; m < CP; m++)
                {
                    const int j = li + G * m;
                    if (j < nx1)
                    {
                        const double bv = qb[j];
                        const double r = bv - x1[j] + au[m];
                        st(ob + j, r);
                        const double a = fabs(r);
                        R.m1 = fmax(R.m1, a);
                        R.f1 |= (a != a);
                        R.a_gap -= bv * pi[j];
                    }
                }
            }
        }
        // last use of the two matrices: request those of the next stage, they arrive during the vector work below
        if (KIND != 2)
        {
            stage_begin();
            res_issue_mat(k + 1);
        }
        else
            fk_sync();
        // ---- box scatter, slack rows
#pragma unroll 1
        for (int i = li; i < nb; i += G)
        {
            const int ix = idxb[i];
            tmp1[i] = ux[ix];
            g_[ix] += tmp0[i];
        }
        if (ns > 0)
        {
#pragma unroll 1
            for (int j = li; j < 2 * ns; j += G)
            {
                const double sj = ux[n + j], zz = qz[j];
                double r = qZ[j] * sj + 2.0 * zz;
                R.a_obj += 0.5 * r * sj;
                r -= zz;
                R.a_gap += r * sj;
                r -= lam[2 * nb + j];
                const int jj = j < ns ? j : j - ns, offl = j < ns ? 0 : nb;
                FK_FOR_SLACK(i, jj) r -= lam[offl + i];
                g_[n + j] = r;
            }
        }
        fk_sync();
        // ---- res_d, res_m
        {
            double *od = v.w + sd.res.d, *om = v.w + sd.res.m, *obk = v.w + sd.w_rmb;
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                const double dv = qd[i];
                double r;
                if (i < 2 * nb)
                {
                    const int up = i >= nb, ii = up ? i - nb : i;
                    const double x = tmp1[ii];
                    r = t[i] + dv + (up ? x : -x);
                    if (ns > 0 && rev[ii] >= 0) r -= ux[n + (up ? ns : 0) + rev[ii]];
                }
                else
                    r = t[i] - ux[n + (i - 2 * nb)] + dv;
                r *= msk[i];
                st(od + i, r);
                double a = fabs(r);
                R.m2 = fmax(R.m2, a);
                R.f2 |= (a != a);
                R.a_gap -= dv * lam[i];
                double mm = lam[i] * t[i] - A.o.m_relax;        // qp->m = m_relax everywhere (ocp_qp_hpipm.c:338-342)
                mm *= msk[i];
                R.a_mu += fabs(mm);
                st(obk + i, mm);
                double ma = mm - A.o.tau_min;
                ma *= msk[i];
                st(om + i, ma);                                  // affine rhs of the next iteration
                const double a4 = fabs(mm - A.o.tau_min * msk[i]);
                R.m4 = fmax(R.m4, a4);
                R.f4 |= (a4 != a4);
                a = fabs(mm);
                R.m3 = fmax(R.m3, a);
                R.f3 |= (a != a);
            }
            double *og = v.w + sd.res.g;
#pragma unroll 1
            for (int i = li; i < n + 2 * ns; i += G)
            {
                const double r = g_[i];
                st(og + i, r);
                const double a = fabs(r);
                R.m0 = fmax(R.m0, a);
                R.f0 |= (a != a);
            }
        }
#pragma unroll 1
        for (int j = li; j < nx1; j += G) pim[j] = pi[j];      // pi_k is "pi_{k-1}" of the next stage
        if (nx1 > 0 && (lin_a || lin_f))
        {
            // the entries of dpi_k the rows of this lane take in the next stage (row i: i - nu of that stage)
            const int nun = k + 1 < A.N ? NU : 0;
            const double *dpa = AF + (sd.ires.b - sd.ires.g);
#pragma unroll
            for (int m = 0; m < RPM; m++)
            {
                const int j = li + G * m - nun;
                const bool in = j >= 0 && j < nx1;
                R.pa[m] = in && lin_a ? dpa[j] : 0.0;
                R.pf[m] = in && lin_f ? dp[j] : 0.0;
            }
        }
    }

    // update: move along the step first; then also the stationarity norms of the residual of the linear system of the iteration
    // that computed the step, into L.aff_g / L.fin_g (lin_check tests them)
    FK_DEV void res_pass(int update, double alpha_u, QpState &Q, LinNrm &L)
    {
        fk_fence_async_global();        // the records this sweep reads with bulk copies were written with plain stores by the sweeps before

        const bool lin_a = update && A.o.lq_fact == 1, lin_f = update && A.o.pred_corr == 1 && A.o.itref_corr_max > 0;
        ResAcc R;
        R.a_mu = R.a_obj = R.a_gap = R.m0 = R.m1 = R.m2 = R.m3 = R.m4 = 0.0;
        R.f0 = R.f1 = R.f2 = R.f3 = R.f4 = 0;
        R.ma = R.mf = 0.0;
        R.fa = R.ff = 0;
#pragma unroll
        for (int m = 0; m < (RPM > 0 ? RPM : 1); m++) R.pa[m] = R.pf[m] = 0.0;
        if (update && alpha_u < 1.0) alpha_u = alpha_u * ((1.0 - alpha_u) * 0.99 + alpha_u * 0.9999999);
        res_stage<0>(0, update, lin_a, lin_f, alpha_u, R);
        for (int k = 1; k < A.N; k++) res_stage<1>(k, update, lin_a, lin_f, alpha_u, R);
        res_stage<2>(A.N, update, lin_a, lin_f, alpha_u, R);
        if (lin_a) L.aff_g = gmax_nan(R.ma, R.fa);
        if (lin_f) L.fin_g = gmax_nan(R.mf, R.ff);
        Q.res_max[0] = gmax_nan(R.m0, R.f0);
        Q.res_max[1] = gmax_nan(R.m1, R.f1);
        Q.res_max[2] = gmax_nan(R.m2, R.f2);
        Q.res_max[3] = gmax_nan(R.m3, R.f3);
        Q.mu = gsum(R.a_mu) * nc_mask_inv;
        Q.obj = gsum(R.a_obj);
        Q.gap = gsum(R.a_gap);
        Q.res_m_tau = gmax_nan(R.m4, R.f4);
    }

    // ---------------------------------------------------------------------------------------------
    // slack elimination (x_ocp_qp_kkt.c:220-335, 431-520): tmp0/tmp1 = effective Gamma / gamma of the
    // softened constraints; ds = slack part of the step rhs; Zi = inverse of the slack Hessian.
    // ---------------------------------------------------------------------------------------------
    FK_DEV void cond_slacks(int nb, int ns, const int *rev, const int *inv, const double *Z, int fact, const double *Gam, const double *gam,
                            const double *rgs, double *Zi, double *ds, double *tmp0, double *tmp1) const
    {
#pragma unroll 1
        for (int j = li; j < 2 * ns; j += G)
        {
            const int jj = j < ns ? j : j - ns, offc = j < ns ? 0 : nb;
            double zi = 0.0, d = rgs[j] + gam[2 * nb + j];
            if (fact) zi = Z[j] + A.o.reg_prim + Gam[2 * nb + j];
            FK_FOR_SLACK(i, jj)
            {
                if (fact) zi += Gam[offc + i];
                d += gam[offc + i];
            }
            if (fact) Zi[j] = 1.0 / zi;
            ds[j] = d;
        }
        fk_sync();
#pragma unroll 1
        for (int i = li; i < nb; i += G)
        {
            const int j = rev[i];
            double t0l, t0u, t1l, t1u;
            if (j != -1)
            {
                t0l = Gam[i] - Gam[i] * Zi[j] * Gam[i];
                t0u = Gam[nb + i] - Gam[nb + i] * Zi[ns + j] * Gam[nb + i];
                t1l = gam[i] - Gam[i] * Zi[j] * ds[j];
                t1u = gam[nb + i] - Gam[nb + i] * Zi[ns + j] * ds[ns + j];
            }
            else
            {
                t0l = Gam[i]; t0u = Gam[nb + i]; t1l = gam[i]; t1u = gam[nb + i];
            }
            if (fact) tmp0[i] = t0l + t0u;
            tmp1[i] = t1l - t1u;
        }
    }

    // ---------------------------------------------------------------------------------------------
    // W-column panel (W <= 8: one tile) of the left-looking Cholesky: x[m][0..W-1] hold the raw (updated) entries of columns
    // j0..j0+W-1 of this lane's rows, hh[m] the gradient entries of those rows.  The W x W diagonal block and its W
    // gradient entries are published through DD8 (8 x 8 column-major + 8), the block is factorised redundantly by every
    // lane (pivot rule blasfeo_ref/x_lapack_ref.c:84-91: a non-positive pivot gives a zero column) -- one chain of W
    // reciprocal square roots per tile for all QPs of the warp --, every row then runs the same substitution against it (for
    // a row of the block itself that reproduces the factor's row, the entries right of the diagonal are zero); the gradient
    // takes W steps of the forward substitution l = L^{-1} h.
    // Results: ML (final columns of L), the work record (lower part), lvec / lrow (gradient), Linv.
    // ---------------------------------------------------------------------------------------------
    template <int n, int nu, int RP, int W>
    FK_DEV void panel8(int j0, int m0, double (&x)[RPM > 0 ? RPM : 1][8], double (&hh)[RPM > 0 ? RPM : 1], double *DD8, double *Lg, double *Lxg,
                       double *lrow, double *lvec, double *Linv)
    {
#pragma unroll
        for (int m = 0; m < RP; m++)
        {
            if (m < m0) continue;
            const int rr = li + G * m - j0;
            if (rr >= 0 && rr < W)
            {
#pragma unroll
                for (int q = 0; q < W; q++) DD8[rr + 8 * q] = x[m][q];
                DD8[64 + rr] = hh[m];
            }
        }
        fk_sync();
        double d[8][8], iv[8], g[8];       // d[i][j], i >= j: block entries, overwritten by the factor
#pragma unroll
        for (int j = 0; j < W; j++)
        {
#pragma unroll
            for (int i = j; i < W; i++) d[i][j] = DD8[i + 8 * j];
            g[j] = DD8[64 + j];
        }
#pragma unroll
        for (int j = 0; j < W; j++)
        {
            double dj = d[j][j];
#pragma unroll
            for (int c = 0; c < j; c++) dj -= d[j][c] * d[j][c];
            iv[j] = dj > 0.0 ? fk_rsqrt(dj) : 0.0;
            double gj = g[j];
#pragma unroll
            for (int c = 0; c < j; c++) gj -= d[j][c] * g[c];
            g[j] = gj * iv[j];
#pragma unroll
            for (int i = j + 1; i < W; i++)
            {
                double v = d[i][j];
#pragma unroll
                for (int c = 0; c < j; c++) v -= d[i][c] * d[j][c];
                d[i][j] = v * iv[j];
            }
        }
#pragma unroll
        for (int m = 0; m < RP; m++)
        {
            if (m < m0) continue;
            const int r = li + G * m, rr = r - j0;     // position relative to the panel: rows 0..W-1 form the diagonal block
            double xs[8];
#pragma unroll
            for (int q = 0; q < W; q++)
            {
                double v = x[m][q];
#pragma unroll
                for (int c = 0; c < q; c++) v -= xs[c] * d[q][c];
                v *= iv[q];
                xs[q] = rr >= q ? v : 0.0;              // a row of the block ends at its diagonal entry
            }
            if (rr >= W)
            {
                double hv = hh[m];
#pragma unroll
                for (int q = 0; q < W; q++) hv -= xs[q] * g[q];
                hh[m] = hv;
            }
            if (rr >= 0 && r < n)
            {
                double *mr = ML + r + LDW * j0;
#pragma unroll
                for (int q = 0; q < W; q++) mr[q * LDW] = xs[q];
                if (act)
                {
                    double *gr = Lg + r + n * j0;
#pragma unroll
                    for (int q = 0; q < W; q++)
                        if (rr >= q) gr[q * n] = xs[q];
                    // state block once more with an odd leading dimension, for the forward sweeps (zeros right of the diagonal
                    // inside the block; what lies above the block is never written and stays zero)
                    constexpr int nxk = n - nu, ldx = nxk | 1;
                    if (nxk > 0 && r >= nu)
                    {
#pragma unroll
                        for (int q = 0; q < W; q++)
                            if (j0 + q >= nu) Lxg[(r - nu) + ldx * (j0 + q - nu)] = xs[q];
                    }
                }
            }
        }
        if (li == 0)
        {
#pragma unroll
            for (int q = 0; q < W; q++) { Linv[j0 + q] = iv[q]; lvec[j0 + q] = g[q]; }
            if (act)
#pragma unroll
                for (int q = 0; q < W; q++) lrow[j0 + q] = g[q];
        }
        fk_sync();
    }

    // inputs of stage k of the factorisation sweep (any stage: the offsets come from its descriptor at run time)
    FK_DEV void fact_issue_vec(int k)
    {
        const StageDesc &s = sdr(k);
        const unsigned kk = (k >= 1 && k < A.N) ? (unsigned) (k - 1) : 0u;
        const int kind = k == 0 ? 0 : (k == A.N ? 2 : 1);
        const int oRES = voff(V), oLT = oRES + (A.nve + NXe + 2 * A.nce), oZQ = oLT + 2 * A.nce;
        vcopy<2>((smem0 + (size_t) gq * A.gstride + oRES), (size_t) kk * A.ws + s.res.g, (int) (s.res.m - s.res.g) + evn(s.nc));
        vcopy<1>((smem0 + (size_t) gq * A.gstride + oLT), (size_t) kk * A.ss + s.sol.lam, (int) (s.sol.t - s.sol.lam) + evn(s.nc));
        if (s.ns > 0) vcopy<0>((smem0 + (size_t) gq * A.gstride + oZQ), (size_t) A.kq[kind] + (size_t) kk * A.kqs + A.kV[kind] + (s.q_Z - s.q_b), evn(2 * s.ns));
    }
    FK_DEV void fact_issue_mat(int k)
    {
        const StageDesc &s = sdr(k);
        const unsigned kk = (k >= 1 && k < A.N) ? (unsigned) (k - 1) : 0u;
        if (s.nx1 > 0) bulk<3>(voff(MA), (size_t) kk * A.qs + s.q_BAt, evn(s.n * s.nx1));      // the caller's block: leading dimension n
        stage_arm_mat();
    }

    // ---------------------------------------------------------------------------------------------
    // one stage of the backward Riccati sweep with factorisation (OCP_QP_FACT_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:880-966),
    // right-hand side = residual set 0.  ML holds L_{k+1} on entry and L_k on exit, lprev the x part of the gradient
    // vector of stage k+1.
    //   A -> MA (bulk copy), in place  AL = A * Lxx_{k+1}                               (TRMM_RLNN)
    //   gradient:  alb = Lxx' b + l_{k+1,x},  h = g + AL alb                             (the (n+1)-th row of the reference's block)
    //   8-column tiles:  acc = H + diag + AL AL' - (columns already factorised)         (SYRK + left-looking POTRF)
    // ---------------------------------------------------------------------------------------------
    template <int KIND>
    FK_DEV void fact_stage(int k)
    {
        constexpr int nx = KD<KIND>::nx, nu = KD<KIND>::nu, n = nx + nu, nx1 = KD<KIND>::nx1;
        constexpr int RP = (n + G - 1) / G, CP = (nx1 + G - 1) / G;
        FK_PROF_T2();
        const StageDesc &sd = sdk<KIND>();
        const View v = view<KIND>(k);
        const int nb = sd.nb, ns = sd.ns, nc = sd.nc;
        const int *idxb = IDX + 4 * (A.nmaps == 3 ? KIND : k) * A.nbe, *rev = idxb + nb, *inv = rev + nb;
        const int nu1 = (nx1 > 0 && k + 1 < A.N) ? NU : 0;
        double *RES = V, *LT = RES + (A.nve + NXe + 2 * A.nce), *ZQ = LT + 2 * A.nce, *Gam = ZQ + A.ns2e, *gam = Gam + A.nce;
        double *tmp0 = gam + A.nce, *tmp1 = tmp0 + A.nbe, *Zi = tmp1 + A.nbe, *ds = Zi + A.ns2e, *ddx = ds + A.ns2e;
        // Gam .. ds are dead once the gradient and the diagonal additions are formed: the diagonal blocks of the tiles are
        // published there (72 doubles; ddx pads the block where the constraint arrays are shorter)
        const int ddpad = 72 - (2 * A.nce + 2 * A.nbe + 2 * A.ns2e) > 0 ? 72 - (2 * A.nce + 2 * A.nbe + 2 * A.ns2e) : 0;
        double *DD8 = Gam, *dadd = ddx + ddpad, *Linv = dadd + NMe, *alb = Linv + NMe, *lvec = alb + NXe, *lprev = lvec + NMe;
        // the inputs of stage N are fetched here; those of every other stage were requested by the stage before it in the sweep
        // (vector images after its prologue, dynamics block after its last use of MA)
        if (KIND == 2)
        {
            stage_begin();
            fact_issue_vec(k);
            fact_issue_mat(k);
        }
        wait_vec();
        double *rowv = RES;
        const double *rb = RES + (sd.res.b - sd.res.g), *rd = RES + (sd.res.d - sd.res.g), *rm = RES + (sd.res.m - sd.res.g);
        const double *gl = LT, *gt = LT + (sd.sol.t - sd.sol.lam);
        {
            // Gamma, gamma (COMPUTE_GAMMA_GAMMA_QP, x_core_qp_ipm_aux.c:38-86)
            const double t_min_inv = A.o.t_min > 0 ? 1.0 / A.o.t_min : 1e30;
            recip_vec(gt, Gam, nc);                  // same lane, same index below: no barrier needed
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                const double l = gl[i], tt = gt[i], ti = Gam[i];
                if (A.o.t_lam_min == 1)
                    Gam[i] = (tt < A.o.t_min ? t_min_inv : ti) * (l < A.o.lam_min ? A.o.lam_min : l);
                else
                    Gam[i] = ti * l;
                gam[i] = ti * (rm[i] - l * rd[i]);
            }
#pragma unroll 1
            for (int i = li; i < n; i += G) dadd[i] = A.o.reg_prim;
        }
        fk_sync();
        if (ns > 0)
        {
            cond_slacks(nb, ns, rev, inv, ZQ, 1, Gam, gam, rowv + n, Zi, ds, tmp0, tmp1);
            fk_sync();
#pragma unroll 1
            for (int j = li; j < 2 * ns; j += G)
            {
                st(v.w + sd.w_Zsi + j, Zi[j]);
                st(v.w + sd.step.ux + n + j, ds[j]);
            }
        }
        else
        {
#pragma unroll 1
            for (int i = li; i < nb; i += G)
            {
                tmp0[i] = Gam[i] + Gam[nb + i];
                tmp1[i] = gam[i] - gam[nb + i];
            }
            fk_sync();
        }
#pragma unroll 1
        for (int i = li; i < nb; i += G)
        {
            const int ix = idxb[i];
            dadd[ix] += tmp0[i];
            rowv[ix] += tmp1[i];
        }
        wait_mat();
        fk_sync();
        FK_PROF_ADD2(10);      /* prologue + waits */
        double hh[RPM > 0 ? RPM : 1];
#pragma unroll
        for (int m = 0; m < RP; m++) hh[m] = rowv[(li + G * m) < n ? li + G * m : 0];
        if (nx1 > 0)
        {
            const double *Lx = ML + nu1 + LDW * nu1;                 // Lxx(c, j) = Lx[c + LDW*j], lower triangular
            // ---- gradient: alb = Lxx' b (lane = column), Pb = Lxx alb (lane = row), then alb += l_{k+1,x}
            // (ML is zero above the diagonal for the whole sweep: fact_backward clears it, the panels write zeros there)
            {
                double tt_[RPM > 0 ? RPM : 1];
                cols_dot<nx1, nx1>(Lx, LDW, rb, tt_);
#pragma unroll
                for (int m = 0; m < CP; m++)
                    if (li + G * m < nx1) alb[li + G * m] = tt_[m];
                fk_sync();
                rows_dot<nx1, nx1>(Lx, LDW, alb, tt_);
                double *Pb = v.w + sd.w_Pb;
#pragma unroll
                for (int m = 0; m < CP; m++)
                    if (li + G * m < nx1) st(Pb + li + G * m, tt_[m]);
            }
            fk_sync();
#pragma unroll 1
            for (int j = li; j < nx1; j += G) alb[j] += lprev[j];
        }
        // the vector images are dead from here on (gradient and diagonal additions are in registers / in their own arrays):
        // request those of the next stage of the sweep, they arrive during the matrix work below
        if (k > 0)
        {
            stage_begin();
            fact_issue_vec(k - 1);
        }
        if (nx1 > 0)
        {
            const double *Lx = ML + nu1 + LDW * nu1;
            FK_PROF_ADD2(11);      /* gradient */
            // ---- in place: AL = A * Lxx
            if (MMA<nx1>::on)
            {
                // one QP per warp, FP64 tensor cores: 8 x 8 tiles of AL as sums of (8 x 4)(4 x 8) products, all row blocks of a
                // column tile kept in fragments (Lxx is lower triangular and ML reads as zero above its diagonal: k starts at the tile)
                const int l4 = fk_lane() & 3, r8 = fk_lane() >> 2;
                constexpr int NRB = (n + 7) / 8;
#pragma unroll 1
                for (int jt = 0; jt < nx1; jt += 8)
                {
                    double C[NRB][2];
#pragma unroll
                    for (int i = 0; i < NRB; i++) C[i][0] = C[i][1] = 0.0;
                    const double *bp = Lx + l4 + LDW * (jt + r8), *ap = MA + r8 + n * l4;
#pragma unroll 2
                    for (int k0 = jt; k0 < nx1; k0 += 4)
                    {
                        const double b = bp[k0];
#pragma unroll
                        for (int i = 0; i < NRB; i++) fk_dmma(C[i][0], C[i][1], ap[8 * i + n * k0], b);
                    }
#pragma unroll
                    for (int i = 0; i < NRB; i++)
                        if (8 * i + r8 < n)
                        {
                            MA[8 * i + r8 + n * (jt + 2 * l4)] = C[i][0];
                            MA[8 * i + r8 + n * (jt + 2 * l4 + 1)] = C[i][1];
                        }
                }
            }
            else
#pragma unroll
            for (int jt = 0; jt < nx1; jt += 8)
            {
                const int w = nx1 - jt < 8 ? nx1 - jt : 8;
                double acc[RPM > 0 ? RPM : 1][8];
#pragma unroll
                for (int m = 0; m < RP; m++)
#pragma unroll
                    for (int q = 0; q < 8; q++) acc[m][q] = 0.0;
                // triangular head: column jt+q of Lxx starts at row jt+q
#pragma unroll
                for (int h = 0; h < 8; h++)
                {
                    if (h >= w) continue;
                    const int c = jt + h;
                    double a[RPM > 0 ? RPM : 1];
#pragma unroll
                    for (int m = 0; m < RP; m++) a[m] = MA[(li + G * m < n ? li + G * m : 0) + n * c];
#pragma unroll
                    for (int q = 0; q <= h; q++)
                    {
                        const double l = Lx[c + LDW * (jt + q)];
#pragma unroll
                        for (int m = 0; m < RP; m++) acc[m][q] += a[m] * l;
                    }
                }
#pragma unroll 4
                for (int c = jt + 8; c < nx1; c++)
                {
                    double a[RPM > 0 ? RPM : 1];
#pragma unroll
                    for (int m = 0; m < RP; m++) a[m] = MA[(li + G * m < n ? li + G * m : 0) + n * c];
#pragma unroll
                    for (int q = 0; q < 8; q++)
                    {
                        const double l = Lx[c + LDW * (jt + q)];
#pragma unroll
                        for (int m = 0; m < RP; m++) acc[m][q] += a[m] * l;
                    }
                }
#pragma unroll
                for (int m = 0; m < RP; m++)
                {
                    const int r = li + G * m;
                    if (r < n)
                    {
#pragma unroll
                        for (int q = 0; q < 8; q++)
                            if (q < w) MA[r + n * (jt + q)] = acc[m][q];
                    }
                }
            }
            fk_sync();
        }
        FK_PROF_ADD2(12);      /* TRMM */
        // ---- column tiles: SYRK + left-looking Cholesky, rows r >= jt; gradient h = g + AL alb in the first tile
        const double *Hk = v.k + A.kH[KIND];
        double *Lg = v.w + sd.w_L, *lrow = v.w + sd.w_lrow;
#pragma unroll
        for (int jt = 0; jt < n; jt += 8)
        {
            const int w = n - jt < 8 ? n - jt : 8;
            const int m0 = jt / G;                      // first row slot that reaches into the tile
            double acc[RPM > 0 ? RPM : 1][8], h[RPM > 0 ? RPM : 1][8];
            // H (lower; issued first so that the loads overlap the products)
#pragma unroll
            for (int m = 0; m < RP; m++)
            {
                if (m < m0) continue;
                const int r = li + G * m;
#pragma unroll
                for (int q = 0; q < 8; q++)
                {
                    acc[m][q] = 0.0;
                    h[m][q] = (q < w && r < n && r >= jt + q) ? fk_ldg(Hk + r + LDK * (jt + q)) : 0.0;
                }
            }
            if (MMA<nx1>::on)
            {
                // the rows jt .. n-1 of the tile's columns in blocks of eight, as fragments of the tensor-core product: Gram product
                // of the rows of AL, minus the columns of L already factorised; the fragments go through shared memory (TT, the
                // buffer of the substitution sweeps' panel) into the row slots the panel factorisation works on
                const int l4 = fk_lane() & 3, r8 = fk_lane() >> 2;
                constexpr int NRBmax = (n + 7) / 8, LDT = 66;
                const int nrb = (n - jt + 7) / 8;
                double C[NRBmax][2];
#pragma unroll
                for (int i = 0; i < NRBmax; i++) C[i][0] = C[i][1] = 0.0;
                if (nx1 > 0)
                {
                    const double *ap = MA + jt + r8 + n * l4;
#pragma unroll 2
                    for (int k0 = 0; k0 < nx1; k0 += 4)
                    {
                        const double b = ap[n * k0];
#pragma unroll
                        for (int i = 0; i < NRBmax; i++)
                            if (i < nrb) fk_dmma(C[i][0], C[i][1], i == 0 ? b : ap[8 * i + n * k0], b);
                    }
                    if (jt == 0)
                    {
#pragma unroll 4
                        for (int c = 0; c < nx1; c++)
                        {
                            const double ab = alb[c];
#pragma unroll
                            for (int m = 0; m < RP; m++) hh[m] += MA[(li + G * m < n ? li + G * m : 0) + n * c] * ab;
                        }
                    }
                }
                if (jt + 8 >= n && k > 0)
                {   // last use of the dynamics block: request the one of the next stage of the sweep
                    stage_begin();
                    fact_issue_mat(k - 1);
                }
                {
                    const double *lp = ML + jt + r8 + LDW * l4;
#pragma unroll 2
                    for (int k0 = 0; k0 < jt; k0 += 4)
                    {
                        const double b = lp[LDW * k0];
#pragma unroll
                        for (int i = 0; i < NRBmax; i++)
                            if (i < nrb) fk_dmma(C[i][0], C[i][1], -(i == 0 ? b : lp[8 * i + LDW * k0]), b);
                    }
                }
                double *TT = LU;
#pragma unroll
                for (int i = 0; i < NRBmax; i++)
                    if (i < nrb)
                    {
                        TT[8 * i + r8 + LDT * (2 * l4)] = C[i][0];
                        TT[8 * i + r8 + LDT * (2 * l4 + 1)] = C[i][1];
                    }
                fk_sync();
#pragma unroll
                for (int m = 0; m < RP; m++)
                    if (m >= m0)
                    {
                        const int r = li + G * m;
                        const int rr = (r >= jt && r < n) ? r - jt : 0;
#pragma unroll
                        for (int q = 0; q < 8; q++) acc[m][q] = TT[rr + LDT * q];
                    }
            }
            else {
            if (nx1 > 0)
            {
#pragma unroll 3
                for (int c = 0; c < nx1; c++)
                {
                    double a[RPM > 0 ? RPM : 1], b[8];
#pragma unroll
                    for (int m = 0; m < RP; m++) a[m] = m >= m0 ? MA[(li + G * m < n ? li + G * m : 0) + n * c] : 0.0;
#pragma unroll
                    for (int q = 0; q < 8; q += 2)
                    {
                        const fk_double2 t2 = ld_pair<n % 2 == 0>(MA + jt + q + n * c);       // rows jt+q, jt+q+1 of column c
                        b[q] = t2.x; b[q + 1] = t2.y;
                    }
#pragma unroll
                    for (int m = 0; m < RP; m++)
                        if (m >= m0)
#pragma unroll
                            for (int q = 0; q < 8; q++) acc[m][q] += a[m] * b[q];
                    if (jt == 0)
                    {
                        const double ab = alb[c];
#pragma unroll
                        for (int m = 0; m < RP; m++) hh[m] += a[m] * ab;
                    }
                }
            }
            if (jt + 8 >= n && k > 0)
            {   // last use of the dynamics block: request the one of the next stage of the sweep
                stage_begin();
                fact_issue_mat(k - 1);
            }
#pragma unroll 2
            for (int c = 0; c < jt; c++)
            {
                double a[RPM > 0 ? RPM : 1], b[8];
#pragma unroll
                for (int m = 0; m < RP; m++) a[m] = m >= m0 ? ML[(li + G * m < n ? li + G * m : 0) + LDW * c] : 0.0;
#pragma unroll
                for (int q = 0; q < 8; q += 2)
                {
                    const fk_double2 t2 = fk_ld2(ML + jt + q + LDW * c);
                    b[q] = t2.x; b[q + 1] = t2.y;
                }
#pragma unroll
                for (int m = 0; m < RP; m++)
                    if (m >= m0)
#pragma unroll
                        for (int q = 0; q < 8; q++) acc[m][q] -= a[m] * b[q];
            }
            }
#pragma unroll
            for (int m = 0; m < RP; m++)
                if (m >= m0)
                {
                    const int r = li + G * m;
#pragma unroll
                    for (int q = 0; q < 8; q++)
                    {
                        acc[m][q] += h[m][q];
                        if (q < w && r == jt + q) acc[m][q] += dadd[r < n ? r : 0];
                    }
                }
            FK_PROF_ADD2(13);      /* SYRK + update + H */
            // ---- the tile's columns: diagonal block, rows below, gradient
            // (a stage has full tiles and at most one narrower tile, its last)
            constexpr int WL = n % 8 ? n % 8 : 8;
            if (w >= 8) panel8<n, nu, RP, 8>(jt, m0, acc, hh, DD8, Lg, v.w + sd.w_Lxx, lrow, lvec, Linv);
            else panel8<n, nu, RP, WL>(jt, m0, acc, hh, DD8, Lg, v.w + sd.w_Lxx, lrow, lvec, Linv);
            FK_PROF_ADD2(14);      /* panels */
        }
        {
            double *li_ = v.w + sd.w_Linv;
#pragma unroll 1
            for (int j = li; j < n; j += G) st(li_ + j, Linv[j]);
#pragma unroll 1
            for (int j = li; j < nx; j += G) lprev[j] = lvec[nu + j];
        }
    }

    FK_DEV void fact_backward()
    {
        // the factor is built in ML; its strict upper triangle must read as zero (the triangular products of the sweep run
        // over full rows / columns), and the other sweeps leave the Hessian there
        fk_sync();
#pragma unroll 1
        for (int e = li; e < SZL; e += G) ML[e] = 0.0;
        fk_fence_async_global();        // the records this sweep reads with bulk copies were written with plain stores by the sweeps before

        fact_stage<2>(A.N);
        for (int k = A.N - 1; k >= 1; k--) fact_stage<1>(k);
        fact_stage<0>(0);
    }

    // ---------------------------------------------------------------------------------------------
    // one stage of the backward substitution with the existing factorisation (OCP_QP_SOLVE_KKT_STEP, x_ocp_qp_kkt.c:
    // 1582-1680), right-hand side = residual set 0, result (backward quantities) into the step.  The complementarity
    // right-hand side of the corrector (x_core_qp_ipm_aux.c:695-754) is formed on the fly:
    // rm_mode 1: res_m = bkp + dt*dlam - sigma_mu; 2: res_m = bkp - sigma_mu.
    // ---------------------------------------------------------------------------------------------
    template <int KIND>
    FK_DEV void solve_stage(int k, int rm_mode, double sigma_mu, bool stw)
    {
        constexpr int nx = KD<KIND>::nx, nu = KD<KIND>::nu, n = nx + nu, nx1 = KD<KIND>::nx1;
        constexpr int nsolve = nu;                  // stage 0 has nx = 0: n = nu
        constexpr int RP = (n + G - 1) / G;
        const StageDesc &sd = sdk<KIND>();
        const View v = view<KIND>(k);
        const int nb = sd.nb, ns = sd.ns, nc = sd.nc;
        const int *idxb = IDX + 4 * (A.nmaps == 3 ? KIND : k) * A.nbe, *rev = idxb + nb, *inv = rev + nb;
        const int resN = (int) (sd.res.m - sd.res.g) + evn(nc), ltN = (int) (sd.sol.t - sd.sol.lam) + evn(nc);
        const int fvN = (int) (sd.w_Zsi - sd.w_Linv) + evn(2 * ns), stN = (int) (sd.step.t - sd.step.lam) + evn(nc);
        const int qmN = (int) (sd.q_Z - sd.q_dmask) + evn(2 * ns);
        double *RES = V, *LT = RES + (A.nve + NXe + 2 * A.nce), *FV = LT + 2 * A.nce, *RMB = FV + (2 * NMe + NXe + A.ns2e), *STL = RMB + A.nce;
        double *QM = STL + 2 * A.nce, *Gam = QM + (A.nce + A.ns2e), *gam = Gam + A.nce, *tmp0 = gam + A.nce, *tmp1 = tmp0 + A.nbe;
        double *ds = tmp1 + A.nbe, *xprev = ds + A.ns2e, *tmpx = xprev + NXe;
        const bool so = act && stw;
        stage_begin();
        vcopy<2>(RES, (size_t) v.kk * A.ws + sd.res.g, resN);
        vcopy<1>(LT, (size_t) v.kk * A.ss + sd.sol.lam, ltN);
        vcopy<2>(FV, (size_t) v.kk * A.ws + sd.w_Linv, fvN);
        vcopy<2>(RMB, (size_t) v.kk * A.ws + sd.w_rmb, evn(nc));
        vcopy<2>(STL, (size_t) v.kk * A.ws + sd.step.lam, stN);
        vcopy<0>(QM, (size_t) A.kq[KIND] + (size_t) v.kk * A.kqs + A.kV[KIND] + (sd.q_dmask - sd.q_b), qmN);
        if (nx1 > 0) bulk<0>(voff(MA), (size_t) A.kq[KIND] + (size_t) v.kk * A.kqs, evn(LDK * nx1));
        if (nsolve > 0) bulk<2>(voff(LU), (size_t) v.kk * A.ws + sd.w_L, evn(n * nsolve));
        stage_arm();
        wait_vec();
        double *vv = RES;
        const double *rd = RES + (sd.res.d - sd.res.g), *gl = LT, *gt = LT + (sd.sol.t - sd.sol.lam);
        const double *Lis = FV, *pbs = FV + (sd.w_Pb - sd.w_Linv), *Zi = FV + (sd.w_Zsi - sd.w_Linv);
        const double *dl = STL, *dtt = STL + (sd.step.t - sd.step.lam), *gm = QM, *qZ = QM + (sd.q_Z - sd.q_dmask);
        {
            double *grm = v.w + sd.res.m;
            const double t_min_inv = A.o.t_min > 0 ? 1.0 / A.o.t_min : 1e30;
            recip_vec(gt, Gam, nc);
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                const double l = gl[i], tt = gt[i], ti = Gam[i];
                double m = rm_mode == 1 ? RMB[i] + dtt[i] * dl[i] - sigma_mu : RMB[i] - sigma_mu;
                m *= gm[i];
                if (so) grm[i] = m;
                // the slack elimination needs the Gamma of the factorisation (clipped when t_lam_min==1)
                Gam[i] = (ns > 0 && A.o.t_lam_min == 1) ? (tt < A.o.t_min ? t_min_inv : ti) * (l < A.o.lam_min ? A.o.lam_min : l) : ti * l;
                gam[i] = ti * (m - l * rd[i]);
            }
        }
        fk_sync();
        if (ns > 0)
        {
            cond_slacks(nb, ns, rev, inv, qZ, 0, Gam, gam, vv + n, const_cast<double *>(Zi), ds, tmp0, tmp1);
            fk_sync();
            double *o_ = v.w + sd.step.ux + n;
#pragma unroll 1
            for (int j = li; j < 2 * ns; j += G)
                if (so) o_[j] = ds[j];
        }
        else
        {
#pragma unroll 1
            for (int i = li; i < nb; i += G) tmp1[i] = gam[i] - gam[nb + i];
            fk_sync();
        }
#pragma unroll 1
        for (int i = li; i < nb; i += G) vv[idxb[i]] += tmp1[i];
#pragma unroll 1
        for (int j = li; j < nx1; j += G) tmpx[j] = xprev[j] + pbs[j];
        wait_mat();
        fk_sync();
        double x[RPM > 0 ? RPM : 1];
#pragma unroll
        for (int m = 0; m < RP; m++) x[m] = vv[(li + G * m) < n ? li + G * m : 0];
        if (nx1 > 0)
        {
            double ap[RPM > 0 ? RPM : 1];
            rows_dot<n, nx1>(MA, LDK, tmpx, ap);
#pragma unroll
            for (int m = 0; m < RP; m++) x[m] += ap[m];
            fk_sync();
#pragma unroll
            for (int m = 0; m < RP; m++)
                if (li + G * m < nsolve) vv[li + G * m] = x[m];
            fk_sync();
        }
        // TRSV_LNN(_MN): forward substitution on the first nsolve unknowns (redundantly by every lane), then the rows below
        {
            double u[NU > 0 ? NU : 1];
#pragma unroll
            for (int j = 0; j < nsolve; j++)
            {
                double part = 0.0;
#pragma unroll
                for (int c = 0; c < j; c++) part += LU[j + n * c] * u[c];
                u[j] = (vv[j] - part) * Lis[j];
            }
            fk_sync();
#pragma unroll
            for (int m = 0; m < RP; m++)
            {
                const int i = li + G * m;
                if (i < n)
                {
                    double xi = x[m];
                    if (i < nsolve)
                    {
#pragma unroll
                        for (int j = 0; j < nsolve; j++)
                            if (i == j) xi = u[j];
                    }
                    else
                    {
                        double part = 0.0;
#pragma unroll
                        for (int c = 0; c < nsolve; c++) part += LU[i + n * c] * u[c];
                        xi -= part;
                    }
                    if (so) (v.w + sd.step.ux)[i] = xi;
                    if (i >= nu) xprev[i - nu] = xi;
                }
            }
        }
    }

    FK_DEV void solve_backward(int rm_mode, double sigma_mu, bool stw)
    {
        fk_fence_async_global();        // the records this sweep reads with bulk copies were written with plain stores by the sweeps before

        solve_stage<2>(A.N, rm_mode, sigma_mu, stw);
        for (int k = A.N - 1; k >= 1; k--) solve_stage<1>(k, rm_mode, sigma_mu, stw);
        solve_stage<0>(0, rm_mode, sigma_mu, stw);
    }

    // ---------------------------------------------------------------------------------------------
    // one stage of the forward sweep (x_ocp_qp_kkt.c:968-1006 / 1682-1722) + step of the constraint variables
    // (:1176-1193, EXPAND_SLACKS :524-598, COMPUTE_LAM_T_QP x_core_qp_ipm_aux.c:164-189) + the ratio test
    // (COMPUTE_ALPHA_QP :375-398) + the norms of the b, d and m rows of the residual of the linear system
    // (OCP_QP_RES_COMPUTE_LIN).  Its stationarity rows need the Hessian: the residual sweep that applies the step computes
    // them (res_stage), so this sweep streams the factor only.  The affine step (after_fact) is overwritten by the
    // corrector before that sweep: with do_lin its dux, dpi and masked dlam are kept in the residual set 1 area of the work
    // record (ires.g / .b / .d), which this kernel uses for nothing else.
    // after_fact: start from -lrow, pi = P x + p with p from lrow; else: start from the backward quantities stored in
    // the step, pi = p_backward + P x.
    // ---------------------------------------------------------------------------------------------
    struct FwdAcc
    {
        double alpha, m1, m2, m3;
        int f1, f2, f3;
    };

    template <int KIND>
    FK_DEV void fwd_stage(int k, int after_fact, int do_lin, bool stw, FwdAcc &F)
    {
        constexpr int nx = KD<KIND>::nx, nu = KD<KIND>::nu, n = nx + nu, nx1 = KD<KIND>::nx1;
        constexpr int nsolve = nu;
        constexpr int CP = (nx1 + G - 1) / G;
        FK_PROF_T2();
        const StageDesc &sd = sdk<KIND>();
        const View v = view<KIND>(k);
        const int nb = sd.nb, ns = sd.ns, nc = sd.nc;
        const int *idxb = IDX + 4 * (A.nmaps == 3 ? KIND : k) * A.nbe, *rev = idxb + nb, *inv = rev + nb;
        const int nu1 = (nx1 > 0 && k + 1 < A.N) ? NU : 0, n1 = nx1 + nu1, n1e = (n1 + 1) & ~1;
        const int resN = (int) (sd.res.m - sd.res.b) + evn(nc), ltN = (int) (sd.sol.t - sd.sol.lam) + evn(nc);
        const int fvN = (int) (sd.w_Zsi - sd.w_Linv) + evn(2 * ns);
        double *RES = V, *LT = RES + (A.nve + NXe + 2 * A.nce), *FV = LT + 2 * A.nce, *SUX = FV + (2 * NMe + NXe + A.ns2e), *P1 = SUX + A.nve;
        double *QM = P1 + NMe, *vv = QM + (A.nce + A.ns2e), *x1 = vv + A.nve, *tmp = x1 + NXe;
        double *dt = tmp + A.nve, *tis = dt + A.nce, *dsv = tis + A.nce;
        const bool so = act && stw, sa = so && after_fact && do_lin;      // sa: keep the affine step for the residual sweep
        View v1 = v;
        const StageDesc *s1p = &sd;
        if (nx1 > 0) { s1p = &sdr(k + 1); v1 = viewr(k + 1); }
        stage_begin();
        vcopy<2>(RES, (size_t) v.kk * A.ws + sd.res.b, resN);
        vcopy<1>(LT, (size_t) v.kk * A.ss + sd.sol.lam, ltN);
        vcopy<2>(FV, (size_t) v.kk * A.ws + sd.w_Linv, fvN);
        vcopy<2>(SUX, (size_t) v.kk * A.ws + sd.step.ux, evn(n + 2 * ns));
        vcopy<0>(QM, (size_t) A.kq[KIND] + (size_t) v.kk * A.kqs + A.kV[KIND] + (sd.q_dmask - sd.q_b), evn(nc));
        if (nx1 > 0)
        {
            // p part (gradient vector of stage k+1) / backward value of x_{k+1}
            vcopy<2>(P1, (size_t) v1.kk * A.ws + (after_fact ? s1p->w_lrow : s1p->step.ux), n1e);
            bulk<0>(voff(MA), (size_t) A.kq[KIND] + (size_t) v.kk * A.kqs, evn(LDK * nx1));
        }
        if (nsolve > 0) bulk<2>(voff(LU), (size_t) v.kk * A.ws + sd.w_L, evn(n * nsolve));
        if (nx1 > 0) bulk<2>(voff(ML), (size_t) v1.kk * A.ws + s1p->w_Lxx, evn((nx1 | 1) * nx1));
        stage_arm();
        wait_vec();
        const double *bs = RES, *rds = RES + (sd.res.d - sd.res.b), *rms = RES + (sd.res.m - sd.res.b);
        const double *lam = LT, *ts = LT + (sd.sol.t - sd.sol.lam);
        const double *Lis = FV, *lrow_ = FV + (sd.w_lrow - sd.w_Linv), *Zi = FV + (sd.w_Zsi - sd.w_Linv);
        const double *mks = QM;
        {
            const double *src = after_fact ? lrow_ : SUX;
#pragma unroll 1
            for (int i = li; i < nsolve; i += G) vv[i] = -src[i];
            // x part (k>0) was written into vv by the previous stage
#pragma unroll 1
            for (int j = li; j < 2 * ns; j += G) dsv[j] = SUX[n + j];
        }
        wait_mat();
        fk_sync();
        FK_PROF_ADD2(16);      /* issue + waits */
        // ---- TRSV_LTN(_MN): u = -Luu^{-T} (l_u + Lxu' x): the dot products over the x rows by the group, the small triangle
        // redundantly by every lane
        if (nsolve > 0)
        {
            double wv[NU > 0 ? NU : 1];
#pragma unroll
            for (int j = 0; j < nsolve; j++)
            {
                double part = 0.0;
                for (int i = nsolve + li; i < n; i += G) part += LU[i + n * j] * vv[i];
                if (n > nsolve) part = gsum(part);
                wv[j] = vv[j] - part;
            }
#pragma unroll
            for (int j = nsolve - 1; j >= 0; j--)
            {
                double part = 0.0;
#pragma unroll
                for (int i = j + 1; i < nsolve; i++) part += LU[i + n * j] * wv[i];
                wv[j] = (wv[j] - part) * Lis[j];
            }
            fk_sync();
#pragma unroll
            for (int j = 0; j < nsolve; j++)
                if (li == j % G) vv[j] = wv[j];
            fk_sync();
        }
        {
            double *o_ = v.w + sd.step.ux, *oa = v.w + sd.ires.g;
#pragma unroll 1
            for (int i = li; i < n; i += G)
            {
                if (so) o_[i] = vv[i];
                if (sa) oa[i] = vv[i];
            }
        }
        FK_PROF_ADD2(17);      /* u */
        // ---- x+ = A' v + b
        if (nx1 > 0)
        {
            double av[RPM > 0 ? RPM : 1];
            cols_dot<n, nx1>(MA, LDK, vv, av);
#pragma unroll
            for (int m = 0; m < CP; m++)
            {
                const int j = li + G * m;
                if (j < nx1)
                {
                    const double acc = av[m], bv = bs[j];
                    const double xj = bv + acc;
                    x1[j] = xj;
                    if (do_lin)
                    {
                        const double r = bv - xj + acc;
                        const double a = fabs(r);
                        F.m1 = fmax(F.m1, a);
                        F.f1 |= (a != a);
                    }
                }
            }
        }
        FK_PROF_ADD2(19);      /* x+ */
        // ---- constraint part of the step at this stage
        {
            recip_vec(ts, tis, nc);
#pragma unroll 1
            for (int i = li; i < nb; i += G)
            {
                const double a = vv[idxb[i]];
                dt[i] = a;
                dt[nb + i] = -a;
            }
            if (ns > 0)
            {
                fk_sync();
                const double t_min_inv = A.o.t_min > 0 ? 1.0 / A.o.t_min : 1e30;
#pragma unroll 1
                for (int j = li; j < 2 * ns; j += G)
                {
                    const int jj = j < ns ? j : j - ns, offc = j < ns ? 0 : nb;
                    double d = dsv[j];
                    FK_FOR_SLACK(i, jj)
                        {
                            const double l = lam[offc + i], tt = ts[offc + i];
                            const double Gm = A.o.t_lam_min == 1 ? (tt < A.o.t_min ? t_min_inv : tis[offc + i]) * (l < A.o.lam_min ? A.o.lam_min : l) : tis[offc + i] * l;
                            d += Gm * dt[offc + i];
                        }
                    d = -Zi[j] * d;
                    dsv[j] = d;
                    dt[2 * nb + j] = d;
                }
                fk_sync();
#pragma unroll 1
                for (int i = li; i < 2 * nb; i += G)
                {
                    const int up = i >= nb, ii = up ? i - nb : i;
                    if (rev[ii] >= 0) dt[i] += dsv[(up ? ns : 0) + rev[ii]];
                }
                double *o_ = v.w + sd.step.ux + n, *oa = v.w + sd.ires.g + n;
#pragma unroll 1
                for (int j = li; j < 2 * ns; j += G)
                {
                    if (so) o_[j] = dsv[j];
                    if (sa) oa[j] = dsv[j];
                }
            }
            fk_sync();
            double *odl = v.w + sd.step.lam, *odt = v.w + sd.step.t, *oa = v.w + sd.ires.d;
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                const double l = lam[i], tt = ts[i], ti = tis[i], rdi = rds[i], rmi = rms[i];
                const double dtr = dt[i];
                double dl = -ti * (rmi + (l * dtr) - (l * rdi));
                double dti = dtr - rdi;
                const double mk = mks[i];
                dl *= mk;
                dti *= mk;
                if (so) { odl[i] = dl; odt[i] = dti; }
                if (sa) oa[i] = dl * mk;       // masked step multipliers (tmp_lam_mask of the linear residual)
                // ratio test (min over constraints, see COMPUTE_ALPHA_QP)
                if (l + dl < 0.0) F.alpha = fmin(F.alpha, -l / dl);
                if (tt + dti < 0.0) F.alpha = fmin(F.alpha, -tt / dti);
                if (do_lin)
                {
                    // res_d = rhs_d + dt -/+ (v[idxb] | C'v) [- ds] = rhs_d + dt - dtr ;  res_m = rhs_m + lam dt + dlam t
                    double r = (dti + rdi) - dtr;
                    r *= mk;
                    double a = fabs(r);
                    F.m2 = fmax(F.m2, a);
                    F.f2 |= (a != a);
                    double mm = rmi + l * dti + dl * tt;
                    mm *= mk;
                    a = fabs(mm);
                    F.m3 = fmax(F.m3, a);
                    F.f3 |= (a != a);
                }
            }
        }
        FK_PROF_ADD2(20);      /* constraint step */
        // ---- pi = P x+ + p with the factor of the next stage
        if (nx1 > 0)
        {
            fk_sync();
            const double *Lx = ML;                                          // Lxx of stage k+1, odd leading dimension, zero above the diagonal
            constexpr int ldx = nx1 | 1;
            double tt_[RPM > 0 ? RPM : 1];
            cols_dot<nx1, nx1>(Lx, ldx, x1, tt_);
#pragma unroll
            for (int m = 0; m < CP; m++)
            {
                const int j = li + G * m;
                if (j < nx1) tmp[j] = after_fact ? tt_[m] + P1[nu1 + j] : tt_[m];
            }
            fk_sync();
            double *pi = v.w + sd.step.pi, *oa = v.w + sd.ires.b;
            rows_dot<nx1, nx1>(Lx, ldx, tmp, tt_);
#pragma unroll
            for (int m = 0; m < CP; m++)
            {
                const int i = li + G * m;
                if (i < nx1)
                {
                    const double pv = after_fact ? tt_[m] : tt_[m] + P1[nu1 + i];
                    if (so) pi[i] = pv;
                    if (sa) oa[i] = pv;
                }
            }
        }
        fk_sync();
        FK_PROF_ADD2(21);      /* pi */
        if (nx1 > 0)
        {
#pragma unroll 1
            for (int j = li; j < nx1; j += G) vv[nu1 + j] = x1[j];
        }
    }

    // returns the step length; lin_nrm[1..3] = inf-norms of the b, d, m rows of the residual of the linear system (do_lin)
    FK_DEV double forward_pass(int after_fact, int do_lin, bool stw, double lin_nrm[4])
    {
        fk_fence_async_global();        // the records this sweep reads with bulk copies were written with plain stores by the sweeps before

        FwdAcc F;
        F.alpha = 1.0;
        F.m1 = F.m2 = F.m3 = 0.0;
        F.f1 = F.f2 = F.f3 = 0;
        fwd_stage<0>(0, after_fact, do_lin, stw, F);
        for (int k = 1; k < A.N; k++) fwd_stage<1>(k, after_fact, do_lin, stw, F);
        fwd_stage<2>(A.N, after_fact, do_lin, stw, F);
        if (do_lin)
        {
            lin_nrm[1] = gmax_nan(F.m1, F.f1);
            lin_nrm[2] = gmax_nan(F.m2, F.f2);
            lin_nrm[3] = gmax_nan(F.m3, F.f3);
        }
        return gmin(F.alpha);
    }

    // COMPUTE_MU_AFF_QP (x_core_qp_ipm_aux.c:636-668): a streaming reduction over (lam, t) of the solution record and
    // (dlam, dt) of the step.  Nothing here depends on anything but the loads, so the sweep is limited by how many of them are in
    // flight: the interior stages (same layout, record strides ss / ws) are taken two at a time, up to four constraints per lane
    // each, all 32 loads of a lane issued before the first use; stages 0 and N, and shapes with more than 4 G constraints per
    // stage, take the plain loop.
    FK_DEV double mu_aff_pass(double alpha)
    {
        const int N = A.N;
        double acc = 0.0;
        auto plain = [&](int k) {
            const StageDesc &s = sdr(k);
            const View v = viewr(k);
            const double *l = v.s + s.sol.lam, *t = v.s + s.sol.t, *dl = v.w + s.step.lam, *dt = v.w + s.step.t;
#pragma unroll 1
            for (int i = li; i < s.nc; i += G) acc += fabs((l[i] + alpha * dl[i]) * (t[i] + alpha * dt[i]));
        };
        plain(0);
        const int nc1 = A.s1.nc, ni = N - 1;       // interior stages 1 .. N-1
        if (ni > 0 && nc1 <= 4 * G)
        {
            const double *l0 = sol + A.s1.sol.lam, *t0 = sol + A.s1.sol.t, *d0 = wk + A.s1.step.lam, *e0 = wk + A.s1.step.t;
            int io[4];
            bool iv[4];
#pragma unroll
            for (int j = 0; j < 4; j++) { iv[j] = li + G * j < nc1; io[j] = iv[j] ? li + G * j : 0; }
            for (int kk = 0; kk < ni; kk += 2)
            {
                double L[2][4], T[2][4], DL[2][4], DT[2][4];
#pragma unroll
                for (int u = 0; u < 2; u++)
                {
                    const unsigned k2 = (unsigned) (kk + u < ni ? kk + u : kk);
                    const double *l = l0 + k2 * A.ss, *t = t0 + k2 * A.ss, *dl = d0 + k2 * A.ws, *dt = e0 + k2 * A.ws;
#pragma unroll
                    for (int j = 0; j < 4; j++) { L[u][j] = l[io[j]]; T[u][j] = t[io[j]]; DL[u][j] = dl[io[j]]; DT[u][j] = dt[io[j]]; }
                }
#pragma unroll
                for (int u = 0; u < 2; u++)
#pragma unroll
                    for (int j = 0; j < 4; j++)
                    {
                        const double p = fabs((L[u][j] + alpha * DL[u][j]) * (T[u][j] + alpha * DT[u][j]));
                        if (iv[j] && kk + u < ni) acc += p;
                    }
            }
        }
        else
            for (int k = 1; k < N; k++) plain(k);
        if (N > 0) plain(N);
        return gsum(acc) * nc_mask_inv;
    }

    // OCP_QP_INIT_VAR, var_init_scheme 1 (x_ocp_qp_ipm.c:1611-1760,1884-2022); no general constraints here
    FK_DEV void init_var()
    {
        const double thr0 = 0.1;
        const int N = A.N;
        // the reference's plugin zeroes the primal iterate before every solve, whatever warm_start says
        // (acados/ocp_qp/ocp_qp_hpipm.c:333-336): warm starts carry over pi, lam and t only
        if (A.o.warm_start >= 2)
        {
            const double lmin = A.o.warm_start >= 3 ? A.o.lam0_min : thr0, tmin = A.o.warm_start >= 3 ? A.o.t0_min : thr0;
            for (int k = 0; k <= N; k++)
            {
                const StageDesc &s = sdr(k);
                const View v = viewr(k);
                double *l = v.s + s.sol.lam, *t = v.s + s.sol.t, *gux = v.s + s.sol.ux, *gpi = v.s + s.sol.pi;
                // keep what the caller passed in for the case that this QP is handed back to the generic kernel
                double *kl = v.w + s.itref.lam, *kt = v.w + s.itref.t, *kp = v.w + s.itref.pi;
#pragma unroll 1
                for (int i = li; i < s.n + 2 * s.ns; i += G) st(gux + i, 0.0);
#pragma unroll 1
                for (int i = li; i < s.nx1; i += G) st(kp + i, gpi[i]);
#pragma unroll 1
                for (int i = li; i < s.nc; i += G)
                {
                    st(kl + i, l[i]);
                    st(kt + i, t[i]);
                    if (l[i] < lmin) st(l + i, lmin);
                    if (t[i] < tmin) st(t + i, tmin);
                }
            }
            fk_sync();
            return;
        }
        double *ux = V, *tt = ux + A.nve;
        for (int k = 0; k <= N; k++)
        {
            const StageDesc &s = sdr(k);
            const View v = viewr(k);
            const int n = s.n, nb = s.nb, ns = s.ns, nc = s.nc;
            const int *idxb = IDX + 4 * (A.nmaps == 3 ? (k == 0 ? 0 : (k == A.N ? 2 : 1)) : k) * A.nbe, *rev = idxb + nb;
            const double *d = v.q + s.q_d;
            double *gux = v.s + s.sol.ux, *gpi = v.s + s.sol.pi, *gl = v.s + s.sol.lam, *gt = v.s + s.sol.t;
#pragma unroll 1
            for (int i = li; i < s.nx1; i += G) st(gpi + i, 0.0);
            if (A.o.t0_init == 0 || A.o.t0_init == 1)
            {
                const double l0 = A.o.t0_init == 0 ? sqrt(A.o.mu0) : A.o.mu0, t0 = A.o.t0_init == 0 ? sqrt(A.o.mu0) : 1.0;
#pragma unroll 1
                for (int i = li; i < n + 2 * ns; i += G) st(gux + i, 0.0);
#pragma unroll 1
                for (int i = li; i < nc; i += G) { st(gl + i, l0); st(gt + i, t0); }
                continue;
            }
#pragma unroll 1
            for (int i = li; i < n + 2 * ns; i += G) ux[i] = 0.0;
            fk_sync();
#pragma unroll 1
            for (int j = li; j < 2 * ns; j += G)
            {
                double tj = ux[n + j] - d[2 * nb + j];
                if (tj < thr0)
                {
                    tj = thr0;
                    ux[n + j] = d[2 * nb + j] + tj;
                }
                tt[2 * nb + j] = tj;
            }
            fk_sync();
#pragma unroll 1
            for (int j = li; j < nb; j += G)
            {
                const int ix = idxb[j];
                double tl = ux[ix], tu = -ux[ix];
                if (ns > 0 && rev[j] != -1) { tl += ux[n + rev[j]]; tu += ux[n + ns + rev[j]]; }
                tl -= d[j];
                tu -= d[nb + j];
                if (tl < thr0)
                {
                    if (tu < thr0)
                    {
                        ux[ix] = 0.5 * (d[j] - d[nb + j]);
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
                    ux[ix] = -d[nb + j] - thr0;
                }
                tt[j] = tl;
                tt[nb + j] = tu;
            }
            fk_sync();
#pragma unroll 1
            for (int i = li; i < n + 2 * ns; i += G) st(gux + i, ux[i]);
#pragma unroll 1
            for (int i = li; i < nc; i += G)
            {
                st(gt + i, tt[i]);
                st(gl + i, A.o.mu0 / tt[i]);
            }
            fk_sync();
        }
        fk_sync();
    }

    // ---------------------------------------------------------------------------------------------
    // driver (OCP_QP_IPM_SOLVE x_ocp_qp_ipm.c:2684-3120 + OCP_QP_IPM_DELTA_STEP :2208-2682) for the QPs of this warp;
    // q = index of this group's QP (clamped to a valid one; valid = it exists)
    // ---------------------------------------------------------------------------------------------
    FK_DEV void bind(int q, bool valid)
    {
        qp = A.qp + (size_t) q * A.qp_stride;
        qk = A.qpk + (size_t) q * A.qpk_stride;
        sol = A.sol + (size_t) q * A.sol_stride;
        wk = A.work + (size_t) q * A.work_stride;
        act = valid;
    }

    // start of a solve: statistics cleared, mask census, initial point; the QP is handed back if no constraint is active
    FK_DEV void prologue(int q, cuipm_info *info, double *stat)
    {
        const int N = A.N;
        const int SM = CUIPM_STAT_M;
        if (stat && act)
#pragma unroll 1
            for (int i = li; i < SM * (A.o.stat_max + 1); i += G) stat[i] = 0.0;

        // constraint mask census (x_ocp_qp_ipm.c:2774-2806)
        int cnt = 0;
        for (int k = 0; k <= N; k++)
        {
            const StageDesc &s = sdr(k);
            const double *gm = viewr(k).q + s.q_dmask;
#pragma unroll 1
            for (int i = li; i < s.nc; i += G) cnt += fk_ldg(gm + i) != 0.0;
        }
        const int nc_mask = (int) (gsum((double) cnt) + 0.5);
        nc_mask_inv = nc_mask > 0 ? 1.0 / nc_mask : 0.0;
        bool redo = nc_mask == 0;          // no active constraint: the unconstrained branch lives in the generic kernel

        if (act && redo) { hand_back(q, info); act = false; }
        init_var();
        // masked constraints start with zero multipliers (the generic kernel does this only when some constraint is masked;
        // multiplying by 1.0 is exact)
        for (int k = 0; k <= N; k++)
        {
            const StageDesc &s = sdr(k);
            const View v = viewr(k);
            double *l = v.s + s.sol.lam;
            const double *gm = v.q + s.q_dmask;
#pragma unroll 1
            for (int i = li; i < s.nc; i += G) st(l + i, l[i] * fk_ldg(gm + i));
        }
        fk_sync();
    }

    // statistics row of pass kk, loop condition of the QP (x_ocp_qp_ipm.c:3017-3031); a QP that stops gets its summary written
    // and its stores disabled
    FK_DEV void close_pass(int kk, const QpState &Q, cuipm_info *info, double *stat)
    {
        const int SM = CUIPM_STAT_M;
        if (stat && act && kk < A.o.stat_max && li == 0)
        {
            double *sr = stat + SM * (size_t) kk;
            if (kk > 0) sr[6] = Q.mu;
            sr[7] = Q.res_max[0]; sr[8] = Q.res_max[1]; sr[9] = Q.res_max[2]; sr[10] = Q.res_max[3];
            sr[11] = Q.gap; sr[12] = Q.obj;
        }
        const bool go = kk < A.o.iter_max && Q.alpha > A.o.alpha_min
                        && (Q.res_max[0] > A.o.res_g_max || Q.res_max[1] > A.o.res_b_max || Q.res_max[2] > A.o.res_d_max
                            || Q.res_m_tau > A.o.res_m_max || Q.gap > A.o.dual_gap_max);
        if (act && !go)
        {
            int status;
            if (kk == A.o.iter_max) status = CUIPM_MAX_ITER;
            else if (Q.alpha <= A.o.alpha_min) status = CUIPM_MIN_STEP;
            else if (Q.mu != Q.mu) status = CUIPM_NAN_SOL;
            else status = CUIPM_SUCCESS;
            if (li == 0)
            {
                info->status = status;
                info->iter = kk;
                for (int i = 0; i < 4; i++) info->res_max[i] = Q.res_max[i];
                info->mu = Q.mu;
                info->obj = Q.obj;
                info->dual_gap = Q.gap;
                info->lq_count = 0;
                info->reserved = 0;
            }
            act = false;
        }
    }

    // one interior-point iteration after pass kk: predictor / corrector / conditional corrector (OCP_QP_IPM_DELTA_STEP); leaves
    // the step length in Q.alpha.  Every sweep has exactly one call site (everything is inlined into the kernel, and the hot code
    // should exist once): the phases 0 / 1 / 2 of one inner loop.
    FK_DEV void iteration(int q, int kk, QpState &Q, LinNrm &L, cuipm_info *info, double *stat)
    {
        const int SM = CUIPM_STAT_M;
        double *stt = (stat && kk + 1 < A.o.stat_max) ? stat + SM * (size_t) (kk + 1) : nullptr;
        double nrm[4] = {0, 0, 0, 0};
        double alpha = 1.0, mu_aff = 0.0, sigma_mu = 0.0;
        bool need = true;
        // affine direction: res_m already holds lam*t - tau_min (written by the residual sweep)
        for (int ph = 0; ph < 3; ph++)
        {
            const bool stw = ph < 2 ? true : need;
            { FK_PROF_T0(); if (ph == 0) fact_backward(); else solve_backward(ph, sigma_mu, stw); FK_PROF_ADD(ph == 0 ? 1 : 3); }
            const int do_lin = ph == 0 ? A.o.lq_fact == 1 : A.o.itref_corr_max > 0;
            double nr[4] = {0, 0, 0, 0};
            double al; { FK_PROF_T0(); al = forward_pass(ph == 0, do_lin, stw, nr); FK_PROF_ADD(2); }
            if (stw) { alpha = al; nrm[1] = nr[1]; nrm[2] = nr[2]; nrm[3] = nr[3]; }
            if (ph == 0)
            {
                // (the test itself waits for the stationarity rows: lin_check)
                L.aff_bdm_large = nr[1] > 1e-5 || nr[2] > 1e-5 || nr[3] > 1e-5;
                if (stt && act && li == 0) { stt[13] = 0; stt[0] = alpha; stt[1] = alpha; }
                if (A.o.pred_corr != 1) break;
            }
            else if (ph == 2 || A.o.cond_pred_corr != 1)
                break;
            const double mu_aff0 = mu_aff;
            { FK_PROF_T0(); mu_aff = mu_aff_pass(alpha); FK_PROF_ADD(4); }
            if (ph == 0)
            {
                const double tmp = mu_aff / Q.mu;
                const double sigma = tmp * tmp * tmp;
                sigma_mu = sigma * Q.mu;
                sigma_mu = sigma_mu > A.o.tau_min ? sigma_mu : A.o.tau_min;
                if (stt && act && li == 0) { stt[2] = mu_aff; stt[3] = sigma; }
            }
            else
            {
                need = mu_aff > 2.0 * mu_aff0;
                if (!fk_any(act && need)) break;
            }
        }
        if (A.o.pred_corr == 1)
        {
            if (A.o.itref_corr_max > 0)
            {
                // (the test itself waits for the stationarity rows: lin_check; stt[16] is written there)
                L.res0_g = Q.res_max[0];
                L.fin_bdm_small = (nrm[1] < A.o.res_b_max || nrm[1] < 1e-3 * Q.res_max[1]) && (nrm[2] < A.o.res_d_max || nrm[2] < 1e-3 * Q.res_max[2])
                                  && (nrm[3] < A.o.res_m_max || nrm[3] < 1e-3 * Q.res_max[3]);
                if (stt && act && li == 0) { stt[17] = nrm[1]; stt[18] = nrm[2]; stt[19] = nrm[3]; }
            }
            if (stt && act && li == 0) { stt[4] = alpha; stt[5] = alpha; }
        }
        if (stt && act && li == 0) stt[15] = 0;
        Q.alpha = alpha;
    }

    // the tests on the residual of the linear system of the iteration that led to pass kk, once the residual sweep of pass kk has
    // formed its stationarity rows; a QP that fails one is handed back (it restarts from scratch in the generic kernel: the
    // sweeps it ran here after the step that failed change none of its results)
    FK_DEV void lin_check(int q, int kk, const LinNrm &L, cuipm_info *info, double *stat)
    {
        if (A.o.lq_fact == 1)
        {
            // a Cholesky step that leaves a large residual in the linear system switches the solve to the LQ
            // refactorisation (x_ocp_qp_ipm.c:2246-2346): cold path, generic kernel
            if (L.aff_g > 1e-5 || L.aff_bdm_large)
                if (act) { hand_back(q, info); act = false; }
        }
        if (A.o.pred_corr == 1 && A.o.itref_corr_max > 0)
        {
            // iterative refinement is needed when the residual of the corrector system is not small
            // (x_ocp_qp_ipm.c:2540-2620): cold path, generic kernel
            const bool small_ = (L.fin_g < A.o.res_g_max || L.fin_g < 1e-3 * L.res0_g) && L.fin_bdm_small;
            if (!small_ && act) { hand_back(q, info); act = false; }
            if (stat && kk < A.o.stat_max && act && li == 0) stat[CUIPM_STAT_M * (size_t) kk + 16] = L.fin_g;
        }
    }

    FK_DEV void solve(int q, bool valid)
    {
        const int SM = CUIPM_STAT_M;
        bind(q, valid);
        cuipm_info *info = A.info + q;
        double *stat = A.stat ? A.stat + (size_t) q * SM * (A.o.stat_max + 1) : nullptr;
        QpState Q;
        Q.mu = Q.obj = Q.gap = 0.0; Q.alpha = 1.0; Q.res_m_tau = 0.0;
        Q.res_max[0] = Q.res_max[1] = Q.res_max[2] = Q.res_max[3] = 0.0;
        LinNrm L;
        prologue(q, info, stat);
        // the residual sweep opens each pass of the loop (pass 0: residuals of the initial point; pass kk: move along the step
        // of iteration kk-1, then residuals)
        for (int kk = 0;; kk++)
        {
            { FK_PROF_T0(); res_pass(kk > 0, Q.alpha, Q, L); FK_PROF_ADD(0); }
            if (kk > 0) lin_check(q, kk, L, info, stat);
            close_pass(kk, Q, info, stat);
            // the warp leaves when none of its QPs continues
            if (!fk_any(act)) break;
            iteration(q, kk, Q, L, info, stat);
        }
    }

    // ---------------------------------------------------------------------------------------------
    // Iteration-sliced scheduling.  A 4096-QP batch is 1.73 waves of the QPs an SM array can hold; with a QP bound to its warp for
    // the whole solve every slot serves one or two QPs and the launch lasts two of the longest solves.  Here a QP is bound to a
    // warp for ONE iteration: all its state between iterations lives in its records (plus a dozen scalars in rr_state), so the QPs
    // that are not finished circulate through a FIFO ring -- every group pops one QP per pass, runs the iteration and the residual
    // sweep, and pushes the QP back unless it stopped.  All QPs advance at the same rate, the slots stay filled until fewer QPs
    // than slots are alive.  Two launches: rr_first (initial point + residual sweep 0 of every QP, fills the ring), rr_loop.
    // Which QP next: the launch ends with the slowest QP, and how far a QP is from the end shows in its duality measure (on the
    // benchmark batch log mu after three iterations correlates 0.7-0.77 with the final iteration count), so the ring is RRK rings,
    // one per decade of mu, and a warp takes the QPs with the largest mu first -- "longest remaining first" with mu as the estimate.
    // A simulation on the measured per-iteration statistics gives 19 passes for the 4096 batch against 22-23 for one FIFO ring
    // (17 with the true remaining counts, 16.3 = work / slots).
    //   rr_ctr[b], b < RRK: head of ring b; rr_ctr[RRK + b]: tail (positions, monotonic; slot = b*nbatch + position mod nbatch,
    //   -1 = empty); rr_ctr[2 RRK]: QPs that stopped
    // ---------------------------------------------------------------------------------------------
    static constexpr int RRS = 12;             // doubles of a QP's scalar state
    static constexpr int RRK = CUIPM_RR_RINGS; // rings: mu >= 1e-1, >= 1e-2, ..., the rest (a NaN goes first)
    FK_DEV static int rr_bucket(double mu)
    {
        int b = 0;
        double th = 0.1;
#pragma unroll
        for (int i = 0; i < RRK - 1; i++) { b += mu < th; th *= 0.1; }
        return b;
    }
    FK_DEV void rr_save(int q, int kk, const QpState &Q) const
    {
        double *r = A.rr_state + (size_t) q * RRS;
        r[0] = Q.mu; r[1] = Q.obj; r[2] = Q.gap; r[3] = Q.alpha; r[4] = Q.res_m_tau;
        r[5] = Q.res_max[0]; r[6] = Q.res_max[1]; r[7] = Q.res_max[2]; r[8] = Q.res_max[3];
        r[9] = nc_mask_inv; r[10] = (double) kk;
    }
    FK_DEV int rr_load(int q, QpState &Q)
    {
        const double *r = A.rr_state + (size_t) q * RRS;
        Q.mu = r[0]; Q.obj = r[1]; Q.gap = r[2]; Q.alpha = r[3]; Q.res_m_tau = r[4];
        Q.res_max[0] = r[5]; Q.res_max[1] = r[6]; Q.res_max[2] = r[7]; Q.res_max[3] = r[8];
        nc_mask_inv = r[9];
        return (int) r[10];
    }
    FK_DEV int wmax_i(int v) const
    {
#pragma unroll
        for (int m = 16; m > 0; m >>= 1)
        {
            const int o = fk_shfl_xor_i(v, m);
            v = o > v ? o : v;
        }
        return v;
    }
    FK_DEV int gmax_i(int v) const
    {
#pragma unroll
        for (int m = G / 2; m > 0; m >>= 1)
        {
            const int o = fk_shfl_xor_i(v, m);
            v = o > v ? o : v;
        }
        return v;
    }
    // the QP of this group stopped (or was handed back) / goes on: count it / put it back into the ring.  All lanes have made their
    // stores of the pass visible before lane 0 of the group publishes the index.
    FK_DEV void rr_publish(int q, bool have, int kk, const QpState &Q)
    {
        fk_threadfence();
        fk_sync();
        if (have && li == 0)
        {
            if (!act)
                fk_atomic_add(A.rr_ctr + 2 * RRK, 1);
            else
            {
                rr_save(q, kk, Q);
                fk_threadfence();
                const int b = rr_bucket(Q.mu);
                const int pos = fk_atomic_add(A.rr_ctr + RRK + b, 1);
                int *slot = A.rr_ring + ((size_t) b * A.nbatch + pos % A.nbatch);
                while (fk_ld_volatile(slot) >= 0) {}          // (the previous lap's entry has been popped; its reader clears it at once)
                fk_st_volatile(slot, q);
            }
        }
        fk_sync();
    }

    // first launch: QPs first_qp .. first_qp + QPW - 1
    FK_DEV void rr_first(int first_qp)
    {
        const int SM = CUIPM_STAT_M;
        int q = first_qp + gq;
        const bool valid = q < A.nbatch;
        if (!valid) q = A.nbatch - 1;
        bind(q, valid);
        cuipm_info *info = A.info + q;
        double *stat = A.stat ? A.stat + (size_t) q * SM * (A.o.stat_max + 1) : nullptr;
        QpState Q;
        Q.mu = Q.obj = Q.gap = 0.0; Q.alpha = 1.0; Q.res_m_tau = 0.0;
        Q.res_max[0] = Q.res_max[1] = Q.res_max[2] = Q.res_max[3] = 0.0;
        LinNrm L;
        prologue(q, info, stat);
        res_pass(0, 1.0, Q, L);
        close_pass(0, Q, info, stat);
        rr_publish(q, valid, 0, Q);
        fk_sync();
    }

    // second launch: the loop over the ring
    FK_DEV void rr_loop()
    {
        const int SM = CUIPM_STAT_M;
        unsigned nap = 4000;        // nanoseconds between two looks at an empty ring: doubled up to 128 us while nothing turns up (a
                                    // thousand idle warps polling the counters every few microseconds starve the atomics of the
                                    // warps that still work: measured 4.6x on a batch with a handful of 50-iteration stragglers)
        for (;;)
        {
            // one lane reserves positions for all groups of the warp (a compare-and-swap per group made thousands of lanes retry
            // against each other on shapes with many QPs per warp); a position below the tail counter has a writer on its way
            // (the rings are visited from the largest mu down until every group has a QP)
            int cnt = 0;
            size_t myslot = 0;
            bool mine = false;
            for (int b = 0; b < RRK && cnt < QPW; b++)
            {
                int base = -1, got = 0;
                if (fk_lane() == 0)
                    for (;;)
                    {
                        const int h = fk_ld_volatile(A.rr_ctr + b), t = fk_ld_volatile(A.rr_ctr + RRK + b);
                        if (h >= t) break;                               // nothing queued here right now
                        const int want = t - h < QPW - cnt ? t - h : QPW - cnt;
                        if (fk_atomic_cas(A.rr_ctr + b, h, h + want) == h) { base = h; got = want; break; }
                    }
                base = wmax_i(base);
                got = wmax_i(got);
                if (got > 0 && gq >= cnt && gq < cnt + got)
                {
                    mine = true;
                    myslot = (size_t) b * A.nbatch + (base + gq - cnt) % A.nbatch;
                }
                cnt += got;
            }
            int q = -1;
            if (li == 0 && mine)
            {
                int *slot = A.rr_ring + myslot;
                while ((q = fk_ld_volatile(slot)) < 0) {}
                fk_st_volatile(slot, -1);
            }
            q = gmax_i(q);
            const bool have = q >= 0;
            if (!fk_any(have))
            {
                int d = fk_lane() == 0 ? fk_ld_volatile(A.rr_ctr + 2 * RRK) : 0;
                d = fk_any(d >= A.nbatch) ? 1 : 0;
                if (d) break;                                        // every QP has stopped
                fk_nanosleep(nap);
                if (nap < 128000) nap *= 2;
                continue;
            }
            nap = 4000;
            fk_threadfence();
            if (!have) q = 0;
            bind(q, have);
            cuipm_info *info = A.info + q;
            double *stat = A.stat ? A.stat + (size_t) q * SM * (A.o.stat_max + 1) : nullptr;
            QpState Q;
            LinNrm L;
            int kk = rr_load(q, Q);
            fk_sync();
            iteration(q, kk, Q, L, info, stat);
            kk++;
            { FK_PROF_T0(); res_pass(1, Q.alpha, Q, L); FK_PROF_ADD(0); }
            lin_check(q, kk, L, info, stat);
            close_pass(kk, Q, info, stat);
            rr_publish(q, have, kk, Q);
        }
    }

    // this QP needs a cold path: give it to the generic kernel (which starts from scratch)
    FK_DEV void hand_back(int q, cuipm_info *info)
    {
        if (li == 0)
        {
            info->status = CUIPM_FAST_REDO;
            const int slot = fk_atomic_inc(A.redo_count);
            A.redo_list[slot] = q;
        }
    }
};

// doubles of the per-QP vector pool the sweeps carve out of shared memory (record images + scratch)
inline int vector_pool_doubles(int NX, int NM, int nce, int nbe, int ns2e, int nve)
{
    const int nxe = (NX + 1) & ~1, nme = (NM + 2) & ~1;
    const int img = nve + nxe + 2 * nce;                                  // image of a (ux|g, pi|b, lam|d, t|m) record range
    const int v_res = 2 * img + 2 * nme + (nxe + nme + 2 * nce + 2 * ns2e) + 2 * nbe + nve + 2 * nxe + (nve + nxe + nce);
    const int dd8 = 72 - (2 * nce + 2 * nbe + 2 * ns2e) > 0 ? 72 - (2 * nce + 2 * nbe + 2 * ns2e) : 0;
    const int v_fact = img + 2 * nce + ns2e + 2 * nce + 2 * nbe + 2 * ns2e + dd8 + 2 * nme + nxe + nme + nxe;
    const int v_slv = img + 2 * nce + (2 * nme + nxe + ns2e) + nce + 2 * nce + (nce + ns2e) + 2 * nce + 2 * nbe + ns2e + 2 * nxe;
    const int v_fwd = img + 2 * nce + (2 * nme + nxe + ns2e) + nve + nme + (nce + ns2e) + nve + nxe + nve + 2 * nce + ns2e;
    const int v_init = nve + nce, v_mu = 16 * nce;
    int m = v_res;
    if (v_mu > m) m = v_mu;
    if (v_fact > m) m = v_fact;
    if (v_slv > m) m = v_slv;
    if (v_fwd > m) m = v_fwd;
    if (v_init > m) m = v_init;
    return m + 8;
}

// Shared-memory layout of instance <NX, NU, G> for the shape planned in F: sets F.vsize (vector pool) and F.gstride (doubles
// per QP) and returns the dynamic shared memory of one CTA (one warp) in bytes: the index maps, then the areas of its groups.
// 32 / G groups share a warp; 64-bit shared loads are served per half-warp: a group stride of 8 (mod 16) doubles puts the
// consecutive-row accesses of the two groups of a half-warp on disjoint banks.
template <int NX, int NU, int G>
inline size_t layout(FastArgs &F)
{
    using K = Ker<NX, NU, G>;
    F.vsize = vector_pool_doubles(NX, NX + NU, F.nce, F.nbe, F.ns2e, F.nve);
    int gs = K::MATS + F.vsize;
    while (gs % 16 != 8) gs++;
    F.gstride = gs;
    return sizeof(double) * ((size_t) F.gstride * K::QPW + 2 * (size_t) F.nmaps * F.nbe);
}

}  // namespace fastk
}  // namespace cuipm
#endif
