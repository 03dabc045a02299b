// cuipm_condense_core.h -- batched partial (block) condensing and expansion, one CTA per QP, written against an execution
// policy so that the SAME code runs as a CUDA kernel (threads of the CTA, __syncthreads between phases) and, for the tests, as a
// sequential emulation on the host (oracle/condense_emul.cpp: the lanes of a phase one after the other).
//
// Reference: d_part_cond_qp_cond / d_part_cond_qp_expand_sol (external/hpipm/cond/x_part_cond.c:410-866, x_cond_aux.c) behind
// ocp_qp_partial_condensing (acados/ocp_qp/ocp_qp_partial_condensing.c:523-689).  The algorithm is the one of
// acados_b200/condensing.py (which is pinned against the reference): per block, x_j = T_j [u2; x] + c_j with T_j = [Gam_j | Phi_j];
// H2 = sum_j T_j' Q_j T_j + (E_j' S_j T_j + its transpose) + E_j' R_j E_j; dynamics of the block end; input bounds stay boxes, the
// first stage's state bounds stay boxes, inner state bounds / general constraints become general constraints with shifted bounds.
//
// Data parallelism inside a QP: every phase is "thread t handles elements t, t+NT, ... of an output array" (column-major, so
// consecutive threads touch consecutive addresses of the records); the small operands T, c, Q T live in the CTA's scratch
// (shared memory, or the QP's slice of a device buffer where the blocks need more than a block may have: cuipm_condense.cu).
#ifndef CUIPM_CONDENSE_CORE_H_
#define CUIPM_CONDENSE_CORE_H_

#ifdef __CUDACC__
#define CC_HD __host__ __device__
#else
#define CC_HD
#endif

namespace cuipm_cond {

// offsets (doubles) of the per-stage arrays of one layout + the dims of its shape; all arrays live where the executor can read them
struct LayoutTab
{
    int N;
    const int *nx, *nu, *nb, *ng, *ns;
    const int *idxb_ptr, *idxb;               // idxb of stage k: idxb[idxb_ptr[k] .. idxb_ptr[k+1])
    const unsigned *BAt, *RSQ, *DCt, *b, *rq, *d, *dmask, *Z, *z, *ux, *pi, *lam, *t;
    unsigned qp_stride, sol_stride;
};

struct Plan
{
    LayoutTab o, c;                           // original (N stages) and condensed (N2 stages) layouts
    const int *blk_k0, *blk_m;                // first stage and number of stages of block b (b < N2)
    const int *st_offu, *st_offs;             // per original stage: offset of its inputs / slacks inside its block's stage
    const int *box_ptr, *box_stage, *box_i;   // condensed box p of block b (p in box_ptr[b]..box_ptr[b+1]): original (stage, bound index)
    const int *gen_ptr, *gen_stage, *gen_kind, *gen_i;   // condensed general constraint: kind 0 = state bound i of an inner stage, 1 = general constraint i
    int nxmax, n2max;                         // scratch sizing: max of nx and nu over stages, max (nu2 + nx) over blocks
    // lhs / rhs split (condense_lhs / condense_rhs of acados/ocp_qp/ocp_qp_partial_condensing.c:575-630): the matrices T_j =
    // [Gam_j | Phi_j] of every original stage (nx_j x n2 of its block) kept per QP by the lhs pass at t_off[j] of a resident buffer
    // of t_stride doubles per QP, read by the rhs pass
    const unsigned *t_off;
    unsigned t_stride;
};

// what a pass computes: everything; everything + T_j kept (lhs); the vectors only, with the T_j of an earlier lhs pass (rhs)
enum { COND_ALL = 0, COND_LHS = 1, COND_RHS = 2 };

CC_HD inline int scratch_doubles(const Plan &P) { return 2 * P.nxmax * P.n2max + 4 * P.nxmax + 2 * P.n2max + 16; }
// the part of it expand_one uses (xv, xn, pv, pn)
CC_HD inline int expand_scratch_doubles(const Plan &P) { return 4 * P.nxmax; }

// symmetric access to the lower-stored Hessian block of the ORIGINAL record (column-major, ld n)
CC_HD inline double hsym(const double *H, int n, int i, int j) { return i >= j ? H[i + n * j] : H[j + n * i]; }

template <int MODE, class Exec>
CC_HD void condense_one(Exec &ex, const Plan &P, const double *q, double *o, double *scr, double *tbuf)
{
    constexpr bool MAT = MODE != COND_RHS;    // the matrices of the condensed QP are (re)computed
    const LayoutTab &L = P.o, &C = P.c;
    const int NT = ex.nthreads();
    double *T = scr, *T2 = T + P.nxmax * P.n2max, *cv = T2 + P.nxmax * P.n2max, *cv2 = cv + P.nxmax, *qc = cv2 + P.nxmax;
    for (int b = 0; b < C.N; b++)
    {
        const int k0 = P.blk_k0[b], m = P.blk_m[b];
        const int nx0 = C.nx[b], nuu = C.nu[b], n2 = nuu + nx0, nb2 = C.nb[b], ng2 = C.ng[b], ns2 = C.ns[b];
        double *H2 = o + C.RSQ[b], *g2 = o + C.rq[b], *d2 = o + C.d[b], *m2 = o + C.dmask[b];
        // T_0 = [0 | I], c_0 = 0 (T is nx_j x n2, column-major, ld = nx_j); H2, g2 cleared
        ex.phase([&](int t) {
            if (MAT)
            {
                for (int e = t; e < nx0 * n2; e += NT) T[e] = (e / nx0 - nuu == e % nx0) ? 1.0 : 0.0;
                for (int e = t; e < n2 * n2; e += NT) H2[e] = 0.0;
            }
            for (int e = t; e < nx0; e += NT) cv[e] = 0.0;
            for (int e = t; e < n2; e += NT) g2[e] = 0.0;
        });
        int nxj = nx0;
        for (int jj = 0; jj < m; jj++)
        {
            const int j = k0 + jj, nu = L.nu[j], n = nu + nxj, nx1 = L.nx[j + 1], ou = P.st_offu[j];
            const double *Hj = q + L.RSQ[j], *rqj = q + L.rq[j], *BA = q + L.BAt[j], *bj = q + L.b[j];
            // T_j: in the scratch (computed by this pass) or in the resident buffer (rhs pass); the lhs pass keeps it
            const double *Tj = MODE == COND_RHS ? tbuf + P.t_off[j] : T;
            if (MODE == COND_LHS)
                ex.phase([&](int t) { for (int e = t; e < nxj * n2; e += NT) tbuf[P.t_off[j] + e] = T[e]; });
            // T2 = Q_j T (nx_j x n2); qc = Q_j c + q_j
            ex.phase([&](int t) {
                if (MAT)
                for (int e = t; e < nxj * n2; e += NT)
                {
                    const int i = e % nxj, c = e / nxj;
                    double acc = 0.0;
                    for (int l = 0; l < nxj; l++) acc += hsym(Hj, n, nu + i, nu + l) * T[l + nxj * c];
                    T2[e] = acc;
                }
                for (int i = t; i < nxj; i += NT)
                {
                    double acc = rqj[nu + i];
                    for (int l = 0; l < nxj; l++) acc += hsym(Hj, n, nu + i, nu + l) * cv[l];
                    qc[i] = acc;
                }
            });
            // H2 += T' (Q T);  g2 += T' qc
            ex.phase([&](int t) {
                if (MAT)
                for (int e = t; e < n2 * n2; e += NT)
                {
                    const int r = e % n2, c = e / n2;
                    double acc = 0.0;
                    for (int i = 0; i < nxj; i++) acc += T[i + nxj * r] * T2[i + nxj * c];
                    H2[e] += acc;
                }
                for (int r = t; r < n2; r += NT)
                {
                    double acc = 0.0;
                    for (int i = 0; i < nxj; i++) acc += Tj[i + nxj * r] * qc[i];
                    g2[r] += acc;
                }
            });
            // input part: ST = S_j T (nu x n2) added to rows / columns ou.., R_j on the diagonal block, S_j c + r_j on the gradient
            if (nu > 0)
            {
                if (MAT) {
                ex.phase([&](int t) {
                    for (int e = t; e < nu * n2; e += NT)
                    {
                        const int a = e % nu, c = e / nu;
                        double acc = 0.0;
                        for (int l = 0; l < nxj; l++) acc += hsym(Hj, n, a, nu + l) * T[l + nxj * c];     // S_j(a, l) = RSQ(u_a, x_l)
                        T2[e] = acc;                                                                     // T2 reused as ST, ld nu
                    }
                });
                ex.phase([&](int t) {
                    for (int e = t; e < nu * n2; e += NT)
                    {
                        const int a = e % nu, c = e / nu;
                        const double v = T2[e];
                        // row ou+a, column c and its mirror; the two coincide on the diagonal element (added twice there, as
                        // S T + (S T)' prescribes); no two threads share a target inside one of the two passes
                        H2[(ou + a) + n2 * c] += v;
                    }
                });
                ex.phase([&](int t) {
                    for (int e = t; e < nu * n2; e += NT)
                    {
                        const int a = e % nu, c = e / nu;
                        H2[c + n2 * (ou + a)] += T2[e];
                    }
                });
                }
                ex.phase([&](int t) {
                    if (MAT)
                    for (int e = t; e < nu * nu; e += NT)
                    {
                        const int a = e % nu, a2 = e / nu;
                        H2[(ou + a) + n2 * (ou + a2)] += hsym(Hj, n, a, a2);
                    }
                    for (int a = t; a < nu; a += NT)
                    {
                        double acc = rqj[a];
                        for (int l = 0; l < nxj; l++) acc += hsym(Hj, n, a, nu + l) * cv[l];
                        g2[ou + a] += acc;
                    }
                });
            }
            // general constraints of the condensed stage that stem from stage j (rows of T, or C_j T + D_j), with shifted bounds
            if (ng2 > 0)
            {
                double *DC2 = o + C.DCt[b];
                const double *dj = q + L.d[j], *mj = q + L.dmask[j], *DCj = q + L.DCt[j];
                const int nbj = L.nb[j], ngj = L.ng[j];
                for (int p = P.gen_ptr[b]; p < P.gen_ptr[b + 1]; p++)
                {
                    if (P.gen_stage[p] != j) continue;
                    const int pl = p - P.gen_ptr[b], kind = P.gen_kind[p], i = P.gen_i[p];
                    const int xi = kind == 0 ? L.idxb[L.idxb_ptr[j] + i] - nu : 0, pos = kind == 0 ? i : nbj + i;
                    ex.phase([&](int t) {
                        if (MAT)
                        for (int r = t; r < n2; r += NT)
                        {
                            double acc;
                            if (kind == 0) acc = T[xi + nxj * r];
                            else
                            {
                                acc = 0.0;
                                for (int l = 0; l < nxj; l++) acc += DCj[(nu + l) + n * i] * T[l + nxj * r];
                                if (r >= ou && r < ou + nu) acc += DCj[(r - ou) + n * i];
                            }
                            DC2[r + n2 * pl] = acc;
                        }
                        if (t == 0)
                        {
                            double shift;
                            if (kind == 0) shift = cv[xi];
                            else
                            {
                                shift = 0.0;
                                for (int l = 0; l < nxj; l++) shift += DCj[(nu + l) + n * i] * cv[l];
                            }
                            d2[nb2 + pl] = dj[pos] - shift;
                            d2[2 * nb2 + ng2 + pl] = dj[nbj + ngj + pos] + shift;        // upper bounds are stored negated
                            m2[nb2 + pl] = mj[pos];
                            m2[2 * nb2 + ng2 + pl] = mj[nbj + ngj + pos];
                        }
                    });
                }
            }
            // slacks of stage j
            if (L.ns[j] > 0)
            {
                const int ns = L.ns[j], os = P.st_offs[j], nbg = L.nb[j] + L.ng[j];
                const double *dj = q + L.d[j], *mj = q + L.dmask[j], *Zj = q + L.Z[j], *zj = q + L.z[j];
                double *Z2 = o + C.Z[b], *z2 = o + C.z[b];
                ex.phase([&](int t) {
                    for (int e = t; e < 2 * ns; e += NT)
                    {
                        const int half = e / ns, s = e % ns;
                        Z2[half * ns2 + os + s] = Zj[e];
                        z2[half * ns2 + os + s] = zj[e];
                        d2[2 * (nb2 + ng2) + half * ns2 + os + s] = dj[2 * nbg + e];
                        m2[2 * (nb2 + ng2) + half * ns2 + os + s] = mj[2 * nbg + e];
                    }
                });
            }
            // transition: T <- A_j T (+ B_j in the columns of u_j), c <- A_j c + b_j   (BAt_j = [B'; A'], (nu+nx) x nx1, ld n)
            ex.phase([&](int t) {
                if (MAT)
                for (int e = t; e < nx1 * n2; e += NT)
                {
                    const int i = e % nx1, c = e / nx1;
                    double acc = 0.0;
                    for (int l = 0; l < nxj; l++) acc += BA[(nu + l) + n * i] * T[l + nxj * c];
                    if (c >= ou && c < ou + nu) acc += BA[(c - ou) + n * i];
                    T2[e] = acc;
                }
                for (int i = t; i < nx1; i += NT)
                {
                    double acc = bj[i];
                    for (int l = 0; l < nxj; l++) acc += BA[(nu + l) + n * i] * cv[l];
                    cv2[i] = acc;
                }
            });
            ex.phase([&](int t) {
                if (MAT)
                    for (int e = t; e < nx1 * n2; e += NT) T[e] = T2[e];
                for (int i = t; i < nx1; i += NT) cv[i] = cv2[i];
            });
            nxj = nx1;
        }
        // dynamics of the block end: BAt2 = [Gam'; Phi'] = T' ((nu2+nx) x nx1, ld n2), b2 = c; boxes
        {
            double *BA2 = o + C.BAt[b], *b2 = o + C.b[b];
            const int nx1 = nxj;
            ex.phase([&](int t) {
                if (MAT)
                for (int e = t; e < n2 * nx1; e += NT)
                {
                    const int r = e % n2, c = e / n2;
                    BA2[e] = T[c + nx1 * r];
                }
                for (int i = t; i < nx1; i += NT) b2[i] = cv[i];
                for (int p = P.box_ptr[b] + t; p < P.box_ptr[b + 1]; p += NT)
                {
                    const int pl = p - P.box_ptr[b], j = P.box_stage[p], i = P.box_i[p], nbgj = L.nb[j] + L.ng[j];
                    const double *dj = q + L.d[j], *mj = q + L.dmask[j];
                    d2[pl] = dj[i];
                    d2[nb2 + ng2 + pl] = dj[nbgj + i];
                    m2[pl] = mj[i];
                    m2[nb2 + ng2 + pl] = mj[nbgj + i];
                }
            });
        }
    }
    // terminal stage: copied
    {
        const int kN = L.N, k2 = C.N, n = L.nu[kN] + L.nx[kN], ng = L.ng[kN], nc = 2 * (L.nb[kN] + ng + L.ns[kN]), ns2 = 2 * L.ns[kN];
        ex.phase([&](int t) {
            if (MAT)
            {
                for (int e = t; e < n * n; e += NT) o[C.RSQ[k2] + e] = q[L.RSQ[kN] + e];
                for (int e = t; e < n * ng; e += NT) o[C.DCt[k2] + e] = q[L.DCt[kN] + e];
            }
            for (int e = t; e < n; e += NT) o[C.rq[k2] + e] = q[L.rq[kN] + e];
            for (int e = t; e < nc; e += NT) { o[C.d[k2] + e] = q[L.d[kN] + e]; o[C.dmask[k2] + e] = q[L.dmask[kN] + e]; }
            for (int e = t; e < ns2; e += NT) { o[C.Z[k2] + e] = q[L.Z[kN] + e]; o[C.z[k2] + e] = q[L.z[kN] + e]; }
        });
    }
}

// solution of the condensed QP (s2) -> solution of the original QP (s); q: original QP record
template <class Exec>
CC_HD void expand_one(Exec &ex, const Plan &P, const double *q, const double *s2, double *s, double *scr)
{
    const LayoutTab &L = P.o, &C = P.c;
    const int NT = ex.nthreads();
    double *xv = scr, *xn = xv + P.nxmax, *pv = xn + P.nxmax, *pn = pv + P.nxmax;
    for (int b = 0; b < C.N; b++)
    {
        const int k0 = P.blk_k0[b], m = P.blk_m[b];
        const int nx0 = C.nx[b], nuu = C.nu[b], nb2 = C.nb[b], ng2 = C.ng[b], ns2 = C.ns[b];
        const double *ux2 = s2 + C.ux[b], *lam2 = s2 + C.lam[b], *t2 = s2 + C.t[b];
        ex.phase([&](int t) { for (int i = t; i < nx0; i += NT) xv[i] = ux2[nuu + i]; });
        int nxj = nx0;
        for (int jj = 0; jj < m; jj++)
        {
            const int j = k0 + jj, nu = L.nu[j], n = nu + nxj, nx1 = L.nx[j + 1], ou = P.st_offu[j], ns = L.ns[j], os = P.st_offs[j];
            const int nbg = L.nb[j] + L.ng[j];
            const double *BA = q + L.BAt[j], *bj = q + L.b[j];
            double *uxj = s + L.ux[j], *lamj = s + L.lam[j], *tj = s + L.t[j];
            ex.phase([&](int t) {
                for (int a = t; a < nu; a += NT) uxj[a] = ux2[ou + a];
                for (int i = t; i < nxj; i += NT) uxj[nu + i] = xv[i];
                for (int e = t; e < 2 * ns; e += NT)
                {
                    const int half = e / ns, sidx = e % ns;
                    uxj[n + e] = ux2[nuu + nx0 + half * ns2 + os + sidx];
                    lamj[2 * nbg + e] = lam2[2 * (nb2 + ng2) + half * ns2 + os + sidx];
                    tj[2 * nbg + e] = t2[2 * (nb2 + ng2) + half * ns2 + os + sidx];
                }
                for (int i = t; i < nx1; i += NT)
                {
                    double acc = bj[i];
                    for (int l = 0; l < nxj; l++) acc += BA[(nu + l) + n * i] * xv[l];
                    for (int a = 0; a < nu; a++) acc += BA[a + n * i] * ux2[ou + a];
                    xn[i] = acc;
                }
            });
            ex.phase([&](int t) { for (int i = t; i < nx1; i += NT) xv[i] = xn[i]; });
            nxj = nx1;
        }
        // multipliers and slacks of the inequality constraints, by the index maps
        ex.phase([&](int t) {
            for (int p = P.box_ptr[b] + t; p < P.box_ptr[b + 1]; p += NT)
            {
                const int pl = p - P.box_ptr[b], j = P.box_stage[p], i = P.box_i[p], nbgj = L.nb[j] + L.ng[j];
                (s + L.lam[j])[i] = lam2[pl]; (s + L.lam[j])[nbgj + i] = lam2[nb2 + ng2 + pl];
                (s + L.t[j])[i] = t2[pl]; (s + L.t[j])[nbgj + i] = t2[nb2 + ng2 + pl];
            }
            for (int p = P.gen_ptr[b] + t; p < P.gen_ptr[b + 1]; p += NT)
            {
                const int pl = p - P.gen_ptr[b], j = P.gen_stage[p], nbgj = L.nb[j] + L.ng[j];
                const int pos = P.gen_kind[p] == 0 ? P.gen_i[p] : L.nb[j] + P.gen_i[p];
                (s + L.lam[j])[pos] = lam2[nb2 + pl]; (s + L.lam[j])[nbgj + pos] = lam2[2 * nb2 + ng2 + pl];
                (s + L.t[j])[pos] = t2[nb2 + pl]; (s + L.t[j])[nbgj + pos] = t2[2 * nb2 + ng2 + pl];
            }
        });
        // pi of the block end from the condensed QP; inner ones backwards: pi_{j-1} = Q_j x_j + S_j' u_j + q_j + A_j' pi_j + multipliers on x_j
        {
            const int jl = k0 + m - 1, nxe = L.nx[jl + 1];
            const double *pi2 = s2 + C.pi[b];
            ex.phase([&](int t) { for (int i = t; i < nxe; i += NT) { pv[i] = pi2[i]; (s + L.pi[jl])[i] = pi2[i]; } });
        }
        for (int j = k0 + m - 1; j > k0; j--)
        {
            const int nu = L.nu[j], nxj2 = L.nx[j], n = nu + nxj2, nx1 = L.nx[j + 1], nbj = L.nb[j], ngj = L.ng[j];
            const double *Hj = q + L.RSQ[j], *rqj = q + L.rq[j], *BA = q + L.BAt[j], *DCj = q + L.DCt[j];
            const double *uxj = s + L.ux[j], *lamj = s + L.lam[j];
            const int *ib = L.idxb + L.idxb_ptr[j];
            ex.phase([&](int t) {
                for (int i = t; i < nxj2; i += NT)
                {
                    double acc = rqj[nu + i];
                    for (int l = 0; l < n; l++) acc += hsym(Hj, n, nu + i, l) * uxj[l];
                    for (int c = 0; c < nx1; c++) acc += BA[(nu + i) + n * c] * pv[c];
                    for (int p = 0; p < nbj; p++)
                        if (ib[p] == nu + i) acc += lamj[nbj + ngj + p] - lamj[p];
                    for (int g = 0; g < ngj; g++) acc += DCj[(nu + i) + n * g] * (lamj[nbj + ngj + nbj + g] - lamj[nbj + g]);
                    pn[i] = acc;
                }
            });
            ex.phase([&](int t) { for (int i = t; i < nxj2; i += NT) { pv[i] = pn[i]; (s + L.pi[j - 1])[i] = pn[i]; } });
        }
    }
    {
        const int kN = L.N, k2 = C.N, n = L.nu[kN] + L.nx[kN] + 2 * L.ns[kN], nc = 2 * (L.nb[kN] + L.ng[kN] + L.ns[kN]);
        ex.phase([&](int t) {
            for (int e = t; e < n; e += NT) s[L.ux[kN] + e] = s2[C.ux[k2] + e];
            for (int e = t; e < nc; e += NT) { s[L.lam[kN] + e] = s2[C.lam[k2] + e]; s[L.t[kN] + e] = s2[C.t[k2] + e]; }
        });
    }
}

}  // namespace cuipm_cond
#endif
