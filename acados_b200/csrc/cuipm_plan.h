// cuipm_plan.h -- host-side construction of the stage descriptor tables (no CUDA): shared by the solver object
// (cuipm_api.cu) and by the host emulation of the throughput kernel used in the CPU test-suite (oracle/fast_emul.cpp).
#ifndef CUIPM_PLAN_H_
#define CUIPM_PLAN_H_

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "cuipm.h"
#include "cuipm_device.h"

namespace cuipm {

static inline unsigned plan_ev2u(size_t n) { return (unsigned) ((n + 1) & ~(size_t) 1); }

// Fills sd (one descriptor per stage), the index pool and P from the shape and its record layout.
// Returns CUIPM_OK or an error code with a message in err.
inline int build_plan(const cuipm_shape *sh, const cuipm_layout *l, std::vector<StageDesc> &sd, std::vector<int> &ipool, ProbDesc &P,
                      std::string &err)
{
    const int N = sh->N;
    ipool.clear();
    sd.assign(N + 1, StageDesc{});
    P = ProbDesc{};
    P.N = N;
    size_t w = 0;
    for (int k = 0; k <= N; k++)
    {
        StageDesc &d = sd[k];
        d.nx = sh->nx[k]; d.nu = sh->nu[k]; d.n = d.nx + d.nu; d.nb = sh->nb[k]; d.ng = sh->ng[k]; d.ns = sh->ns[k];
        d.nbg = d.nb + d.ng; d.nc = 2 * (d.nbg + d.ns);
        d.nx1 = k < N ? sh->nx[k + 1] : 0; d.nu1 = k < N ? sh->nu[k + 1] : 0; d.n1 = d.nx1 + d.nu1;
        if (d.nx < 0 || d.nu < 0 || d.nb < 0 || d.ng < 0 || d.ns < 0) { err = "negative dimension"; return CUIPM_ERR_INVALID; }
        if (d.ns > 0 && !sh->idxs_rev) { err = "ns>0 needs idxs_rev"; return CUIPM_ERR_INVALID; }
        d.idx_off = (int) ipool.size();
        d.dup_idxb = 0;
        for (int i = 0; i < d.nb; i++)
        {
            const int ix = sh->idxb[k][i];
            if (ix < 0 || ix >= d.n) { err = "idxb out of range"; return CUIPM_ERR_INVALID; }
            for (int j = 0; j < i; j++) d.dup_idxb |= sh->idxb[k][j] == ix;
            ipool.push_back(ix);
        }
        for (int i = 0; i < d.nbg; i++)
        {
            const int r = (d.ns > 0 && sh->idxs_rev) ? sh->idxs_rev[k][i] : -1;
            if (r < -1 || r >= d.ns) { err = "idxs_rev out of range"; return CUIPM_ERR_INVALID; }
            ipool.push_back(r);
        }
        d.q_BAt = (unsigned) l->off_BAt[k]; d.q_RSQ = (unsigned) l->off_RSQ[k]; d.q_DCt = (unsigned) l->off_DCt[k];
        d.q_b = (unsigned) l->off_b[k]; d.q_rq = (unsigned) l->off_rq[k]; d.q_d = (unsigned) l->off_d[k];
        d.q_dmask = (unsigned) l->off_dmask[k]; d.q_Z = (unsigned) l->off_Z[k]; d.q_z = (unsigned) l->off_z[k];
        d.sol = VOff{(unsigned) l->off_ux[k], (unsigned) l->off_pi[k], (unsigned) l->off_lam[k], (unsigned) l->off_t[k]};
        const size_t nvs = (size_t) d.n + 2 * d.ns;
        auto take = [&](size_t n) { unsigned o = (unsigned) w; w += plan_ev2u(n); return o; };
        // factor first (read by two sweeps per solve), then the vectors
        d.q_stage = (unsigned) l->qp_stage[k];
        d.q_stage_bytes = (unsigned) ((l->qp_stage[k + 1] - l->qp_stage[k]) * sizeof(double));
        d.w_fac = (unsigned) w;
        d.w_L = take((size_t) d.n * d.n); d.w_Linv = take(d.n); d.w_lrow = take(d.n); d.w_Pb = take(d.nx1); d.w_Zsi = take(2 * d.ns);
        d.w_Lxx = take((size_t) (d.nx | 1) * d.nx);
        d.w_fac_bytes = (unsigned) ((w - d.w_fac) * sizeof(double));
        d.w_vec = (unsigned) w;
        d.step = VOff{take(nvs), take(d.nx1), take(d.nc), take(d.nc)};
        d.res = ROff{take(nvs), take(d.nx1), take(d.nc), take(d.nc)};
        d.w_rmb = take(d.nc);
        d.ires = ROff{take(nvs), take(d.nx1), take(d.nc), take(d.nc)};
        d.itref = VOff{take(nvs), take(d.nx1), take(d.nc), take(d.nc)};
        d.w_vec_bytes = (unsigned) ((w - d.w_vec) * sizeof(double));
        P.nmax = std::max(P.nmax, d.n); P.nxmax = std::max(P.nxmax, std::max(d.nx, d.nx1)); P.ngmax = std::max(P.ngmax, d.ng);
        P.nsmax = std::max(P.nsmax, d.ns); P.nbgmax = std::max(P.nbgmax, d.nbg); P.ncmax = std::max(P.ncmax, d.nc);
        P.nvsmax = std::max(P.nvsmax, (int) nvs);
        P.nct += d.nc;
    }
    // uniform interior stages? (stages 1..N-1 share (nx, nu); stage N has the same nx) -> compile-time specialised sweeps
    P.mid_nx = P.mid_nu = 0;
    if (N >= 3)
    {
        bool uni = true;
        for (int k = 1; k <= N - 1; k++) uni = uni && sh->nx[k] == sh->nx[1] && sh->nu[k] == sh->nu[1];
        uni = uni && sh->nx[N] == sh->nx[1];
        if (uni) { P.mid_nx = sh->nx[1]; P.mid_nu = sh->nu[1]; }
    }
    P.w_lq = (unsigned) w;
    w += plan_ev2u((size_t) P.nmax * (P.nbgmax + P.nxmax));
    P.w_bkp = (unsigned) w;
    w += plan_ev2u(l->sol_stride);
    if (w >= (size_t) 1 << 32 || l->qp_stride >= (size_t) 1 << 32) { err = "QP record too large for 32-bit offsets"; return CUIPM_ERR_TOO_LARGE; }
    // the stage-block buffers below are indexed with int offsets (on chip or in the scratch slice of one QP)
    if ((size_t) (P.nmax + 2) * ((size_t) P.nmax + P.nxmax + 3 * (size_t) P.ngmax) + 4 * (size_t) P.ncmax + 64 >= (size_t) 1 << 31)
    {
        err = "stage blocks too large for 32-bit offsets";
        return CUIPM_ERR_TOO_LARGE;
    }
    P.qp_stride = l->qp_stride; P.sol_stride = l->sol_stride; P.work_stride = w;
    auto e = [](int n) { return (n + 1) & ~1; };
    // leading dimensions used on chip: nmax|1 (odd, conflict-free row/column access) or even(nmax+1) (factorisation:
    // rows incl. the gradient row, 16-byte aligned column starts); both <= nmax+2
    P.sm_M = e((P.nmax + 2) * P.nmax + 8);                       // factor of the stage being eliminated (rows incl. gradient row)
    P.sm_A = 0;                                                  // (matrices of the substitution / residual sweeps are streamed from global memory)
    P.sm_AL = e(std::max((P.nmax + 2) * (P.nxmax + P.ngmax), e(P.nmax) + e(P.nxmax) + 4 * e(P.ncmax)) + 8);   // [A; b'] -> A L_xx in place (+ general-constraint columns); staging area of the substitution sweeps
    P.sm_C = P.ngmax > 0 ? 2 * e((P.nmax + 2) * P.ngmax) + 8 : 0;
    {
        const int nvs = e(P.nvsmax), nx = e(P.nxmax), nc = e(P.ncmax), nbg = e(P.nbgmax), n = e(P.nmax + 1), ns2 = e(2 * P.nsmax);
        const int v_res = 2 * nvs + 3 * nx + 4 * nc + 2 * nbg;
        const int v_fwd = 2 * nvs + 5 * nx + 4 * nc + 2 * ns2 + nbg;
        const int v_fact = 2 * nc + 2 * nbg + 3 * n + 2 * ns2 + 16;
        const int v_slv = nvs + 2 * nc + 2 * nbg + 2 * ns2 + 3 * nx;
        const int v_init = nvs + nc + e(P.ngmax);
        P.sm_V = std::max(std::max(std::max(v_res, v_fwd), std::max(v_fact, v_slv)), v_init) + 8;
    }
    // whether this fits in shared memory is the device's question (GenericPath::create)
    P.sm_total = P.sm_M + P.sm_A + P.sm_AL + P.sm_C + P.sm_V;
    return CUIPM_OK;
}

// ---- throughput ("fast") path ----------------------------------------------------------------------------------------
// Eligibility: x0 eliminated (nx_0 = 0), the same (nx, nu, nb, ns, index maps' sizes) on stages 1..N-1, nx_N = nx, nu_N = 0,
// no general constraints, no repeated bound index, N >= 3; then every array offset of an interior stage is the offset of
// stage 1 plus (k-1) times a constant stride, and the kernel needs three descriptors only (first, interior, last).
// Fills F (records / pointers are set by the caller); returns false if the shape is not eligible.
inline bool fast_plan(const std::vector<StageDesc> &sd, const std::vector<int> &ipool, const ProbDesc &P, FastArgs &F)
{
    const int N = P.N;
    if (N < 3) return false;
    const StageDesc &a = sd[1];
    if (sd[0].nx != 0 || sd[0].nu != a.nu || sd[N].nu != 0 || sd[N].nx != a.nx || a.nx <= 0 || a.nu <= 0) return false;
    for (int k = 0; k <= N; k++)
        if (sd[k].ng != 0 || sd[k].dup_idxb) return false;
    if (P.nct == 0) return false;
    // affine offsets over the interior stages: compare every unsigned offset field
    const unsigned qs = N >= 3 ? sd[2].q_stage - a.q_stage : 0, ss = N >= 3 ? sd[2].sol.ux - a.sol.ux : 0, ws = N >= 3 ? sd[2].w_fac - a.w_fac : 0;
    const int is = N >= 3 ? sd[2].idx_off - a.idx_off : 0;
    bool same_maps = true;
    for (int k = 1; k <= N - 1; k++)
    {
        const StageDesc &d = sd[k];
        if (d.nx != a.nx || d.nu != a.nu || d.nb != a.nb || d.ns != a.ns) return false;
        for (int i = 0; i < 2 * a.nb; i++)       // one copy of the index maps on chip if the interior stages share them, else one per stage
            if (ipool[d.idx_off + i] != ipool[a.idx_off + i]) same_maps = false;
        const unsigned dq = qs * (unsigned) (k - 1), dsol = ss * (unsigned) (k - 1), dw = ws * (unsigned) (k - 1);
        bool ok = d.idx_off == a.idx_off + is * (k - 1);
        ok = ok && d.q_BAt == a.q_BAt + dq && d.q_RSQ == a.q_RSQ + dq && d.q_b == a.q_b + dq && d.q_rq == a.q_rq + dq && d.q_d == a.q_d + dq
             && d.q_dmask == a.q_dmask + dq && d.q_Z == a.q_Z + dq && d.q_z == a.q_z + dq && d.q_stage == a.q_stage + dq;
        ok = ok && d.sol.ux == a.sol.ux + dsol && d.sol.pi == a.sol.pi + dsol && d.sol.lam == a.sol.lam + dsol && d.sol.t == a.sol.t + dsol;
        ok = ok && d.w_L == a.w_L + dw && d.w_Linv == a.w_Linv + dw && d.w_lrow == a.w_lrow + dw && d.w_Pb == a.w_Pb + dw && d.w_Zsi == a.w_Zsi + dw && d.w_Lxx == a.w_Lxx + dw
             && d.step.ux == a.step.ux + dw && d.step.pi == a.step.pi + dw && d.step.lam == a.step.lam + dw && d.step.t == a.step.t + dw
             && d.res.g == a.res.g + dw && d.res.b == a.res.b + dw && d.res.d == a.res.d + dw && d.res.m == a.res.m + dw && d.w_rmb == a.w_rmb + dw
             && d.ires.g == a.ires.g + dw && d.ires.b == a.ires.b + dw && d.ires.d == a.ires.d + dw
             && d.itref.pi == a.itref.pi + dw && d.itref.lam == a.itref.lam + dw && d.itref.t == a.itref.t + dw;
        if (!ok) return false;
    }
    F.N = N;
    F.nct = P.nct;
    F.nmaps = same_maps ? 3 : N + 1;
    F.s0 = sd[0]; F.s1 = sd[1]; F.sN = sd[N];
    F.qs = qs; F.ss = ss; F.ws = ws; F.is = is;
    F.qp_stride = P.qp_stride; F.sol_stride = P.sol_stride; F.work_stride = P.work_stride; F.w_bkp = P.w_bkp;
    auto e = [](int n) { return (n + 1) & ~1; };
    F.nce = e(P.ncmax); F.nbe = e(P.nbgmax); F.ns2e = e(2 * P.nsmax); F.nve = e(P.nvsmax);
    // kernel-side record: dynamics block with an odd leading dimension >= nu+nx (row and column accesses in shared memory are
    // both bank-conflict free), Hessian as its packed lower triangle (n (n + 1) / 2 doubles) or with the same leading dimension
    const int NM = a.nx + a.nu;
    F.ld = NM | 1;
    F.packed = fast_packed(a.nx, a.nu);
    unsigned o = 0;
    const StageDesc *three[3] = {&sd[0], &sd[1], &sd[N]};
    unsigned size[3];
    for (int t = 0; t < 3; t++)
    {
        const StageDesc &d = *three[t];
        const unsigned szA = (unsigned) e(F.ld * d.nx1), szH = (unsigned) e(F.packed ? d.n * (d.n + 1) / 2 : F.ld * d.n);
        const unsigned szV = (d.q_stage + (unsigned) (d.q_stage_bytes / sizeof(double))) - d.q_b;
        F.kH[t] = szA; F.kV[t] = szA + szH;
        size[t] = szA + szH + (unsigned) e((int) szV);
    }
    F.kq[0] = 0; F.kq[1] = size[0]; F.kqs = size[1]; F.kq[2] = size[0] + (unsigned) (N - 1) * size[1];
    o = F.kq[2] + size[2];
    F.qpk_stride = (size_t) e((int) o);
    return true;
}

// Caller's QP record -> kernel-side QP record of the throughput kernel (host version of the repack pass; the device version is
// in cuipm_fast.cu): dynamics block with leading dimension F.ld, the lower triangle of the Hessian packed column by column
// (fastk::tri) if F.packed, else the full symmetric matrix with leading dimension F.ld, the vector part verbatim.
inline void repack_host(const FastArgs &F, const std::vector<StageDesc> &sd, const double *qp, double *qpk)
{
    const int N = F.N, ld = F.ld;
    for (int k = 0; k <= N; k++)
    {
        const StageDesc &d = sd[k];
        const int kind = k == 0 ? 0 : (k == N ? 2 : 1);
        double *o = qpk + F.kq[kind] + (kind == 1 ? (size_t) (k - 1) * F.kqs : 0);
        for (int c = 0; c < d.nx1; c++)
            for (int r = 0; r < d.n; r++) o[r + ld * c] = qp[d.q_BAt + r + d.n * c];
        double *H = o + F.kH[kind];
        if (F.packed)
            for (int j = 0, p = 0; j < d.n; j++)
                for (int i = j; i < d.n; i++) H[p++] = qp[d.q_RSQ + i + d.n * j];
        else
            for (int j = 0; j < d.n; j++)
                for (int i = 0; i < d.n; i++) H[i + ld * j] = i >= j ? qp[d.q_RSQ + i + d.n * j] : qp[d.q_RSQ + j + d.n * i];
        const unsigned nv = d.q_stage + (unsigned) (d.q_stage_bytes / sizeof(double)) - d.q_b;
        for (unsigned i = 0; i < nv; i++) o[F.kV[kind] + i] = qp[d.q_b + i];
    }
}

}  // namespace cuipm
#endif
