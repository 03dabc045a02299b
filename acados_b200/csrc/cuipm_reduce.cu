// cuipm_reduce.cu -- stage-0 equality elimination and restore for a whole batch, on the device.
//
// Reference: d_ocp_qp_reduce_eq_dof (external/hpipm/ocp_qp/x_ocp_qp_red.c:278-560) and d_ocp_qp_restore_eq_dof (:848-994), which
// acados runs in front of / behind every QP solve through ocp_qp_partial_condensing (acados/ocp_qp/ocp_qp_partial_condensing.c:
// 523-689); with the default N2 = N they are ALL that module does.  The state bounds of stage 0 marked as equalities
// (x0 = lbx_0) leave the QP: b_0 += A_0[:,E] x_E, r/q += H[:,E] x_E, lg/ug -= C_0[:,E] x_E, the rows / columns / bounds of the
// eliminated states are dropped; afterwards x_E is put back and the multipliers of the dropped bounds are recovered from the
// stationarity residual of the original stage 0.  Stages 1..N are copied.
//
// One CTA per QP; records in, records out (layouts of the full and of the reduced shape); everything is HBM-bound copy work
// with a few short dot products, so the only design rule is coalescing: thread t handles element t of the destination array.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "cuipm.h"
#include "cuipm_internal.h"

using namespace cuipm;

namespace {

struct RedDesc
{
    // stage-0 dimensions of the full and of the reduced QP
    int nu, nx_f, nx_r, n_f, n_r, nb_f, nb_r, ng, ns, nx1, ne;
    int pad_;
    // offsets (doubles) of the stage-0 arrays in the full (f_) and reduced (r_) QP / solution records
    unsigned f_BAt, f_RSQ, f_DCt, f_b, f_rq, f_d, f_dmask, f_Z, f_z, f_ux, f_pi, f_lam, f_t;
    unsigned r_BAt, r_RSQ, r_DCt, r_b, r_rq, r_d, r_dmask, r_Z, r_z, r_ux, r_pi, r_lam, r_t;
    // stages 1..N: one contiguous block each, same length in both layouts
    unsigned f_qp1, r_qp1, qp_tail, f_sol1, r_sol1, sol_tail;
    size_t f_qp_stride, r_qp_stride, f_sol_stride, r_sol_stride;
    // index tables (device): keep[n_r] variable kept at reduced position i; elim[ne] eliminated variable; elim_b[ne] its bound;
    // keep_b[nb_r] bound kept at reduced position i; idxb_f[nb_f]
    const int *keep, *elim, *elim_b, *keep_b, *idxb_f;
};

__device__ __forceinline__ double sym(const double *H, int n, int i, int j) { return i >= j ? H[i + n * j] : H[j + n * i]; }

__global__ void reduce_kernel(RedDesc D, const double *qf_all, double *qr_all, int nbatch)
{
    const int q = blockIdx.x, t = threadIdx.x, NT = blockDim.x;
    if (q >= nbatch) return;
    const double *qf = qf_all + (size_t) q * D.f_qp_stride;
    double *qr = qr_all + (size_t) q * D.r_qp_stride;
    extern __shared__ double xe[];   // values of the eliminated states
    for (int e = t; e < D.ne; e += NT) xe[e] = qf[D.f_d + D.elim_b[e]];
    // stages 1..N
    for (unsigned i = t; i < D.qp_tail; i += NT) qr[D.r_qp1 + i] = qf[D.f_qp1 + i];
    __syncthreads();
    const int n_f = D.n_f, n_r = D.n_r, nx1 = D.nx1, ng = D.ng, nb_f = D.nb_f, nb_r = D.nb_r, ns = D.ns, ne = D.ne;
    // dynamics
    for (int i = t; i < n_r * nx1; i += NT)
    {
        const int r = i % n_r, c = i / n_r;
        qr[D.r_BAt + i] = qf[D.f_BAt + D.keep[r] + n_f * c];
    }
    for (int j = t; j < nx1; j += NT)
    {
        double acc = qf[D.f_b + j];
        for (int e = 0; e < ne; e++) acc += qf[D.f_BAt + D.elim[e] + n_f * j] * xe[e];
        qr[D.r_b + j] = acc;
    }
    // cost: the record holds the full symmetric block
    const double *H = qf + D.f_RSQ;
    for (int i = t; i < n_r * n_r; i += NT)
    {
        const int r = i % n_r, c = i / n_r;
        qr[D.r_RSQ + i] = sym(H, n_f, D.keep[r], D.keep[c]);
    }
    for (int i = t; i < n_r; i += NT)
    {
        double acc = qf[D.f_rq + D.keep[i]];
        for (int e = 0; e < ne; e++) acc += sym(H, n_f, D.keep[i], D.elim[e]) * xe[e];
        qr[D.r_rq + i] = acc;
    }
    // general constraints
    for (int i = t; i < n_r * ng; i += NT)
    {
        const int r = i % n_r, c = i / n_r;
        qr[D.r_DCt + i] = qf[D.f_DCt + D.keep[r] + n_f * c];
    }
    // bounds: d = [lb, lg, -ub, -ug, lls, lus]
    for (int i = t; i < nb_r; i += NT)
    {
        const int b = D.keep_b[i];
        qr[D.r_d + i] = qf[D.f_d + b];
        qr[D.r_d + nb_r + ng + i] = qf[D.f_d + nb_f + ng + b];
        qr[D.r_dmask + i] = qf[D.f_dmask + b];
        qr[D.r_dmask + nb_r + ng + i] = qf[D.f_dmask + nb_f + ng + b];
    }
    for (int g = t; g < ng; g += NT)
    {
        double cx = 0.0;
        for (int e = 0; e < ne; e++) cx += qf[D.f_DCt + D.elim[e] + n_f * g] * xe[e];
        qr[D.r_d + nb_r + g] = qf[D.f_d + nb_f + g] - cx;
        qr[D.r_d + 2 * nb_r + ng + g] = qf[D.f_d + 2 * nb_f + ng + g] + cx;     // upper bounds are stored negated
        qr[D.r_dmask + nb_r + g] = qf[D.f_dmask + nb_f + g];
        qr[D.r_dmask + 2 * nb_r + ng + g] = qf[D.f_dmask + 2 * nb_f + ng + g];
    }
    for (int j = t; j < 2 * ns; j += NT)
    {
        qr[D.r_d + 2 * (nb_r + ng) + j] = qf[D.f_d + 2 * (nb_f + ng) + j];
        qr[D.r_dmask + 2 * (nb_r + ng) + j] = qf[D.f_dmask + 2 * (nb_f + ng) + j];
        qr[D.r_Z + j] = qf[D.f_Z + j];
        qr[D.r_z + j] = qf[D.f_z + j];
    }
}

__global__ void restore_kernel(RedDesc D, const double *qf_all, const double *sr_all, double *sf_all, int nbatch, double lam_min,
                               double t_min)
{
    const int q = blockIdx.x, t = threadIdx.x, NT = blockDim.x;
    if (q >= nbatch) return;
    const double *qf = qf_all + (size_t) q * D.f_qp_stride;
    const double *sr = sr_all + (size_t) q * D.r_sol_stride;
    double *sf = sf_all + (size_t) q * D.f_sol_stride;
    extern __shared__ double sh[];
    const int n_f = D.n_f, n_r = D.n_r, nx1 = D.nx1, ng = D.ng, nb_f = D.nb_f, nb_r = D.nb_r, ns = D.ns, ne = D.ne;
    double *v = sh, *dl = sh + n_f;          // v: full stage-0 primal; dl: (upper - lower) multipliers of all hard constraints
    for (unsigned i = t; i < D.sol_tail; i += NT) sf[D.f_sol1 + i] = sr[D.r_sol1 + i];
    for (int i = t; i < n_r; i += NT) v[D.keep[i]] = sr[D.r_ux + i];
    for (int e = t; e < ne; e += NT) v[D.elim[e]] = qf[D.f_d + D.elim_b[e]];
    for (int j = t; j < 2 * ns; j += NT) sf[D.f_ux + n_f + j] = sr[D.r_ux + n_r + j];
    for (int j = t; j < nx1; j += NT) sf[D.f_pi + j] = sr[D.r_pi + j];
    // multipliers and slacks of the constraints that stayed; lam_min / t_min on the eliminated bounds (x_ocp_qp_red.c:923-947)
    for (int i = t; i < 2 * (nb_f + ng + ns); i += NT) { sf[D.f_lam + i] = lam_min; sf[D.f_t + i] = t_min; }
    __syncthreads();
    for (int i = t; i < nb_r; i += NT)
    {
        const int b = D.keep_b[i];
        sf[D.f_lam + b] = sr[D.r_lam + i];
        sf[D.f_lam + nb_f + ng + b] = sr[D.r_lam + nb_r + ng + i];
        sf[D.f_t + b] = sr[D.r_t + i];
        sf[D.f_t + nb_f + ng + b] = sr[D.r_t + nb_r + ng + i];
    }
    for (int g = t; g < ng; g += NT)
    {
        sf[D.f_lam + nb_f + g] = sr[D.r_lam + nb_r + g];
        sf[D.f_lam + 2 * nb_f + ng + g] = sr[D.r_lam + 2 * nb_r + ng + g];
        sf[D.f_t + nb_f + g] = sr[D.r_t + nb_r + g];
        sf[D.f_t + 2 * nb_f + ng + g] = sr[D.r_t + 2 * nb_r + ng + g];
    }
    for (int j = t; j < 2 * ns; j += NT)
    {
        sf[D.f_lam + 2 * (nb_f + ng) + j] = sr[D.r_lam + 2 * (nb_r + ng) + j];
        sf[D.f_t + 2 * (nb_f + ng) + j] = sr[D.r_t + 2 * (nb_r + ng) + j];
    }
    for (int i = t; i < n_f; i += NT) sf[D.f_ux + i] = v[i];
    __syncthreads();
    for (int i = t; i < nb_f + ng; i += NT) dl[i] = sf[D.f_lam + nb_f + ng + i] - sf[D.f_lam + i];
    __syncthreads();
    // stationarity residual of the ORIGINAL stage 0 in the eliminated rows = multiplier of the dropped bound (:948-966)
    const double *H = qf + D.f_RSQ;
    for (int e = t; e < ne; e += NT)
    {
        const int i = D.elim[e];
        double acc = qf[D.f_rq + i];
        for (int j = 0; j < n_f; j++) acc += sym(H, n_f, i, j) * v[j];
        for (int j = 0; j < nx1; j++) acc += qf[D.f_BAt + i + n_f * j] * sr[D.r_pi + j];
        for (int b = 0; b < nb_f; b++)
            if (D.idxb_f[b] == i) acc += dl[b];
        for (int g = 0; g < ng; g++) acc += qf[D.f_DCt + i + n_f * g] * dl[nb_f + g];
        const int b = D.elim_b[e];
        sf[D.f_lam + b] = acc >= 0.0 ? acc : lam_min;
        sf[D.f_lam + nb_f + ng + b] = acc >= 0.0 ? lam_min : -acc;
    }
}

}  // namespace

struct cuipm_reducer
{
    int device = 0;
    cuipm_layout *lf = nullptr, *lr = nullptr;
    RedDesc D{};
    int *d_tab = nullptr;
    // reduced shape handed back to the caller (arrays owned here)
    std::vector<int> nx, nu, nb, ng, ns;
    std::vector<std::vector<int>> idxb, rev;
    std::vector<const int *> pidxb, prev;
    cuipm_shape red{};
};

extern "C" void cuipm_reducer_destroy(cuipm_reducer *r)
{
    if (!r) return;
    cudaSetDevice(r->device);
    cudaFree(r->d_tab);
    cuipm_layout_destroy(r->lf);
    cuipm_layout_destroy(r->lr);
    delete r;
}

extern "C" cuipm_reducer *cuipm_reducer_create(const cuipm_shape *full, int nbxe0, const int *idxe0, int device)
{
    if (!full || full->N < 0 || nbxe0 < 0 || (nbxe0 > 0 && !idxe0)) { set_error("cuipm_reducer_create: bad arguments"); return nullptr; }
    const int N = full->N, nu0 = full->nu[0], nx0 = full->nx[0], nb0 = full->nb[0], ng0 = full->ng[0], ns0 = full->ns[0];
    std::vector<char> is_elim_var(nu0 + nx0, 0), is_elim_b(nb0, 0);
    std::vector<int> elim, elim_b;
    for (int e = 0; e < nbxe0; e++)
    {
        const int b = idxe0[e];
        if (b < 0 || b >= nb0) { set_error("idxe out of range"); return nullptr; }
        const int var = full->idxb[0][b];
        if (var < nu0) { set_error("only state bounds can be marked as equalities (as in the reference's Python interface)"); return nullptr; }
        if (full->idxs_rev && ns0 > 0 && full->idxs_rev[0][b] >= 0) { set_error("a softened bound cannot be an equality"); return nullptr; }
        if (is_elim_var[var]) { set_error("two equalities on the same state"); return nullptr; }
        is_elim_var[var] = 1; is_elim_b[b] = 1;
        elim.push_back(var); elim_b.push_back(b);
    }
    cuipm_reducer *r = new cuipm_reducer();
    r->device = device;
    std::vector<int> keep, keep_b, remap(nu0 + nx0, -1);
    for (int i = 0; i < nu0 + nx0; i++)
        if (!is_elim_var[i]) { remap[i] = (int) keep.size(); keep.push_back(i); }
    for (int b = 0; b < nb0; b++)
        if (!is_elim_b[b])
        {
            if (remap[full->idxb[0][b]] < 0) { set_error("a second bound on an eliminated state"); delete r; return nullptr; }
            keep_b.push_back(b);
        }
    // reduced shape
    r->nx.assign(full->nx, full->nx + N + 1); r->nu.assign(full->nu, full->nu + N + 1); r->nb.assign(full->nb, full->nb + N + 1);
    r->ng.assign(full->ng, full->ng + N + 1); r->ns.assign(full->ns, full->ns + N + 1);
    r->nx[0] = nx0 - nbxe0; r->nb[0] = (int) keep_b.size();
    r->idxb.resize(N + 1); r->rev.resize(N + 1);
    for (int k = 0; k <= N; k++)
    {
        if (k == 0)
        {
            for (int b : keep_b) r->idxb[0].push_back(remap[full->idxb[0][b]]);
            for (int b : keep_b) r->rev[0].push_back(full->idxs_rev && ns0 > 0 ? full->idxs_rev[0][b] : -1);
            for (int g = 0; g < ng0; g++) r->rev[0].push_back(full->idxs_rev && ns0 > 0 ? full->idxs_rev[0][nb0 + g] : -1);
        }
        else
        {
            r->idxb[k].assign(full->idxb[k], full->idxb[k] + full->nb[k]);
            for (int i = 0; i < full->nb[k] + full->ng[k]; i++) r->rev[k].push_back(full->idxs_rev && full->ns[k] > 0 ? full->idxs_rev[k][i] : -1);
        }
        if (r->idxb[k].empty()) r->idxb[k].push_back(0);
        if (r->rev[k].empty()) r->rev[k].push_back(-1);
    }
    for (int k = 0; k <= N; k++) { r->pidxb.push_back(r->idxb[k].data()); r->prev.push_back(r->rev[k].data()); }
    r->red = cuipm_shape{N, r->nx.data(), r->nu.data(), r->nb.data(), r->ng.data(), r->ns.data(), r->pidxb.data(), r->prev.data()};
    r->lf = cuipm_layout_create(full);
    r->lr = cuipm_layout_create(&r->red);
    const cuipm_layout *lf = r->lf, *lr = r->lr;
    if (lf->qp_stride >= ((size_t) 1 << 32) || lf->sol_stride >= ((size_t) 1 << 32))
    {
        set_error("QP record too large for 32-bit offsets");
        cuipm_reducer_destroy(r);
        return nullptr;
    }
    RedDesc &D = r->D;
    D.nu = nu0; D.nx_f = nx0; D.nx_r = r->nx[0]; D.n_f = nu0 + nx0; D.n_r = nu0 + r->nx[0]; D.nb_f = nb0; D.nb_r = r->nb[0];
    D.ng = ng0; D.ns = ns0; D.nx1 = N > 0 ? full->nx[1] : 0; D.ne = nbxe0;
    D.f_BAt = (unsigned) lf->off_BAt[0]; D.f_RSQ = (unsigned) lf->off_RSQ[0]; D.f_DCt = (unsigned) lf->off_DCt[0]; D.f_b = (unsigned) lf->off_b[0];
    D.f_rq = (unsigned) lf->off_rq[0]; D.f_d = (unsigned) lf->off_d[0]; D.f_dmask = (unsigned) lf->off_dmask[0]; D.f_Z = (unsigned) lf->off_Z[0];
    D.f_z = (unsigned) lf->off_z[0]; D.f_ux = (unsigned) lf->off_ux[0]; D.f_pi = (unsigned) lf->off_pi[0]; D.f_lam = (unsigned) lf->off_lam[0];
    D.f_t = (unsigned) lf->off_t[0];
    D.r_BAt = (unsigned) lr->off_BAt[0]; D.r_RSQ = (unsigned) lr->off_RSQ[0]; D.r_DCt = (unsigned) lr->off_DCt[0]; D.r_b = (unsigned) lr->off_b[0];
    D.r_rq = (unsigned) lr->off_rq[0]; D.r_d = (unsigned) lr->off_d[0]; D.r_dmask = (unsigned) lr->off_dmask[0]; D.r_Z = (unsigned) lr->off_Z[0];
    D.r_z = (unsigned) lr->off_z[0]; D.r_ux = (unsigned) lr->off_ux[0]; D.r_pi = (unsigned) lr->off_pi[0]; D.r_lam = (unsigned) lr->off_lam[0];
    D.r_t = (unsigned) lr->off_t[0];
    D.f_qp1 = (unsigned) lf->qp_stage[N > 0 ? 1 : N + 1]; D.r_qp1 = (unsigned) lr->qp_stage[N > 0 ? 1 : N + 1];
    D.qp_tail = (unsigned) (lf->qp_stride - D.f_qp1);
    D.f_sol1 = (unsigned) lf->sol_stage[N > 0 ? 1 : N + 1]; D.r_sol1 = (unsigned) lr->sol_stage[N > 0 ? 1 : N + 1];
    D.sol_tail = (unsigned) (lf->sol_stride - D.f_sol1);
    D.f_qp_stride = lf->qp_stride; D.r_qp_stride = lr->qp_stride; D.f_sol_stride = lf->sol_stride; D.r_sol_stride = lr->sol_stride;
    if (lr->qp_stride - D.r_qp1 != D.qp_tail || lr->sol_stride - D.r_sol1 != D.sol_tail) { set_error("internal: tail mismatch"); cuipm_reducer_destroy(r); return nullptr; }
    // device tables
    std::vector<int> tab;
    auto put = [&](const std::vector<int> &v) { size_t o = tab.size(); tab.insert(tab.end(), v.begin(), v.end()); if (tab.size() & 1) tab.push_back(0); return o; };
    std::vector<int> idxbf(full->idxb[0], full->idxb[0] + nb0);
    const size_t o_keep = put(keep), o_elim = put(elim), o_elim_b = put(elim_b), o_keep_b = put(keep_b), o_idxb = put(idxbf);
    tab.push_back(0);
    if (cudaSetDevice(device) != cudaSuccess || cudaMalloc(&r->d_tab, sizeof(int) * tab.size()) != cudaSuccess
        || cudaMemcpy(r->d_tab, tab.data(), sizeof(int) * tab.size(), cudaMemcpyHostToDevice) != cudaSuccess)
    {
        set_error("cuipm_reducer_create: CUDA allocation failed (no CPU fallback)");
        cuipm_reducer_destroy(r);
        return nullptr;
    }
    D.keep = r->d_tab + o_keep; D.elim = r->d_tab + o_elim; D.elim_b = r->d_tab + o_elim_b; D.keep_b = r->d_tab + o_keep_b; D.idxb_f = r->d_tab + o_idxb;
    return r;
}

extern "C" const cuipm_shape *cuipm_reducer_reduced_shape(const cuipm_reducer *r) { return r ? &r->red : nullptr; }
extern "C" const cuipm_layout *cuipm_reducer_full_layout(const cuipm_reducer *r) { return r ? r->lf : nullptr; }
extern "C" const cuipm_layout *cuipm_reducer_reduced_layout(const cuipm_reducer *r) { return r ? r->lr : nullptr; }

extern "C" int cuipm_reduce_device(cuipm_reducer *r, int nbatch, const double *d_qp_full, double *d_qp_red, void *stream)
{
    if (!r || nbatch < 0 || !d_qp_full || !d_qp_red) { set_error("cuipm_reduce_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(r->device));
    reduce_kernel<<<nbatch, 128, sizeof(double) * (r->D.ne + 2), (cudaStream_t) stream>>>(r->D, d_qp_full, d_qp_red, nbatch);
    CK(cudaGetLastError());
    return CUIPM_OK;
}

extern "C" int cuipm_restore_device(cuipm_reducer *r, int nbatch, const double *d_qp_full, const double *d_sol_red, double *d_sol_full,
                                    double lam_min, double t_min, void *stream)
{
    if (!r || nbatch < 0 || !d_qp_full || !d_sol_red || !d_sol_full) { set_error("cuipm_restore_device: bad arguments"); return CUIPM_ERR_INVALID; }
    if (nbatch == 0) return CUIPM_OK;
    CK(cudaSetDevice(r->device));
    const size_t sm = sizeof(double) * (r->D.n_f + r->D.nb_f + r->D.ng + 4);
    restore_kernel<<<nbatch, 128, sm, (cudaStream_t) stream>>>(r->D, d_qp_full, d_sol_red, d_sol_full, nbatch, lam_min, t_min);
    CK(cudaGetLastError());
    return CUIPM_OK;
}
