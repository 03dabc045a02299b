// cuipm_assemble_core.h -- full-shape QP records (the input of the cuipm_xcond_* entries) assembled from strided per-field
// sources, written against an execution policy so that the SAME code runs as the CUDA kernel of cuipm_assemble.cu (a grid-stride
// loop) and, for the CPU tests, sequentially on the host.
//
// The record format is the one of cuipm_layout_create (include/cuipm.h; HPIPM's conventions): BAt = [B'; A'], RSQ with both
// triangles [R S'; S Q] as the host packer writes it, DCt = [D'; C'], rq = [r; q], d = [lbu, lbx, lg, -ubu, -ubx, -ug, lls, lus],
// dmask in the same order, Z = [Zl, Zu], z = [zl, zu], every array padded to an even length with zeros.
//
// The work is ordered by the destination: element t of the batch's records (t = q * qp_stride + i) is computed by one thread
// from the stage and the array i falls into, and written once, padding included.  Consecutive threads write consecutive doubles.
#ifndef CUIPM_ASSEMBLE_CORE_H_
#define CUIPM_ASSEMBLE_CORE_H_

#include <string>
#include <vector>

#include "cuipm.h"

#ifdef __CUDACC__
#define AS_HD __host__ __device__
#else
#define AS_HD
#endif

namespace cuipm_asm {

enum { A_BAT, A_RSQ, A_DCT, A_B, A_RQ, A_D, A_DMASK, A_Z, A_SZ, A_COUNT };   // the arrays of a stage, in record order

struct Stage
{
    unsigned off[A_COUNT + 1];       // record offsets of the stage's arrays; off[A_COUNT] = start of the next stage
    int nu, nx, nxn, nbu, nb, ng, ns;
    int slot[CUIPM_F_COUNT];         // source of (field, this stage): index into Plan::src, or -1 (zeros; masks: ones)
};

struct Src
{
    const double *ptr;
    long long sb, sr, sc;            // strides in doubles: batch, row (element of a vector), column
};

struct Plan
{
    const Stage *st;                 // [N+1]
    const Src *src;
    int N;
    unsigned qp_stride;
    long long total;                 // nbatch * qp_stride
    double *out;
};

// rows x cols of a field at a stage (vectors: cols = 1); 0 x 0 where the field does not exist there
AS_HD inline void field_dims(int f, const Stage &s, int &rows, int &cols)
{
    const int nbx = s.nb - s.nbu;
    cols = 1;
    switch (f)
    {
    case CUIPM_F_A: rows = s.nxn; cols = s.nx; break;
    case CUIPM_F_B: rows = s.nxn; cols = s.nu; break;
    case CUIPM_F_b: rows = s.nxn; break;
    case CUIPM_F_Q: rows = s.nx; cols = s.nx; break;
    case CUIPM_F_R: rows = s.nu; cols = s.nu; break;
    case CUIPM_F_S: rows = s.nu; cols = s.nx; break;
    case CUIPM_F_q: rows = s.nx; break;
    case CUIPM_F_r: rows = s.nu; break;
    case CUIPM_F_lbu: case CUIPM_F_ubu: case CUIPM_F_lbu_mask: case CUIPM_F_ubu_mask: rows = s.nbu; break;
    case CUIPM_F_lbx: case CUIPM_F_ubx: case CUIPM_F_lbx_mask: case CUIPM_F_ubx_mask: rows = nbx; break;
    case CUIPM_F_C: rows = s.ng; cols = s.nx; break;
    case CUIPM_F_D: rows = s.ng; cols = s.nu; break;
    case CUIPM_F_lg: case CUIPM_F_ug: case CUIPM_F_lg_mask: case CUIPM_F_ug_mask: rows = s.ng; break;
    default: rows = s.ns; break;    // Zl, Zu, zl, zu, lls, lus and their masks
    }
    if (rows == 0 || cols == 0) rows = cols = 0;
}

// element (r, c) of QP q's value of the field in `slot` (numpy / torch index order: row r, column c)
AS_HD inline double at(const Plan &P, int slot, long long q, int r, int c, double dflt)
{
    if (slot < 0) return dflt;
    const Src &s = P.src[slot];
    return s.ptr[q * s.sb + r * s.sr + c * s.sc];
}

// the field of piece p of d (lbu, lbx, lg, ubu, ubx, ug, lls, lus) or of dmask (their masks)
AS_HD inline int d_piece_field(int p, bool mask)
{
    switch (p)
    {
    case 0: return mask ? CUIPM_F_lbu_mask : CUIPM_F_lbu;
    case 1: return mask ? CUIPM_F_lbx_mask : CUIPM_F_lbx;
    case 2: return mask ? CUIPM_F_lg_mask : CUIPM_F_lg;
    case 3: return mask ? CUIPM_F_ubu_mask : CUIPM_F_ubu;
    case 4: return mask ? CUIPM_F_ubx_mask : CUIPM_F_ubx;
    case 5: return mask ? CUIPM_F_ug_mask : CUIPM_F_ug;
    case 6: return mask ? CUIPM_F_lls_mask : CUIPM_F_lls;
    default: return mask ? CUIPM_F_lus_mask : CUIPM_F_lus;
    }
}

// double i of QP q's record
AS_HD inline double value(const Plan &P, long long q, unsigned i)
{
    int k = 0, hi = P.N;                                 // the stage: the last one starting at or before i
    while (k < hi)
    {
        const int mid = (k + hi + 1) >> 1;
        if (P.st[mid].off[0] <= i) k = mid; else hi = mid - 1;
    }
    const Stage &s = P.st[k];
    int a = 0;
    while (a < A_COUNT - 1 && s.off[a + 1] <= i) a++;
    const int e = (int) (i - s.off[a]), nu = s.nu, n = nu + s.nx;
    switch (a)
    {
    case A_BAT:                                          // column j = [B(j, :)'; A(j, :)'], ld n
        if (e < n * s.nxn) { const int j = e / n, r = e - j * n; return r < nu ? at(P, s.slot[CUIPM_F_B], q, j, r, 0.0) : at(P, s.slot[CUIPM_F_A], q, j, r - nu, 0.0); }
        break;
    case A_RSQ:                                          // element (r, c) of [R S'; S Q] at c * n + r, both triangles
        if (e < n * n)
        {
            const int c = e / n, r = e - c * n;
            if (c < nu) return r < nu ? at(P, s.slot[CUIPM_F_R], q, c, r, 0.0) : at(P, s.slot[CUIPM_F_S], q, c, r - nu, 0.0);
            return r < nu ? at(P, s.slot[CUIPM_F_S], q, r, c - nu, 0.0) : at(P, s.slot[CUIPM_F_Q], q, c - nu, r - nu, 0.0);
        }
        break;
    case A_DCT:                                          // column g = [D(g, :)'; C(g, :)']
        if (e < n * s.ng) { const int g = e / n, r = e - g * n; return r < nu ? at(P, s.slot[CUIPM_F_D], q, g, r, 0.0) : at(P, s.slot[CUIPM_F_C], q, g, r - nu, 0.0); }
        break;
    case A_B:
        if (e < s.nxn) return at(P, s.slot[CUIPM_F_b], q, e, 0, 0.0);
        break;
    case A_RQ:
        if (e < n) return e < nu ? at(P, s.slot[CUIPM_F_r], q, e, 0, 0.0) : at(P, s.slot[CUIPM_F_q], q, e - nu, 0, 0.0);
        break;
    case A_D: case A_DMASK:                              // pieces lbu, lbx, lg, ubu, ubx, ug, ls, us (no arrays: they would live in local memory)
    {
        const int nbx = s.nb - s.nbu;
        int p = 0, r = e;
        for (; p < 8; p++)
        {
            const int len = p >= 6 ? s.ns : (p % 3 == 0 ? s.nbu : (p % 3 == 1 ? nbx : s.ng));
            if (r < len) break;
            r -= len;
        }
        if (p == 8) break;
        if (a == A_DMASK) return at(P, s.slot[d_piece_field(p, true)], q, r, 0, 1.0);
        const int slot = s.slot[d_piece_field(p, false)];
        if (slot < 0) return 0.0;
        const double v = at(P, slot, q, r, 0, 0.0);
        return (p >= 3 && p < 6) ? -v : v;               // upper bounds stored negated
    }
    case A_Z:
        if (e < 2 * s.ns) return e < s.ns ? at(P, s.slot[CUIPM_F_Zl], q, e, 0, 0.0) : at(P, s.slot[CUIPM_F_Zu], q, e - s.ns, 0, 0.0);
        break;
    default:                                             // z
        if (e < 2 * s.ns) return e < s.ns ? at(P, s.slot[CUIPM_F_zl], q, e, 0, 0.0) : at(P, s.slot[CUIPM_F_zu], q, e - s.ns, 0, 0.0);
        break;
    }
    return 0.0;                                          // padding
}

template <class Exec>
AS_HD void assemble(Exec &ex, const Plan &P)
{
    ex.for_each(P.total, [&](long long t) {
        const long long q = t / P.qp_stride;
        P.out[t] = value(P, q, (unsigned) (t - q * P.qp_stride));
    });
}

}  // namespace cuipm_asm

// ---- host side: the tables the kernel reads ----
namespace cuipm_asm {

// The stage table of a shape and its layout, with no sources; false if the records need offsets beyond 32 bits.
inline bool stage_table(const cuipm_shape *sh, const cuipm_layout *L, std::vector<Stage> &st)
{
    if (L->qp_stride > 0xffffffffu) return false;
    st.assign((size_t) sh->N + 1, Stage{});
    for (int k = 0; k <= sh->N; k++)
    {
        Stage &s = st[k];
        const size_t off[A_COUNT + 1] = {L->off_BAt[k], L->off_RSQ[k], L->off_DCt[k], L->off_b[k], L->off_rq[k], L->off_d[k],
                                         L->off_dmask[k], L->off_Z[k], L->off_z[k], L->qp_stage[k + 1]};
        for (int a = 0; a <= A_COUNT; a++) s.off[a] = (unsigned) off[a];
        s.nu = sh->nu[k]; s.nx = sh->nx[k]; s.nxn = k < sh->N ? sh->nx[k + 1] : 0;
        s.nb = sh->nb[k]; s.ng = sh->ng[k]; s.ns = sh->ns[k];
        s.nbu = 0;                                       // the input bounds come first in idxb (lb = [lbu, lbx])
        for (int j = 0; j < s.nb; j++) s.nbu += sh->idxb[k][j] < s.nu;
        for (int f = 0; f < CUIPM_F_COUNT; f++) s.slot[f] = -1;
    }
    return true;
}

// The stage table `st` (from stage_table) with the sources of one call entered; an empty string, or why the sources are refused.
inline std::string enter_sources(std::vector<Stage> &st, const cuipm_src *src, int nsrc, std::vector<Src> &out)
{
    const int N = (int) st.size() - 1;
    out.clear();
    for (int j = 0; j < nsrc; j++)
    {
        const cuipm_src &c = src[j];
        const std::string at = "source " + std::to_string(j) + " (field " + std::to_string(c.field) + ", stage " + std::to_string(c.stage) + ")";
        if (c.field < 0 || c.field >= CUIPM_F_COUNT) return at + ": no such field";
        if (c.stage < 0 || c.stage > N) return at + ": stage out of range 0.." + std::to_string(N);
        int rows, cols;
        field_dims(c.field, st[c.stage], rows, cols);
        if (rows == 0) return at + ": the field does not exist at this stage";
        if (c.s_batch < 0 || c.s_row < 0 || c.s_col < 0) return at + ": negative stride";
        if (!c.ptr) return at + ": null pointer";
        int &slot = st[c.stage].slot[c.field];
        if (slot >= 0) return at + ": given twice";
        slot = (int) out.size();
        out.push_back(Src{c.ptr, c.s_batch, c.s_row, c.s_col});
    }
    return std::string();
}

}  // namespace cuipm_asm
#endif
