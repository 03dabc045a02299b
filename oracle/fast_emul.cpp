// fast_emul.cpp -- TEST INFRASTRUCTURE ONLY: runs the body of the product's throughput kernel
// (acados_b200/csrc/cuipm_fast_core.h) on a host emulation of a warp (simt_emul.h), so that the CPU test-suite can
// compare the kernel's arithmetic, index maps and barrier placement with the oracle on a machine without a GPU
// (tests/test_fast_emul.py).  The GPU suite then confirms the same body as compiled by nvcc.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "simt_emul.h"

#define FK_DEV inline
static inline int fk_lane() { return simt::lane(); }
static inline void fk_sync() { simt::sync(); }
static inline double fk_shfl_xor(double v, int m) { return simt::shfl(v, simt::lane() ^ m); }
static inline int fk_shfl_xor_i(int v, int m) { return simt::shfl_i(v, simt::lane() ^ m); }
static inline bool fk_any(bool p) { return simt::ballot(p) != 0u; }
static inline void fk_cp16(double *dst, const double *src)
{
    if (((size_t) dst & 15) || ((size_t) src & 15)) { std::fprintf(stderr, "fast_emul: misaligned 16-byte copy\n"); std::abort(); }
    simt::cp_async(dst, src, 16);
}
static inline void fk_cp_wait() { simt::cp_wait(); }
typedef simt::MBar fk_mbar_t;
static inline void fk_mbar_init(fk_mbar_t *b, int count) { simt::mbar_init(b, count); }
static inline void fk_bulk(double *dst, const double *src, unsigned bytes, fk_mbar_t *b) { simt::bulk_copy(b, dst, src, (int) bytes); }
static inline void fk_mbar_arrive_tx(fk_mbar_t *b, unsigned bytes) { simt::mbar_arrive_tx(b, (int) bytes); }
static inline void fk_mbar_wait(fk_mbar_t *b, unsigned parity) { simt::mbar_wait(b, (int) parity); }
static inline void fk_fence_async() {}
static inline void fk_fence_async_global() {}
static inline double fk_ldg(const double *p) { return *p; }
struct fk_double2 { double x, y; };
static inline fk_double2 fk_ld2(const double *p)
{
    if ((size_t) p & 15) { std::fprintf(stderr, "fast_emul: misaligned 16-byte load\n"); std::abort(); }
    return fk_double2{p[0], p[1]};
}
static inline void fk_dmma(double &c0, double &c1, double a, double b) { simt::dmma(c0, c1, a, b); }
static inline double fk_rsqrt(double x) { return 1.0 / std::sqrt(x); }
static inline int fk_atomic_inc(int *p) { return (*p)++; }
static inline int fk_atomic_add(int *p, int v) { const int o = *p; *p += v; return o; }
static inline int fk_atomic_cas(int *p, int cmp, int v) { const int o = *p; if (o == cmp) *p = v; return o; }
static inline int fk_ld_volatile(const int *p) { return *p; }
static inline void fk_st_volatile(int *p, int v) { *p = v; }
static inline void fk_threadfence() {}
static inline void fk_nanosleep(unsigned) {}
using std::fabs;
using std::fmax;
using std::fmin;
using std::sqrt;

#include "cuipm_fast_core.h"
#include "cuipm_plan.h"

namespace {

int g_rr = 0;      // 1: iteration-sliced scheduling (rr_first for every warp, then rr_loop)

template <int NX, int NU, int G>
int run(cuipm::FastArgs F, int order)
{
    using K = cuipm::fastk::Ker<NX, NU, G>;
    std::vector<double> smem(cuipm::fastk::layout<NX, NU, G>(F) / sizeof(double) + 64);
    // 16-byte aligned base
    double *base = smem.data();
    while ((size_t) base & 15) base++;
    const int nwarp = (F.nbatch + K::QPW - 1) / K::QPW;
    std::vector<double> rr_state((size_t) 12 * F.nbatch, std::nan(""));
    std::vector<int> rr_ring((size_t) CUIPM_RR_RINGS * F.nbatch, -1), rr_ctr(CUIPM_RR_CTR, 0);
    F.rr_state = rr_state.data(); F.rr_ring = rr_ring.data(); F.rr_ctr = rr_ctr.data();
    for (int w = 0; w < nwarp; w++)
    {
        for (double &x : smem) x = std::nan("");      // uninitialised shared memory
        simt::MBar bar;
        simt::run_warp([&]() {
            K k(F, base, &bar);
            if (g_rr) k.rr_first(w * K::QPW);
            else k.run(w * K::QPW);
        }, order);
    }
    if (g_rr)
        // the warps of the second launch run one after the other here: the first one finds the whole ring and works it off alone
        // (pops of an empty ring with QPs alive cannot occur), the others see every QP stopped
        for (int w = 0; w < (nwarp < 3 ? nwarp : 3); w++)
        {
            for (double &x : smem) x = std::nan("");
            simt::MBar bar;
            simt::run_warp([&]() {
                K k(F, base, &bar);
                k.rr_loop();
            }, order);
        }
    return 0;
}

}  // namespace

extern "C" void fast_emul_set_rr(int on) { g_rr = on; }

// Solves nbatch QPs of `shape` (records in the layout of cuipm_layout_create) with the throughput kernel body; QPs the
// kernel hands back are listed in redo[0..*nredo) and keep status CUIPM_FAST_REDO.  g = lanes per QP.
// Returns 0, -1 if the shape is not eligible, -2 if no instance for (nx, nu, g) is compiled in.
extern "C" int fast_emul_solve(const cuipm_shape *sh, int nbatch, const double *qp, double *sol, cuipm_info *info, double *stat,
                               const cuipm_opts *opts, int g, int order, int *redo, int *nredo)
{
    cuipm_layout *l = cuipm_layout_create(sh);
    std::vector<cuipm::StageDesc> sd;
    std::vector<int> ipool;
    cuipm::ProbDesc P;
    std::string err;
    if (cuipm::build_plan(sh, l, sd, ipool, P, err) != CUIPM_OK) { cuipm_layout_destroy(l); return -3; }
    cuipm::FastArgs F{};
    if (!cuipm::fast_plan(sd, ipool, P, F)) { cuipm_layout_destroy(l); return -1; }
    std::vector<double> work((size_t) P.work_stride * nbatch, 0.0);
    ipool.push_back(0);
    F.nbatch = nbatch;
    F.ipool = ipool.data(); F.qp = qp; F.sol = sol; F.work = work.data(); F.info = info; F.stat = stat;
    F.redo_list = redo; F.redo_count = nredo; F.o = *opts;
    *nredo = 0;
    std::vector<double> qpk((size_t) F.qpk_stride * nbatch, 0.0);
    for (int i = 0; i < nbatch; i++) cuipm::repack_host(F, sd, qp + (size_t) i * P.qp_stride, qpk.data() + (size_t) i * F.qpk_stride);
    F.qpk = qpk.data();
    const int nx = F.s1.nx, nu = F.s1.nu;
    int rc = -2;
#define INST(NX_, NU_, G_) if (nx == NX_ && nu == NU_ && g == G_) rc = run<NX_, NU_, G_>(F, order);
    INST(21, 3, 8) INST(21, 3, 16) INST(21, 3, 32)
    INST(8, 3, 4) INST(8, 3, 8) INST(8, 3, 16)
    INST(4, 1, 2) INST(4, 1, 4) INST(4, 1, 8)
    INST(12, 4, 8) INST(12, 4, 16)
    INST(5, 2, 4) INST(6, 2, 8)
    INST(48, 12, 32)
#undef INST
    cuipm_layout_destroy(l);
    return rc;
}
