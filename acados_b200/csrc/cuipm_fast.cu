// cuipm_fast.cu -- CUDA instantiation (sm_90a) of the throughput kernel of the batched OCP-QP interior-point solver.
//
// The kernel body is cuipm_fast_core.h (a group of G lanes per QP, 32/G QPs per warp in lock step, register-tiled
// rank-k updates, stage blocks staged with asynchronous copies); this file binds its warp primitives to the hardware
// (shuffles, votes, cp.async, __syncwarp) and launches one warp per CTA, 32/G QPs per CTA.  Replaces, for the shapes
// listed in fast_available(), the reference's d_ocp_qp_ipm_solve (external/hpipm/ocp_qp/x_ocp_qp_ipm.c:2684-3120) on
// BLASFEO's panel-major kernels (dsyrk_dpotrf_ln_mn, dtrmm_rlnn: external/blasfeo/blasfeo_hp_pm/d_lapack_lib4.c:1513,
// d_blas3_lib4.c:4893).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "cuipm_device.h"

#define FK_DEV __device__ __forceinline__
static __device__ __forceinline__ int fk_lane() { return (int) (threadIdx.x & 31u); }
static __device__ __forceinline__ void fk_sync() { __syncwarp(); }
static __device__ __forceinline__ double fk_shfl_xor(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
static __device__ __forceinline__ int fk_shfl_xor_i(int v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
static __device__ __forceinline__ bool fk_any(bool p) { return __any_sync(0xffffffffu, p) != 0; }
// 16-byte asynchronous global -> shared copies by single lanes (LDGSTS, no register staging; L1 bypassed: each range is read once
// per sweep), completed by the per-thread group wait + a warp barrier
static __device__ __forceinline__ void fk_cp16(double *sdst, const double *gsrc)
{
    const unsigned sa = (unsigned) __cvta_generic_to_shared(sdst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gsrc) : "memory");
}
static __device__ __forceinline__ void fk_cp_wait() { asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory"); }
// bulk asynchronous copies (TMA, cp.async.bulk): global -> shared, 16-byte aligned, multiple of 16 bytes, completion
// counted in bytes on an mbarrier in shared memory (no register staging, one instruction per contiguous range)
typedef unsigned long long fk_mbar_t;
static __device__ __forceinline__ void fk_mbar_init(fk_mbar_t *b, int count)
{
    const unsigned ba = (unsigned) __cvta_generic_to_shared(b);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ba), "r"(count) : "memory");
}
static __device__ __forceinline__ void fk_bulk(double *sdst, const double *gsrc, unsigned bytes, fk_mbar_t *b)
{
    const unsigned sa = (unsigned) __cvta_generic_to_shared(sdst), ba = (unsigned) __cvta_generic_to_shared(b);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(sa), "l"(gsrc), "r"(bytes), "r"(ba)
                 : "memory");
}
// the same range of the records of the n QPs of a warp (record stride rstep; the groups beyond nvalid re-read the last one) into
// the n groups' shared memory (group stride gstride doubles); kept out of line
static __device__ __noinline__ void fk_bulk_groups(double *sdst, const double *gsrc, unsigned bytes, fk_mbar_t *b, int n, int gstride, size_t rstep, int nvalid)
{
    for (int g = 0; g < n; g++)
    {
        fk_bulk(sdst, gsrc, bytes, b);
        sdst += gstride;
        if (g + 1 < nvalid) gsrc += rstep;
    }
}
static __device__ __forceinline__ void fk_mbar_arrive_tx(fk_mbar_t *b, unsigned bytes)
{
    const unsigned ba = (unsigned) __cvta_generic_to_shared(b);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ba), "r"(bytes) : "memory");
}
static __device__ __forceinline__ void fk_mbar_wait(fk_mbar_t *b, unsigned parity)
{
    const unsigned ba = (unsigned) __cvta_generic_to_shared(b);
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, 0x989680;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(ba), "r"(parity)
        : "memory");
}
// L2 prefetch of a contiguous range (TMA bulk prefetch): no destination, no completion
static __device__ __forceinline__ void fk_prefetch_l2(const double *gsrc, unsigned bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}
// orders this thread's earlier generic-proxy accesses to shared memory before later asynchronous-proxy (bulk copy) writes to it
static __device__ __forceinline__ void fk_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the same for all state spaces: once per sweep, before bulk copies read what earlier sweeps stored into the records
static __device__ __forceinline__ void fk_fence_async_global() { asm volatile("fence.proxy.async;" ::: "memory"); }
static __device__ __forceinline__ double fk_ldg(const double *p) { return __ldg(p); }
typedef double2 fk_double2;
// two consecutive doubles of shared memory, 16-byte aligned (LDS.128)
static __device__ __forceinline__ fk_double2 fk_ld2(const double *p) { return *reinterpret_cast<const double2 *>(p); }
// FP64 tensor-core product D = A B + C on 8 x 4 / 4 x 8 / 8 x 8 fragments spread over the warp (DMMA): lane l holds
// A[l / 4][l % 4], B[l % 4][l / 4] and C[l / 4][2 (l % 4) .. + 1]
static __device__ __forceinline__ void fk_dmma(double &c0, double &c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
static __device__ __forceinline__ double fk_rsqrt(double x) { return rsqrt(x); }
static __device__ __forceinline__ int fk_atomic_inc(int *p) { return atomicAdd(p, 1); }
static __device__ __forceinline__ int fk_atomic_add(int *p, int v) { return atomicAdd(p, v); }
static __device__ __forceinline__ int fk_atomic_cas(int *p, int cmp, int v) { return atomicCAS(p, cmp, v); }
static __device__ __forceinline__ int fk_ld_volatile(const int *p) { return *reinterpret_cast<const volatile int *>(p); }
static __device__ __forceinline__ void fk_st_volatile(int *p, int v) { *reinterpret_cast<volatile int *>(p) = v; }
static __device__ __forceinline__ void fk_threadfence() { __threadfence(); }
static __device__ __forceinline__ void fk_nanosleep(unsigned ns) { __nanosleep(ns); }

#ifdef FK_PROFILE
// development: cycles per sweep and per kind of wait, accumulated by lane 0 of every warp into cuipm_fast_prof[16]
// (0 residual sweep, 1 factorisation, 2 forward sweeps, 3 backward substitutions, 4 mu_aff, 5 waits for vector images,
// 6 waits for matrices, 7 whole solve, 8 warps)
__device__ unsigned long long cuipm_fast_prof[32];
__shared__ long long g_prof[32];
#define FK_PROF_T0() long long t0_ = clock64()
#define FK_PROF_ADD(slot) do { if (fk_lane() == 0) g_prof[slot] += clock64() - t0_; } while (0)
// consecutive phases inside a stage: each ADD2 charges the time since the previous one
#define FK_PROF_T2() long long t2_ = clock64()
#define FK_PROF_ADD2(slot) do { const long long tn_ = clock64(); if (fk_lane() == 0) g_prof[slot] += tn_ - t2_; t2_ = tn_; } while (0)
#endif
#include "cuipm_fast_core.h"

namespace cuipm {

namespace {

extern __shared__ __align__(16) double g_fsmem[];

// MODE 0: a QP stays with its warp for the whole solve; 1 / 2: iteration-sliced scheduling, first launch (initial points, ring
// filled) / loop over the ring (cuipm_fast_core.h, rr_first / rr_loop)
template <int NX, int NU, int G, int MINB, int MODE>
__global__ void __launch_bounds__(32, MINB) cuipm_fast_kernel(const __grid_constant__ FastArgs A)
{
    using K = fastk::Ker<NX, NU, G>;
    __shared__ __align__(8) fk_mbar_t bars[6];
#ifdef FK_PROFILE
    if (fk_lane() == 0) for (int i = 0; i < 32; i++) g_prof[i] = 0;
    const long long tk0 = clock64();
#endif
    K k(A, g_fsmem, bars);
    // persistent warps: each one fetches the next 32/G QPs of the batch until none is left (QPs need 6..18 iterations, and
    // a launch is a few waves of resident warps: a fixed assignment leaves SMs idle at the end of every wave)
    if (MODE == 2)
        k.rr_loop();
    else
        for (;;)
        {
            int first = 0;
            if (fk_lane() == 0) first = atomicAdd(A.next_qp, K::QPW);
            first = __shfl_sync(0xffffffffu, first, 0);
            if (first >= A.nbatch) break;
            if (MODE == 1) k.rr_first(first);
            else k.run(first);
        }
#ifdef FK_PROFILE
    if (fk_lane() == 0)
    {
        g_prof[7] = clock64() - tk0; g_prof[8] = 1;
        for (int i = 0; i < 32; i++) atomicAdd(&cuipm_fast_prof[i], (unsigned long long) g_prof[i]);
    }
#endif
}

// caller's QP records -> kernel-side records: dynamics block with leading dimension ld, Hessian as a full symmetric matrix
// with leading dimension ld (lower triangle mirrored), vector part verbatim.  One CTA per QP, coalesced writes.
__global__ void __launch_bounds__(256) cuipm_repack_kernel(const FastArgs A, const StageDesc *__restrict__ sd)
{
    const int N = A.N, ld = A.ld;
    for (int q = blockIdx.x; q < A.nbatch; q += gridDim.x)
    {
        const double *__restrict__ qp = A.qp + (size_t) q * A.qp_stride;
        double *__restrict__ qk = const_cast<double *>(A.qpk) + (size_t) q * A.qpk_stride;
        for (int k = 0; k <= N; k++)
        {
            const StageDesc d = sd[k];
            const int kind = k == 0 ? 0 : (k == N ? 2 : 1);
            double *o = qk + A.kq[kind] + (kind == 1 ? (size_t) (k - 1) * A.kqs : 0);
            const int n = d.n, nx1 = d.nx1;
            for (int e = threadIdx.x; e < n * nx1; e += blockDim.x)
            {
                const int c = e / n, r = e - c * n;
                o[r + ld * c] = qp[d.q_BAt + e];
            }
            double *H = o + A.kH[kind];
            for (int e = threadIdx.x; e < n * n; e += blockDim.x)
            {
                const int j = e / n, i = e - j * n;
                H[i + ld * j] = i >= j ? qp[d.q_RSQ + e] : qp[d.q_RSQ + j + n * i];
            }
            const int nv = (int) (d.q_stage + d.q_stage_bytes / 8u - d.q_b);
            for (int e = threadIdx.x; e < nv; e += blockDim.x) o[A.kV[kind] + e] = qp[d.q_b + e];
        }
    }
}

template <int NX, int NU, int G>
void sizes(FastArgs &F, int *qpw)
{
    using K = fastk::Ker<NX, NU, G>;
    F.vsize = fastk::vector_pool_doubles(NX, NX + NU, F.nce, F.nbe, F.ns2e, F.nve);
    int gs = K::MATS + F.vsize;
    // 32 / G groups share a warp; 64-bit shared loads are served per half-warp: a group stride of 8 (mod 16) doubles puts the
    // consecutive-row accesses of the two groups of a half-warp on disjoint banks
    while (gs % 16 != 8) gs++;
    F.gstride = gs;
    *qpw = K::QPW;
}

template <int NX, int NU, int G, int MINB, int MODE>
cudaError_t launch_one(const FastArgs &F, cudaStream_t stream)
{
    using K = fastk::Ker<NX, NU, G>;
    const size_t smem = sizeof(double) * ((size_t) F.gstride * K::QPW + 2 * (size_t) F.nmaps * F.nbe);
    if (((size_t) F.qpk | (size_t) F.sol | (size_t) F.work) & 15) return cudaErrorMisalignedAddress;      // bulk copies need 16-byte aligned records
    cudaError_t err = cudaFuncSetAttribute(cuipm_fast_kernel<NX, NU, G, MINB, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    if (err != cudaSuccess) return err;
    // the CTAs of one SM together need most of its shared memory: ask for the largest carve-out (the default heuristic
    // sized it for a single CTA, which left one warp per SM resident)
    err = cudaFuncSetAttribute(cuipm_fast_kernel<NX, NU, G, MINB, MODE>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (err != cudaSuccess) return err;
    if (getenv("CUIPM_DEBUG"))
    {
        int nblk = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, cuipm_fast_kernel<NX, NU, G, MINB, MODE>, 32, smem);
        fprintf(stderr, "cuipm_fast_kernel<%d,%d,%d>: %zu bytes of shared memory per CTA, %d CTAs (%d QPs) per SM\n", NX, NU, G, smem, nblk, nblk * K::QPW);
    }
    static int resident = 0;        // CTAs per SM x SMs of this instance
    if (!resident)
    {
        int nblk = 0, dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, cuipm_fast_kernel<NX, NU, G, MINB, MODE>, 32, smem);
        resident = (nblk > 0 ? nblk : 1) * (sms > 0 ? sms : 1);
    }
    const int want = (F.nbatch + K::QPW - 1) / K::QPW;
    const int grid = want < resident ? want : resident;       // (the ring loop too: more warps than QP groups would only poll)
    cuipm_fast_kernel<NX, NU, G, MINB, MODE><<<grid, 32, smem, stream>>>(F);
    return cudaGetLastError();
}

}  // namespace

// (interior nx, nu) pairs with an instance of the throughput kernel, and the lanes per QP each one runs with
#define CUIPM_FAST_INSTANCES(X) \
    X(21, 3, 8, 4)              \
    X(8, 3, 4, 8)               \
    X(4, 1, 2, 8)               \
    X(12, 4, 8, 6)              \
    X(48, 12, 32, 3)

// development: other lanes-per-QP mappings of the headline shape, selected with CUIPM_FAST_G=16|32
#ifdef CUIPM_FAST_DEV
#define CUIPM_FAST_DEV_INSTANCES(X) \
    X(21, 3, 16, 8)                 \
    X(21, 3, 32, 16)
#else
#define CUIPM_FAST_DEV_INSTANCES(X)
#endif
static int dev_g() { const char *e = getenv("CUIPM_FAST_G"); return e ? atoi(e) : 0; }

bool fast_available(int nx, int nu, FastArgs &F, int *qp_per_warp)
{
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_ && dev_g() == G_) { sizes<NX_, NU_, G_>(F, qp_per_warp); return sizeof(double) * ((size_t) F.gstride * (32 / G_) + 2 * (size_t) F.nmaps * F.nbe) <= 226 * 1024; }
    CUIPM_FAST_DEV_INSTANCES(X)
#undef X
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_) { sizes<NX_, NU_, G_>(F, qp_per_warp); return sizeof(double) * ((size_t) F.gstride * (32 / G_) + 2 * (size_t) F.nmaps * F.nbe) <= 226 * 1024; }
    CUIPM_FAST_INSTANCES(X)
#undef X
    return false;
}

int launch_repack(const FastArgs &F, const StageDesc *sd, void *stream_)
{
    cudaStream_t stream = (cudaStream_t) stream_;
    static int sms = 0;
    if (!sms)
    {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 1;
    }
    const int grid = F.nbatch < sms * 8 ? F.nbatch : sms * 8;      // eight CTAs per SM, grid-stride over the batch
    cuipm_repack_kernel<<<grid, 256, 0, stream>>>(F, sd);
    return (int) cudaGetLastError();
}

#ifdef FK_PROFILE
extern "C" void cuipm_fast_prof_read(unsigned long long *out, int reset)
{
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, cuipm_fast_prof, sizeof(unsigned long long) * 32);
    if (reset) { unsigned long long z[32] = {0}; cudaMemcpyToSymbol(cuipm_fast_prof, z, sizeof(z)); }
}
#endif

// instances with the iteration-sliced scheduling compiled in (two more kernels each)
#define CUIPM_FAST_RR_INSTANCES(X) CUIPM_FAST_INSTANCES(X)

// QPs the device holds at once with the throughput kernel of this shape (CTAs per SM x SMs x QPs per warp); 0 if unknown
template <int NX, int NU, int G, int MINB>
static int resident_qps(const FastArgs &F)
{
    using K = fastk::Ker<NX, NU, G>;
    const size_t smem = sizeof(double) * ((size_t) F.gstride * K::QPW + 2 * (size_t) F.nmaps * F.nbe);
    int nblk = 0, dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(cuipm_fast_kernel<NX, NU, G, MINB, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    cudaFuncSetAttribute(cuipm_fast_kernel<NX, NU, G, MINB, 0>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, cuipm_fast_kernel<NX, NU, G, MINB, 0>, 32, smem) != cudaSuccess) return 0;
    return nblk * sms * K::QPW;
}

int fast_resident_qps(const FastArgs &F)
{
    const int nx = F.s1.nx, nu = F.s1.nu;
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_) return resident_qps<NX_, NU_, G_, MB_>(F);
    CUIPM_FAST_INSTANCES(X)
#undef X
    return 0;
}

bool fast_rr_available(int nx, int nu)
{
    if (dev_g()) return false;
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_) return true;
    CUIPM_FAST_RR_INSTANCES(X)
#undef X
    return false;
}

int launch_fast(const FastArgs &F, void *stream_, int mode)
{
    cudaStream_t stream = (cudaStream_t) stream_;
    const int nx = F.s1.nx, nu = F.s1.nu;
    if (mode != 0)
    {
#define X(NX_, NU_, G_, MB_) \
        if (nx == NX_ && nu == NU_) return (int) (mode == 1 ? launch_one<NX_, NU_, G_, MB_, 1>(F, stream) : launch_one<NX_, NU_, G_, MB_, 2>(F, stream));
        CUIPM_FAST_RR_INSTANCES(X)
#undef X
        return (int) cudaErrorInvalidValue;
    }
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_ && dev_g() == G_) return (int) launch_one<NX_, NU_, G_, MB_, 0>(F, stream);
    CUIPM_FAST_DEV_INSTANCES(X)
#undef X
#define X(NX_, NU_, G_, MB_) \
    if (nx == NX_ && nu == NU_) return (int) launch_one<NX_, NU_, G_, MB_, 0>(F, stream);
    CUIPM_FAST_INSTANCES(X)
#undef X
    return (int) cudaErrorInvalidValue;
}

}  // namespace cuipm
