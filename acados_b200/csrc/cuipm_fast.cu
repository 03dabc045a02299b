// cuipm_fast.cu -- CUDA instantiation (sm_90a) of the throughput kernel of the batched OCP-QP interior-point solver.
//
// The kernel body is cuipm_fast_core.h (a group of G lanes per QP, 32/G QPs per warp in lock step, register-tiled
// rank-k updates, stage blocks staged with asynchronous copies); this file binds its warp primitives to the hardware
// (shuffles, votes, cp.async, __syncwarp) and launches one warp per CTA, 32/G QPs per CTA.  Replaces, for the shapes
// in CUIPM_FAST_INSTANCES below, the reference's d_ocp_qp_ipm_solve (external/hpipm/ocp_qp/x_ocp_qp_ipm.c:2684-3120) on
// BLASFEO's panel-major kernels (dsyrk_dpotrf_ln_mn, dtrmm_rlnn: external/blasfeo/blasfeo_hp_pm/d_lapack_lib4.c:1513,
// d_blas3_lib4.c:4893).  The host side of the throughput path (FastPath, cuipm_device.h) is at the end of this file.
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "cuipm_device.h"
#include "cuipm_internal.h"
#include "cuipm_plan.h"

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
    __shared__ __align__(8) fk_mbar_t bar;
#ifdef FK_PROFILE
    if (fk_lane() == 0) for (int i = 0; i < 32; i++) g_prof[i] = 0;
    const long long tk0 = clock64();
#endif
    K k(A, g_fsmem, &bar);
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

}  // namespace

// the compiled instances: interior (nx, nu), lanes per QP, minimum CTAs per SM of the launch bounds
#define CUIPM_FAST_INSTANCES(X) \
    X(21, 3, 8, 4)              \
    X(8, 3, 4, 8)               \
    X(4, 1, 2, 8)               \
    X(12, 4, 8, 6)              \
    X(48, 12, 32, 3)

typedef void (*FastKernel)(FastArgs);

// one instance: the interior (nx, nu) it runs, QPs per warp, its shared-memory layout (cuipm_fast_core.h) and its kernels for
// launch mode 0 (a QP stays with its warp), 1 and 2 (iteration-sliced scheduling: initial points and ring filled, loop over the ring)
struct FastInstance
{
    int nx, nu, qpw;
    size_t (*layout)(FastArgs &);
    FastKernel kernel[3];
};

static const FastInstance kInstances[] = {
#define X(NX_, NU_, G_, MB_) \
    {NX_, NU_, 32 / G_, fastk::layout<NX_, NU_, G_>, {cuipm_fast_kernel<NX_, NU_, G_, MB_, 0>, cuipm_fast_kernel<NX_, NU_, G_, MB_, 1>, cuipm_fast_kernel<NX_, NU_, G_, MB_, 2>}},
    CUIPM_FAST_INSTANCES(X)
#undef X
};

#define CKF(what, call)                                                                                 \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess)                                                                          \
        {                                                                                               \
            set_error(std::string(what) + ": " + cudaGetErrorString(e_));                               \
            return CUIPM_ERR_CUDA;                                                                      \
        }                                                                                               \
    } while (0)

// The dynamic shared memory attribute belongs to the kernel, not to a solver: solvers of other shapes may launch the same
// instance with more, so it is set before every launch.  The CTAs of one SM together need most of its shared memory: ask for
// the largest carve-out (the default heuristic sized it for a single CTA, which left one warp per SM resident).
static cudaError_t set_smem(FastKernel k, size_t smem)
{
    cudaError_t err = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
    if (err == cudaSuccess) err = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    return err;
}

int FastPath::create(const std::vector<StageDesc> &sd, const std::vector<int> &ipool, const ProbDesc &P, int max_batch, int nslot_, int device)
{
    if (!fast_plan(sd, ipool, P, F)) return CUIPM_OK;
    const FastInstance *in = nullptr;
    for (const FastInstance &i : kInstances)
        if (i.nx == F.s1.nx && i.nu == F.s1.nu) in = &i;
    if (!in) return CUIPM_OK;
    smem = in->layout(F);
    if (smem > 226 * 1024) return CUIPM_OK;
    inst = in;
    nslot = nslot_;
    const size_t nb = (size_t) max_batch;
    CKF("cudaMalloc", cudaMalloc(&redo_list, sizeof(int) * nb));
    CKF("cudaMalloc", cudaMalloc(&ctr, sizeof(int) * 2 * nslot));
    CKF("cudaMemset", cudaMemset(ctr, 0, sizeof(int) * 2 * nslot));
    CKF("cudaMalloc", cudaMalloc(&qpk, sizeof(double) * F.qpk_stride * nb));
    CKF("cudaMemset", cudaMemset(qpk, 0, sizeof(double) * F.qpk_stride * nb));
    CKF("cudaMalloc", cudaMalloc(&rr_state, sizeof(double) * 12 * nb));
    CKF("cudaMalloc", cudaMalloc(&rr_ring, sizeof(int) * CUIPM_RR_RINGS * nb));
    CKF("cudaMalloc", cudaMalloc(&rr_ctr, sizeof(int) * CUIPM_RR_CTR * nslot));
    // residency with this solver's shared memory, per mode (the three kernels need different numbers of registers)
    CKF("cudaDeviceGetAttribute", cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    for (int m = 0; m < 3; m++)
    {
        int nblk = 0;
        CKF("cudaFuncSetAttribute", set_smem(inst->kernel[m], smem));
        CKF("cudaOccupancyMaxActiveBlocksPerMultiprocessor", cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, inst->kernel[m], 32, smem));
        ctas[m] = (nblk > 0 ? nblk : 1) * sms;
        if (m == 0) ring_qps = nblk * sms * inst->qpw;
    }
    return CUIPM_OK;
}

// the throughput kernel of `mode` over f.nbatch QPs: persistent warps, at most as many CTAs as the device holds at once (the
// ring loop too: more warps than QP groups would only poll)
static cudaError_t launch(const FastPath &p, int mode, const FastArgs &f, cudaStream_t stream)
{
    const FastKernel k = p.inst->kernel[mode];
    cudaError_t err = set_smem(k, p.smem);
    if (err != cudaSuccess) return err;
    const int want = (f.nbatch + p.inst->qpw - 1) / p.inst->qpw;
    k<<<want < p.ctas[mode] ? want : p.ctas[mode], 32, p.smem, stream>>>(f);
    return cudaGetLastError();
}

int FastPath::enqueue(LaunchArgs &a, size_t lo, int slot, void *stream_, int *launches, void *ev_repacked, void *ev_done)
{
    // (m != 0 -- acados' tau_min option -- changes the ratio test into the quadratic rule: generic kernel only, the hot code of
    // the throughput kernel stays as it is; the bulk copies need 16-byte aligned records)
    if (!inst || !use || a.o.lq_fact > 1 || a.o.m_relax != 0.0 || (((size_t) a.sol | (size_t) a.work) & 15)) return CUIPM_OK;
    cudaStream_t stream = (cudaStream_t) stream_;
    FastArgs f = F;
    f.nbatch = a.nbatch; f.ipool = a.ipool; f.qp = a.qp; f.sol = a.sol; f.work = a.work; f.info = a.info; f.stat = a.stat; f.o = a.o;
    f.qpk = qpk + F.qpk_stride * lo;
    f.redo_list = redo_list + lo; f.redo_count = ctr + 2 * slot; f.next_qp = f.redo_count + 1;
    CKF("cudaMemsetAsync", cudaMemsetAsync(f.redo_count, 0, 2 * sizeof(int), stream));
    cuipm_repack_kernel<<<f.nbatch < sms * 8 ? f.nbatch : sms * 8, 256, 0, stream>>>(f, a.sd);      // eight CTAs per SM, grid-stride over the batch
    CKF("kernel launch (repack)", cudaGetLastError());
    (*launches)++;
    if (ev_repacked) cudaEventRecord((cudaEvent_t) ev_repacked, stream);
    // iteration-sliced scheduling pays when the batch is more than one wave of resident QPs and not many; small batches keep the
    // single launch (below one wave the extra launch and the ring traffic cost more than the idle slots they save)
    cudaError_t e;
    if (rr && (rr > 1 || (ring_qps > 0 && a.nbatch > ring_qps)))
    {
        f.rr_state = rr_state + 12 * lo; f.rr_ring = rr_ring + CUIPM_RR_RINGS * lo; f.rr_ctr = rr_ctr + CUIPM_RR_CTR * slot;
        CKF("cudaMemsetAsync", cudaMemsetAsync(f.rr_ring, 0xff, sizeof(int) * CUIPM_RR_RINGS * (size_t) a.nbatch, stream));
        CKF("cudaMemsetAsync", cudaMemsetAsync(f.rr_ctr, 0, CUIPM_RR_CTR * sizeof(int), stream));
        e = launch(*this, 1, f, stream);
        if (e == cudaSuccess) { (*launches)++; e = launch(*this, 2, f, stream); }
    }
    else
        e = launch(*this, 0, f, stream);
    if (ev_done) cudaEventRecord((cudaEvent_t) ev_done, stream);
    CKF("kernel launch (throughput kernel)", e);
    (*launches)++;
    a.redo_list = f.redo_list;
    a.redo_count = f.redo_count;
    return CUIPM_OK;
}

int FastPath::handed_back() const
{
    std::vector<int> h(2 * nslot);
    if (cudaMemcpy(h.data(), ctr, sizeof(int) * h.size(), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    int total = 0;
    for (int c = 0; c < nslot; c++) total += h[2 * c];
    return total;
}

void FastPath::destroy()
{
    cudaFree(qpk); cudaFree(redo_list); cudaFree(ctr);
    cudaFree(rr_state); cudaFree(rr_ring); cudaFree(rr_ctr);
}

#ifdef FK_PROFILE
extern "C" void cuipm_fast_prof_read(unsigned long long *out, int reset)
{
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, cuipm_fast_prof, sizeof(unsigned long long) * 32);
    if (reset) { unsigned long long z[32] = {0}; cudaMemcpyToSymbol(cuipm_fast_prof, z, sizeof(z)); }
}
#endif

}  // namespace cuipm
