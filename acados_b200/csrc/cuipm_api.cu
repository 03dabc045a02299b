// cuipm_api.cu -- solver lifetime and the solve entry points of the C ABI (include/cuipm.h).
//
// Replaces, for a whole batch at once, what ocp_qp_hpipm() does per instance in the reference
// (acados/ocp_qp/ocp_qp_hpipm.c:314-405): hand the QP to the IPM, collect status / iteration count /
// statistics.  All device memory is owned by the solver object (the reference's plugin reports sizes and is
// handed raw host memory, which cannot hold device allocations -- SURVEY.md section 8(b)).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "cuipm.h"
#include "cuipm_device.h"
#include "cuipm_internal.h"
#include "cuipm_plan.h"

using namespace cuipm;

struct cuipm_solver
{
    int device = 0;
    int max_batch = 0;
    int warps = 1;
    cuipm_layout *layout = nullptr;
    ProbDesc P{};
    std::vector<StageDesc> sd_host;
    StageDesc *d_sd = nullptr;
    int *d_ipool = nullptr;
    double *d_qp = nullptr, *d_sol = nullptr, *d_work = nullptr, *d_stat = nullptr, *d_seed = nullptr, *d_sens = nullptr;
    size_t stat_cap = 0;
    cuipm_info *d_info = nullptr;
    cudaStream_t stream = nullptr;
    static constexpr int kPipe = 8;          // streams of the host entry: copy of chunk c+1 overlaps the solve of chunk c
    int npipe = 8;                           // chunks per host call (tuning key "pipe"; 8 measured best for 1.5 GB batches)
    cudaStream_t pipe[kPipe] = {};
    cudaEvent_t pipe_done[kPipe] = {};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int last_launches = 0;
    int pending = 0;                         // an asynchronous host solve has been enqueued and not waited for
    float last_ms = 0.f;
    cuipm_opts last_opts{};
    FastPath fast;                           // throughput kernel (cuipm_fast.cu)
    cudaEvent_t evk0 = nullptr, evk1 = nullptr;   // around the throughput kernel of the last cuipm_solve_device call
    bool timed_fast = false;
};

#define CK(call)                                                                                        \
    do {                                                                                                \
        cudaError_t e_ = (call);                                                                        \
        if (e_ != cudaSuccess)                                                                          \
        {                                                                                               \
            set_error(std::string(#call) + ": " + cudaGetErrorString(e_));                              \
            return CUIPM_ERR_CUDA;                                                                      \
        }                                                                                               \
    } while (0)

static int build_desc(cuipm_solver *s, const cuipm_shape *sh)
{
    std::vector<int> ipool;
    std::string err;
    int rc = build_plan(sh, s->layout, s->sd_host, ipool, s->P, err);
    if (rc != CUIPM_OK) { set_error(err); return rc; }
    const int N = sh->N;
    CK(cudaMalloc(&s->d_sd, sizeof(StageDesc) * (N + 1)));
    CK(cudaMemcpy(s->d_sd, s->sd_host.data(), sizeof(StageDesc) * (N + 1), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&s->d_ipool, sizeof(int) * (ipool.size() + 1)));
    if (!ipool.empty()) CK(cudaMemcpy(s->d_ipool, ipool.data(), sizeof(int) * ipool.size(), cudaMemcpyHostToDevice));
    return s->fast.create(s->sd_host, ipool, s->P, s->max_batch, cuipm_solver::kPipe, s->device);
}

// One batch (or one chunk of it) on `stream`: the throughput kernel where the shape and the options allow it, then the
// generic kernel over the QPs it handed back (cold paths); otherwise the generic kernel over everything.
// slot selects the hand-back counter (chunks run concurrently on different streams).
static int launch_batch(cuipm_solver *s, const LaunchArgs &a0, int slot, size_t lo, cudaStream_t stream, int *launches)
{
    LaunchArgs a = a0;
    a.redo_list = nullptr;
    a.redo_count = nullptr;
    const bool timed = slot == 0 && s->evk0;
    int rc = s->fast.enqueue(a, lo, slot, (void *) stream, launches, timed ? s->evk0 : nullptr, timed ? s->evk1 : nullptr);
    if (rc != CUIPM_OK) return rc;
    if (timed && a.redo_count) s->timed_fast = true;
    rc = launch_solve(a, s->warps, (void *) stream);
    if (rc != 0) { set_error(std::string("kernel launch: ") + cudaGetErrorString((cudaError_t) rc)); return CUIPM_ERR_CUDA; }
    (*launches)++;
    return CUIPM_OK;
}

extern "C" cuipm_solver *cuipm_create(const cuipm_shape *shape, int max_batch, int device)
{
    if (!shape || max_batch <= 0) { set_error("cuipm_create: bad arguments"); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    {
        set_error("no CUDA device available (cuipm has no CPU fallback)");
        return nullptr;
    }
    if (device < 0 || device >= ndev) { set_error("cuipm_create: no such device"); return nullptr; }
    if (cudaSetDevice(device) != cudaSuccess) { set_error("cudaSetDevice failed"); return nullptr; }
    cuipm_solver *s = new cuipm_solver();
    s->device = device;
    s->max_batch = max_batch;
    s->layout = cuipm_layout_create(shape);
    auto fail = [&]() { cuipm_destroy(s); return (cuipm_solver *) nullptr; };
    if (build_desc(s, shape) != CUIPM_OK) return fail();
    auto alloc = [&](void **p, size_t bytes) {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e != cudaSuccess) { set_error(std::string("cudaMalloc: ") + cudaGetErrorString(e)); return false; }
        return true;
    };
    if (!alloc((void **) &s->d_qp, sizeof(double) * s->P.qp_stride * max_batch)) return fail();
    if (!alloc((void **) &s->d_sol, sizeof(double) * s->P.sol_stride * max_batch)) return fail();
    if (!alloc((void **) &s->d_work, sizeof(double) * s->P.work_stride * max_batch)) return fail();
    if (!alloc((void **) &s->d_info, sizeof(cuipm_info) * max_batch)) return fail();
    if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate failed"); return fail(); }
    bool ok = cudaEventCreate(&s->ev0) == cudaSuccess && cudaEventCreate(&s->ev1) == cudaSuccess
              && cudaEventCreate(&s->evk0) == cudaSuccess && cudaEventCreate(&s->evk1) == cudaSuccess;
    for (int i = 0; ok && i < cuipm_solver::kPipe; i++)
        ok = cudaStreamCreateWithFlags(&s->pipe[i], cudaStreamNonBlocking) == cudaSuccess
             && cudaEventCreateWithFlags(&s->pipe_done[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaMemsetAsync(s->d_work, 0, sizeof(double) * s->P.work_stride * max_batch, s->stream) == cudaSuccess
         && cudaMemsetAsync(s->d_sol, 0, sizeof(double) * s->P.sol_stride * max_batch, s->stream) == cudaSuccess
         && cudaStreamSynchronize(s->stream) == cudaSuccess;
    if (!ok) { set_error(std::string("cuipm_create: streams / events / initial clears: ") + cudaGetErrorString(cudaGetLastError())); return fail(); }
    // default warps per QP: one warp owns one QP unless the stage block is large
    s->warps = s->P.nmax > 40 ? 4 : 1;
    return s;
}

extern "C" void cuipm_destroy(cuipm_solver *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    if (s->stream) cudaStreamSynchronize(s->stream);
    cudaFree(s->d_sd); cudaFree(s->d_ipool); cudaFree(s->d_qp); cudaFree(s->d_sol); cudaFree(s->d_work);
    cudaFree(s->d_stat); cudaFree(s->d_info); cudaFree(s->d_seed); cudaFree(s->d_sens);
    s->fast.destroy();
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    if (s->evk0) cudaEventDestroy(s->evk0);
    if (s->evk1) cudaEventDestroy(s->evk1);
    for (int i = 0; i < cuipm_solver::kPipe; i++)
    {
        if (s->pipe[i]) { cudaStreamSynchronize(s->pipe[i]); cudaStreamDestroy(s->pipe[i]); }
        if (s->pipe_done[i]) cudaEventDestroy(s->pipe_done[i]);
    }
    if (s->stream) cudaStreamDestroy(s->stream);
    cuipm_layout_destroy(s->layout);
    delete s;
}

extern "C" void *cuipm_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { set_error("cudaHostAlloc failed"); return nullptr; }
    return p;
}
extern "C" void cuipm_host_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" const cuipm_layout *cuipm_get_layout(const cuipm_solver *s) { return s->layout; }
extern "C" double *cuipm_device_qp_buffer(cuipm_solver *s) { return s->d_qp; }
extern "C" double *cuipm_device_sol_buffer(cuipm_solver *s) { return s->d_sol; }
extern "C" cuipm_info *cuipm_device_info_buffer(cuipm_solver *s) { return s->d_info; }
extern "C" void *cuipm_stream(cuipm_solver *s) { return (void *) s->stream; }
extern "C" int cuipm_last_launch_count(const cuipm_solver *s) { return s->last_launches; }
extern "C" int cuipm_last_handed_back(cuipm_solver *s)
{
    if (!s || !s->fast.inst) return 0;
    cudaSetDevice(s->device);
    cudaStreamSynchronize(s->stream);
    return s->fast.handed_back();
}
extern "C" float cuipm_last_main_kernel_ms(cuipm_solver *s)
{
    float ms = 0.f;
    if (s && s->timed_fast && cudaEventElapsedTime(&ms, s->evk0, s->evk1) == cudaSuccess) return ms;
    return s ? s->last_ms : 0.f;
}
extern "C" float cuipm_last_kernel_ms(const cuipm_solver *s) { return s->last_ms; }

extern "C" int cuipm_set_tuning(cuipm_solver *s, const char *key, int value)
{
    if (!std::strcmp(key, "warps"))
    {
        if (value != 1 && value != 2 && value != 4) { set_error("warps must be 1, 2 or 4"); return CUIPM_ERR_INVALID; }
        s->warps = value;
        return CUIPM_OK;
    }
    if (!std::strcmp(key, "pipe"))
    {
        if (value < 1 || value > cuipm_solver::kPipe) { set_error("pipe must be in 1..8"); return CUIPM_ERR_INVALID; }
        s->npipe = value;
        return CUIPM_OK;
    }
    if (!std::strcmp(key, "rr"))
    {
        s->fast.rr = value;
        return CUIPM_OK;
    }
    if (!std::strcmp(key, "fast"))
    {
        s->fast.use = value != 0;
        return CUIPM_OK;
    }
    set_error("unknown tuning key");
    return CUIPM_ERR_INVALID;
}

extern "C" int cuipm_solve_device(cuipm_solver *s, int nbatch, const double *d_qp, double *d_sol, cuipm_info *d_info,
                                  double *d_stat, const cuipm_opts *opts, int sync)
{
    if (!s || nbatch < 0 || nbatch > s->max_batch || !d_qp || !d_sol || !d_info || !opts)
    {
        set_error("cuipm_solve_device: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    int rc = opts_check(opts);
    if (rc != CUIPM_OK) return rc;
    CK(cudaSetDevice(s->device));
    s->last_launches = 0;
    if (nbatch == 0) return CUIPM_OK;
    LaunchArgs a;
    a.P = s->P; a.sd = s->d_sd; a.ipool = s->d_ipool; a.qp = d_qp; a.sol = d_sol; a.work = s->d_work; a.info = d_info;
    a.stat = d_stat; a.o = *opts; a.nbatch = nbatch; a.seed = nullptr; a.sens = nullptr; a.adjoint = 0;
    s->last_opts = *opts;
    CK(cudaEventRecord(s->ev0, s->stream));
    rc = launch_batch(s, a, 0, 0, s->stream, &s->last_launches);
    if (rc != CUIPM_OK) return rc;
    CK(cudaEventRecord(s->ev1, s->stream));
    if (sync)
    {
        CK(cudaStreamSynchronize(s->stream));
        cudaEventElapsedTime(&s->last_ms, s->ev0, s->ev1);
    }
    return CUIPM_OK;
}

// Enqueues the whole host-buffer solve (copies in, kernels, copies out) on the solver's streams and returns; cuipm_wait
// blocks until it has completed.  Two solver objects used alternately overlap the copies of one batch with the solve of
// the previous one (what a streaming caller -- an RL sweep, the benchmark's end-to-end leg -- wants).
extern "C" int cuipm_solve_host_async(cuipm_solver *s, int nbatch, const double *qp, double *sol, cuipm_info *info, double *stat,
                                      const cuipm_opts *opts)
{
    if (!s || nbatch < 0 || nbatch > s->max_batch || !qp || !sol || !info || !opts)
    {
        set_error("cuipm_solve_host: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    int rc = opts_check(opts);
    if (rc != CUIPM_OK) return rc;
    CK(cudaSetDevice(s->device));
    if (s->pending)
    {   // a previous asynchronous solve of this object is still in flight: its device buffers (and d_stat) are in use
        rc = cuipm_wait(s);
        if (rc != CUIPM_OK) return rc;
    }
    if (nbatch == 0) return CUIPM_OK;
    const size_t stat_n = (size_t) nbatch * CUIPM_STAT_M * (opts->stat_max + 1);
    if (stat && s->stat_cap < stat_n)
    {
        cudaFree(s->d_stat);
        s->d_stat = nullptr;
        CK(cudaMalloc(&s->d_stat, sizeof(double) * stat_n));
        s->stat_cap = stat_n;
    }
    // Chunked pipeline: chunk c is copied in, solved and copied out on its own stream, so the H2D copy of the next chunk
    // (the batch is ~0.4 MB per QP) overlaps the solve of the previous ones; kernels of different chunks share the SMs.
    const int nchunk = nbatch >= 512 ? s->npipe : 1;
    int nlaunch = 0;
    const int per = (nbatch + nchunk - 1) / nchunk;
    CK(cudaEventRecord(s->ev0, s->stream));
    for (int c = 0; c < nchunk; c++)
    {
        const int lo = c * per, n = std::min(per, nbatch - lo);
        if (n <= 0) break;
        cudaStream_t st = s->pipe[c];
        CK(cudaStreamWaitEvent(st, s->ev0, 0));
        const size_t qo = s->P.qp_stride * (size_t) lo, so = s->P.sol_stride * (size_t) lo;
        CK(cudaMemcpyAsync(s->d_qp + qo, qp + qo, sizeof(double) * s->P.qp_stride * n, cudaMemcpyHostToDevice, st));
        if (opts->warm_start >= 1)
            CK(cudaMemcpyAsync(s->d_sol + so, sol + so, sizeof(double) * s->P.sol_stride * n, cudaMemcpyHostToDevice, st));
        LaunchArgs a;
        a.P = s->P; a.sd = s->d_sd; a.ipool = s->d_ipool; a.qp = s->d_qp + qo; a.sol = s->d_sol + so;
        a.work = s->d_work + s->P.work_stride * (size_t) lo; a.info = s->d_info + lo;
        a.stat = stat ? s->d_stat + (size_t) lo * CUIPM_STAT_M * (opts->stat_max + 1) : nullptr;
        a.o = *opts; a.nbatch = n; a.seed = nullptr; a.sens = nullptr; a.adjoint = 0;
        rc = launch_batch(s, a, c, (size_t) lo, st, &nlaunch);
        if (rc != CUIPM_OK) return rc;
        CK(cudaMemcpyAsync(sol + so, s->d_sol + so, sizeof(double) * s->P.sol_stride * n, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(info + lo, s->d_info + lo, sizeof(cuipm_info) * n, cudaMemcpyDeviceToHost, st));
        if (stat)
            CK(cudaMemcpyAsync(stat + (size_t) lo * CUIPM_STAT_M * (opts->stat_max + 1), a.stat,
                               sizeof(double) * (size_t) n * CUIPM_STAT_M * (opts->stat_max + 1), cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(s->pipe_done[c], st));
        CK(cudaStreamWaitEvent(s->stream, s->pipe_done[c], 0));
    }
    s->last_launches = nlaunch;
    s->last_opts = *opts;
    CK(cudaEventRecord(s->ev1, s->stream));
    s->pending = 1;
    return CUIPM_OK;
}

// Chunk-granular form of the host entry: records lo .. lo+n-1 of the batch whose host buffers start at qp / sol / info are copied
// in, solved and copied out on pipe stream `slot`; returns as soon as the work is enqueued.  A caller that produces its records
// chunk by chunk (the acados plugin unpacking ocp_qp_in structs) overlaps that with the copies and solves of the chunks before.
extern "C" int cuipm_solve_host_chunk(cuipm_solver *s, int slot, int lo, int n, const double *qp, double *sol, cuipm_info *info,
                                      const cuipm_opts *opts)
{
    if (!s || slot < 0 || slot >= cuipm_solver::kPipe || lo < 0 || n < 0 || lo + n > s->max_batch || !qp || !sol || !info || !opts)
    {
        set_error("cuipm_solve_host_chunk: bad arguments (slot in 0..7, lo + n <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    int rc = opts_check(opts);
    if (rc != CUIPM_OK) return rc;
    CK(cudaSetDevice(s->device));
    if (n == 0) return CUIPM_OK;
    cudaStream_t st = s->pipe[slot];
    const size_t qo = s->P.qp_stride * (size_t) lo, so = s->P.sol_stride * (size_t) lo;
    CK(cudaMemcpyAsync(s->d_qp + qo, qp + qo, sizeof(double) * s->P.qp_stride * n, cudaMemcpyHostToDevice, st));
    if (opts->warm_start >= 1)
        CK(cudaMemcpyAsync(s->d_sol + so, sol + so, sizeof(double) * s->P.sol_stride * n, cudaMemcpyHostToDevice, st));
    LaunchArgs a;
    a.P = s->P; a.sd = s->d_sd; a.ipool = s->d_ipool; a.qp = s->d_qp + qo; a.sol = s->d_sol + so;
    a.work = s->d_work + s->P.work_stride * (size_t) lo; a.info = s->d_info + lo;
    a.stat = nullptr;
    a.o = *opts; a.nbatch = n; a.seed = nullptr; a.sens = nullptr; a.adjoint = 0;
    int nlaunch = 0;
    rc = launch_batch(s, a, slot, (size_t) lo, st, &nlaunch);
    if (rc != CUIPM_OK) return rc;
    CK(cudaMemcpyAsync(sol + so, s->d_sol + so, sizeof(double) * s->P.sol_stride * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(info + lo, s->d_info + lo, sizeof(cuipm_info) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(s->pipe_done[slot], st));
    s->last_launches = nlaunch;
    s->last_opts = *opts;
    return CUIPM_OK;
}

extern "C" int cuipm_wait_chunk(cuipm_solver *s, int slot)
{
    if (!s || slot < 0 || slot >= cuipm_solver::kPipe) { set_error("cuipm_wait_chunk: bad arguments"); return CUIPM_ERR_INVALID; }
    CK(cudaSetDevice(s->device));
    CK(cudaEventSynchronize(s->pipe_done[slot]));
    return CUIPM_OK;
}

extern "C" int cuipm_wait(cuipm_solver *s)
{
    if (!s) { set_error("cuipm_wait: null solver"); return CUIPM_ERR_INVALID; }
    CK(cudaSetDevice(s->device));
    CK(cudaStreamSynchronize(s->stream));
    if (s->pending) cudaEventElapsedTime(&s->last_ms, s->ev0, s->ev1);
    s->pending = 0;
    return CUIPM_OK;
}

extern "C" int cuipm_solve_host(cuipm_solver *s, int nbatch, const double *qp, double *sol, cuipm_info *info, double *stat,
                                const cuipm_opts *opts)
{
    int rc = cuipm_solve_host_async(s, nbatch, qp, sol, info, stat, opts);
    if (rc != CUIPM_OK) return rc;
    return cuipm_wait(s);
}

// Solution sensitivities (reference: d_ocp_qp_ipm_sens_frw / _adj, external/hpipm/ocp_qp/x_ocp_qp_ipm.c:3285-3444, behind
// ocp_qp_hpipm_eval_forw_sens / _adj_sens, acados/ocp_qp/ocp_qp_hpipm.c:481-506): one substitution per QP with the
// factorisation of the last IPM iteration of the preceding solve, which is still in the solver's work records.
extern "C" int cuipm_sens_device(cuipm_solver *s, int nbatch, const double *d_qp, const double *d_seed, double *d_sens, int adjoint,
                                 const cuipm_opts *opts, int sync)
{
    if (!s || nbatch < 0 || nbatch > s->max_batch || !d_qp || !d_seed || !d_sens || !opts)
    {
        set_error("cuipm_sens_device: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    int rc = opts_check(opts);
    if (rc != CUIPM_OK) return rc;
    CK(cudaSetDevice(s->device));
    s->last_launches = 0;
    if (nbatch == 0) return CUIPM_OK;
    LaunchArgs a;
    a.P = s->P; a.sd = s->d_sd; a.ipool = s->d_ipool; a.qp = d_qp; a.sol = nullptr; a.work = s->d_work; a.info = nullptr;
    a.stat = nullptr; a.o = *opts; a.nbatch = nbatch; a.seed = d_seed; a.sens = d_sens; a.adjoint = adjoint != 0;
    a.redo_list = nullptr; a.redo_count = nullptr;
    CK(cudaEventRecord(s->ev0, s->stream));
    int e = launch_sens(a, s->warps, (void *) s->stream);
    if (e != 0) { set_error(std::string("kernel launch: ") + cudaGetErrorString((cudaError_t) e)); return CUIPM_ERR_CUDA; }
    s->last_launches = 1;
    CK(cudaEventRecord(s->ev1, s->stream));
    if (sync)
    {
        CK(cudaStreamSynchronize(s->stream));
        cudaEventElapsedTime(&s->last_ms, s->ev0, s->ev1);
    }
    return CUIPM_OK;
}

extern "C" int cuipm_sens_host(cuipm_solver *s, int nbatch, const double *seed, double *sens, int adjoint, const cuipm_opts *opts)
{
    if (!s || nbatch < 0 || nbatch > s->max_batch || !seed || !sens || !opts)
    {
        set_error("cuipm_sens_host: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    CK(cudaSetDevice(s->device));
    if (nbatch == 0) return CUIPM_OK;
    const size_t bytes = sizeof(double) * s->P.sol_stride * (size_t) s->max_batch;
    if (!s->d_seed) CK(cudaMalloc(&s->d_seed, bytes));
    if (!s->d_sens) CK(cudaMalloc(&s->d_sens, bytes));
    const size_t n = sizeof(double) * s->P.sol_stride * (size_t) nbatch;
    CK(cudaMemcpyAsync(s->d_seed, seed, n, cudaMemcpyHostToDevice, s->stream));
    // the QP records of the preceding cuipm_solve_host are still resident in the solver's own device buffer
    int rc = cuipm_sens_device(s, nbatch, s->d_qp, s->d_seed, s->d_sens, adjoint, opts, 0);
    if (rc != CUIPM_OK) return rc;
    CK(cudaMemcpyAsync(sens, s->d_sens, n, cudaMemcpyDeviceToHost, s->stream));
    CK(cudaStreamSynchronize(s->stream));
    cudaEventElapsedTime(&s->last_ms, s->ev0, s->ev1);
    return CUIPM_OK;
}

// Riccati quantities of the last factorisation of QP iqp (reference getters: ocp_qp_hpipm_solver_get,
// acados/ocp_qp/ocp_qp_hpipm.c:417-478 -> d_ocp_qp_ipm_get_ric_*, external/hpipm/ocp_qp/x_ocp_qp_ipm.c:1384-1610).
//   Lr : nu x nu lower Cholesky factor of the reduced input Hessian  (L[0:nu,0:nu])
//   P  : nx x nx cost-to-go Hessian  Lxx Lxx'
//   K  : nu x nx feedback matrix     -(Lxu Luu^{-1})'
//   p  : nx      cost-to-go gradient Lxx * l_x    (valid after a factorisation: uses lrow)
//   k  : nu      feed-forward        -Luu^{-T} l_u
extern "C" int cuipm_get_ric(cuipm_solver *s, int iqp, const char *field, int stage, double *value, int size1, int size2)
{
    if (!s || iqp < 0 || iqp >= s->max_batch || stage < 0 || stage > s->P.N || !value) { set_error("cuipm_get_ric: bad arguments"); return CUIPM_ERR_INVALID; }
    const StageDesc &d = s->sd_host[stage];
    const int n = d.n, nu = d.nu, nx = d.nx;
    std::vector<double> L((size_t) n * n + 1), lrow(n + 1);
    CK(cudaSetDevice(s->device));
    CK(cudaStreamSynchronize(s->stream));
    const double *wk = s->d_work + (size_t) iqp * s->P.work_stride;
    CK(cudaMemcpy(L.data(), wk + d.w_L, sizeof(double) * n * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(lrow.data(), wk + d.w_lrow, sizeof(double) * n, cudaMemcpyDeviceToHost));
    auto Lel = [&](int i, int j) { return L[(size_t) i + (size_t) n * j]; };
    if (!std::strcmp(field, "Lr"))
    {
        if (size1 != nu || size2 != nu) { set_error("Lr: wrong size"); return CUIPM_ERR_INVALID; }
        for (int j = 0; j < nu; j++) for (int i = 0; i < nu; i++) value[i + nu * j] = i >= j ? Lel(i, j) : 0.0;
    }
    else if (!std::strcmp(field, "P"))
    {
        if (size1 != nx || size2 != nx) { set_error("P: wrong size"); return CUIPM_ERR_INVALID; }
        for (int j = 0; j < nx; j++)
            for (int i = 0; i < nx; i++)
            {
                double acc = 0.0;
                for (int c = 0; c <= (i < j ? i : j); c++) acc += Lel(nu + i, nu + c) * Lel(nu + j, nu + c);
                value[i + nx * j] = acc;
            }
    }
    else if (!std::strcmp(field, "p"))
    {
        if (size1 * size2 != nx) { set_error("p: wrong size"); return CUIPM_ERR_INVALID; }
        for (int i = 0; i < nx; i++)
        {
            double acc = 0.0;
            for (int c = 0; c <= i; c++) acc += Lel(nu + i, nu + c) * lrow[nu + c];
            value[i] = acc;
        }
    }
    else if (!std::strcmp(field, "K"))
    {
        if (size1 != nu || size2 != nx) { set_error("K: wrong size"); return CUIPM_ERR_INVALID; }
        // K = -(Lxu Luu^{-1})' : solve X Luu = Lxu row by row, K[j,i] = -X[i,j]
        for (int i = 0; i < nx; i++)
        {
            std::vector<double> x(nu);
            for (int j = nu - 1; j >= 0; j--)
            {
                double acc = Lel(nu + i, j);
                for (int c = j + 1; c < nu; c++) acc -= x[c] * Lel(c, j);
                x[j] = acc / Lel(j, j);
            }
            for (int j = 0; j < nu; j++) value[j + nu * i] = -x[j];
        }
    }
    else if (!std::strcmp(field, "k"))
    {
        if (size1 * size2 != nu) { set_error("k: wrong size"); return CUIPM_ERR_INVALID; }
        for (int j = nu - 1; j >= 0; j--)
        {
            double acc = -lrow[j];
            for (int c = j + 1; c < nu; c++) acc -= Lel(c, j) * value[c];
            value[j] = acc / Lel(j, j);
        }
    }
    else { set_error("cuipm_get_ric: unknown field"); return CUIPM_ERR_INVALID; }
    return CUIPM_OK;
}
