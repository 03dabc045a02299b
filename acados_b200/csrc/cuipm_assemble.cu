// cuipm_assemble.cu -- cuipm_xcond_assemble_device: full-shape QP records written on the device from strided per-field sources
// (torch tensors, slices and transposes of them, or one value broadcast to the batch), so that QP data that already lives on the
// GPU reaches the xcond chain without a trip through the host.  The kernel body is cuipm_assemble_core.h; here are its CUDA
// execution policy, the launch and the host side: the source table is checked and built on the host each call, copied to the
// object's device tables on its stream, and read by the one kernel that follows.
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "cuipm.h"
#include "cuipm_assemble_core.h"
#include "cuipm_internal.h"

using namespace cuipm;
using namespace cuipm_asm;

namespace {
constexpr int ASM_THREADS = 256;

struct GridExec
{
    template <class F> __device__ void for_each(long long n, F f)
    {
        const long long step = (long long) gridDim.x * blockDim.x;
        for (long long t = (long long) blockIdx.x * blockDim.x + threadIdx.x; t < n; t += step) f(t);
    }
};

__global__ void __launch_bounds__(ASM_THREADS) assemble_kernel(const Plan P)
{
    GridExec ex;
    assemble(ex, P);
}
}  // namespace

int asm_init(cuipm_xcond *x, const cuipm_shape *full)
{
    std::vector<Stage> st;
    if (!stage_table(full, x->lf, st)) { set_error("cuipm_xcond_create: a record needs offsets beyond 32 bits"); return CUIPM_ERR_TOO_LARGE; }
    x->asm_st = new Stage[st.size()];
    std::memcpy(x->asm_st, st.data(), sizeof(Stage) * st.size());
    return CUIPM_OK;
}

void asm_free(cuipm_xcond *x)
{
    delete[] x->asm_st;
    x->asm_st = nullptr;
    cudaFree(x->d_asm);
    x->d_asm = nullptr;
}

extern "C" int cuipm_xcond_assemble_device(cuipm_xcond *x, int nbatch, const cuipm_src *src, int nsrc, double *d_qp_full, int sync)
{
    if (!x || nbatch < 0 || nbatch > x->max_batch || nsrc < 0 || (nsrc > 0 && !src) || !d_qp_full)
    {
        set_error("cuipm_xcond_assemble_device: bad arguments (nbatch must be <= max_batch)");
        return CUIPM_ERR_INVALID;
    }
    const int N = x->lf->N;
    std::vector<Stage> st(x->asm_st, x->asm_st + N + 1);
    std::vector<Src> srcs;
    const std::string err = enter_sources(st, src, nsrc, srcs);
    if (!err.empty()) { set_error("cuipm_xcond_assemble_device: " + err); return CUIPM_ERR_INVALID; }
    if (nbatch == 0 || x->lf->qp_stride == 0) return CUIPM_OK;
    // one host blob: the sources (8-byte aligned), then the stage table
    const size_t src_bytes = sizeof(Src) * srcs.size(), bytes = src_bytes + sizeof(Stage) * st.size();
    std::vector<unsigned char> blob(bytes);
    if (src_bytes) std::memcpy(blob.data(), srcs.data(), src_bytes);
    std::memcpy(blob.data() + src_bytes, st.data(), sizeof(Stage) * st.size());
    CK(cudaSetDevice(x->device));
    cudaStream_t s = (cudaStream_t) cuipm_stream(x->solver);
    if (bytes > x->asm_bytes)
    {
        CK(cudaStreamSynchronize(s));                    // an earlier launch may still read the old tables
        CK(cudaFree(x->d_asm));
        x->d_asm = nullptr; x->asm_bytes = 0;
        CK(cudaMalloc(&x->d_asm, bytes));
        x->asm_bytes = bytes;
    }
    // from pageable memory: the call returns once `blob` has been staged, so it may go out of scope
    CK(cudaMemcpyAsync(x->d_asm, blob.data(), bytes, cudaMemcpyHostToDevice, s));
    Plan P;
    P.src = (const Src *) x->d_asm;
    P.st = (const Stage *) ((const unsigned char *) x->d_asm + src_bytes);
    P.N = N;
    P.qp_stride = (unsigned) x->lf->qp_stride;
    P.total = (long long) nbatch * (long long) x->lf->qp_stride;
    P.out = d_qp_full;
    const long long blocks = (P.total + ASM_THREADS - 1) / ASM_THREADS;
    assemble_kernel<<<(unsigned) (blocks < (1 << 20) ? blocks : (1 << 20)), ASM_THREADS, 0, s>>>(P);
    CK(cudaGetLastError());
    if (sync) CK(cudaStreamSynchronize(s));
    return CUIPM_OK;
}
