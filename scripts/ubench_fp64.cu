// ubench_fp64.cu -- FP64 micro-benchmarks on H100 (sm_90a): DFMA and DMMA (mma.sync m8n8k4.f64) issue rates as a
// function of resident warps per SM and independent chains per thread, dependent-issue latencies of DFMA / rsqrt /
// shared-memory loads: the measured rates, to set beside the data-sheet FP64 peak bench.py's roofline divides by.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

template <int ILP>
__global__ void k_dfma(double *out, int iters, double a, double b)
{
    double acc[ILP];
#pragma unroll
    for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++)
    {
#pragma unroll
        for (int i = 0; i < ILP; i++) acc[i] = fma(acc[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += acc[i];
    if (s == 123.456) out[0] = s;
}

template <int ILP>
__global__ void k_dmma(double *out, int iters, double a, double b)
{
    double c0[ILP], c1[ILP];
#pragma unroll
    for (int i = 0; i < ILP; i++) { c0[i] = threadIdx.x; c1[i] = i; }
    for (int it = 0; it < iters; it++)
    {
#pragma unroll
        for (int i = 0; i < ILP; i++)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c0[i]), "+d"(c1[i]) : "d"(a), "d"(b));
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += c0[i] + c1[i];
    if (s == 123.456) out[0] = s;
}

__global__ void k_lat(double *out, long long *cyc, int iters, double a, double b)
{
    __shared__ double sm[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = (double) ((i * 7 + 1) & 1023);
    __syncthreads();
    double x = a;
    long long t0 = clock64();
    for (int i = 0; i < iters; i++) x = fma(x, a, b);
    long long t1 = clock64();
    double y = a + 1.5;
    for (int i = 0; i < iters; i++) y = rsqrt(y) + b;
    long long t2 = clock64();
    int idx = threadIdx.x;
    for (int i = 0; i < iters; i++) idx = (int) sm[idx & 1023];
    long long t3 = clock64();
    double z = a + 2.5;
    for (int i = 0; i < iters; i++) z = 1.0 / sqrt(z) + b;
    long long t4 = clock64();
    double w = a;
    for (int i = 0; i < iters; i++) w = __shfl_xor_sync(0xffffffffu, w, 1) + b;
    long long t5 = clock64();
    if (threadIdx.x == 0)
    {
        cyc[0] = t1 - t0; cyc[1] = t2 - t1; cyc[2] = t3 - t2; cyc[3] = t4 - t3; cyc[4] = t5 - t4;
    }
    out[threadIdx.x] = x + y + idx + z + w;
}

template <typename F>
float timeit(F f)
{
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    f();
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    f();
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

int main()
{
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    int sms = p.multiProcessorCount;
    printf("device %s SMs %d clock %d kHz\n", p.name, sms, p.clockRate);
    double *out; long long *cyc;
    CK(cudaMalloc(&out, 1 << 20)); CK(cudaMalloc(&cyc, 64));
    const int iters = 20000;
    printf("# DFMA: warps/SM, ILP, TFLOP/s\n");
    for (int wps : {4, 8, 16, 32, 64})
    {
        int threads = 128, blocks = sms * wps / 4;
        float ms;
        ms = timeit([&] { k_dfma<1><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dfma warps %2d ilp 1  %.2f TF\n", wps, 2.0 * iters * 1 * threads * blocks / ms * 1e-9);
        ms = timeit([&] { k_dfma<4><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dfma warps %2d ilp 4  %.2f TF\n", wps, 2.0 * iters * 4 * threads * blocks / ms * 1e-9);
        ms = timeit([&] { k_dfma<16><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dfma warps %2d ilp 16 %.2f TF\n", wps, 2.0 * iters * 16 * threads * blocks / ms * 1e-9);
    }
    printf("# DMMA m8n8k4: warps/SM, ILP, TFLOP/s\n");
    for (int wps : {4, 8, 16, 32})
    {
        int threads = 128, blocks = sms * wps / 4;
        float ms;
        ms = timeit([&] { k_dmma<1><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dmma warps %2d ilp 1  %.2f TF\n", wps, 2.0 * 256 * iters * 1 * (threads / 32) * blocks / ms * 1e-9);
        ms = timeit([&] { k_dmma<4><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dmma warps %2d ilp 4  %.2f TF\n", wps, 2.0 * 256 * iters * 4 * (threads / 32) * blocks / ms * 1e-9);
        ms = timeit([&] { k_dmma<8><<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); });
        printf("dmma warps %2d ilp 8  %.2f TF\n", wps, 2.0 * 256 * iters * 8 * (threads / 32) * blocks / ms * 1e-9);
    }
    k_lat<<<1, 32>>>(out, cyc, 4096, 1.0000001, 1e-9);
    CK(cudaDeviceSynchronize());
    long long h[5];
    CK(cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost));
    printf("latency cycles: dfma %.1f  rsqrt(double)+add %.1f  lds+cvt %.1f  1/sqrt+add %.1f  shfl64+add %.1f\n", h[0] / 4096.0, h[1] / 4096.0,
           h[2] / 4096.0, h[3] / 4096.0, h[4] / 4096.0);
    return 0;
}
