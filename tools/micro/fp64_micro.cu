// FP64 pipe characterisation of the GPU: dependent-DFMA latency, and DFMA throughput per SM as a function of
// resident warps per scheduler and independent chains per thread (ILP).  Drives the occupancy / ILP decisions of k_rao_fused.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/fp64_micro.bin tools/micro/fp64_micro.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int ILP>
__global__ void k_chain(double *out, int iters, long long *cycles)
{
    double a[ILP], b = 1.0000001, c = 1e-9;
    for (int i = 0; i < ILP; i++) a[i] = threadIdx.x * 1e-3 + i;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 16; u++)
#pragma unroll
            for (int i = 0; i < ILP; i++) a[i] = fma(a[i], b, c);
    }
    long long t1 = clock64();
    double s = 0;
    for (int i = 0; i < ILP; i++) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

__global__ void k_sqrt(double *out, int iters, long long *cycles)
{
    double a = 2.0 + threadIdx.x;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) a = sqrt(a) + 1.5;
    long long t1 = clock64();
    out[threadIdx.x] = a;
    if (threadIdx.x == 0) *cycles = t1 - t0;
}
__global__ void k_div(double *out, int iters, long long *cycles)
{
    double a = 2.0 + threadIdx.x;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) a = 1.0 / a + 1.5;
    long long t1 = clock64();
    out[threadIdx.x] = a;
    if (threadIdx.x == 0) *cycles = t1 - t0;
}
__global__ void k_lds(double *out, int iters, long long *cycles)
{
    __shared__ int idx[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) idx[i] = (i * 33 + 7) & 1023;
    __syncthreads();
    int j = threadIdx.x;
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) j = idx[j];
    long long t1 = clock64();
    out[threadIdx.x] = j;
    if (threadIdx.x == 0) *cycles = t1 - t0;
}

template <int ILP>
static void run(int warps_per_sched, int sms, double *out, long long *cyc)
{
    const int iters = 2000;
    const int threads = 32 * 4 * warps_per_sched;      // one CTA per SM, 4 schedulers
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    k_chain<ILP><<<sms, threads>>>(out, 10, cyc);
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    k_chain<ILP><<<sms, threads>>>(out, iters, cyc);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    long long c = 0;
    cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const double fmas = (double)iters * 16 * ILP * threads;           // per SM
    printf("warps/sched %2d ILP %d : %.2f DFMA/clk/SM (of 64), %.2f cycles per dependent DFMA step, %.1f TFLOP/s\n", warps_per_sched, ILP,
           fmas / c, (double)c / (iters * 16.0), 2.0 * fmas * sms / (ms * 1e-3) * 1e-12);
}

int main()
{
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    double *out; long long *cyc;
    cudaMalloc(&out, 1 << 22); cudaMalloc(&cyc, 8);
    long long c = 0;
    k_chain<1><<<1, 32>>>(out, 2000, cyc); cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("dependent DFMA latency (1 warp): %.2f cycles\n", c / 32000.0);
    k_sqrt<<<1, 32>>>(out, 2000, cyc); cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("dependent sqrt(double)+add: %.1f cycles\n", c / 2000.0);
    k_div<<<1, 32>>>(out, 2000, cyc); cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("dependent 1/x (double)+add: %.1f cycles\n", c / 2000.0);
    k_lds<<<1, 32>>>(out, 20000, cyc); cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("dependent LDS.32 latency: %.1f cycles\n", c / 20000.0);
    for (int w : {1, 2, 3, 4, 8}) {
        run<1>(w, sms, out, cyc); run<2>(w, sms, out, cyc); run<4>(w, sms, out, cyc); run<8>(w, sms, out, cyc);
    }
    return 0;
}
