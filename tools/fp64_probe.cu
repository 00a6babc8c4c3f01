// fp64_probe.cu -- development aid: non-fused FP64 issue rate and dependent-issue latency of one GPU, the
// denominator of the BAQ roofline (SURVEY.md 8d: BAQ must not contract a*b+c, so an FMA slot carries ONE operation).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o tools/_build/fp64_probe tools/fp64_probe.cu
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

template <int ILP>
__global__ void k_chain(double *out, int iters, double a, double b)
{
    double x[ILP];
#pragma unroll
    for (int j = 0; j < ILP; ++j) x[j] = threadIdx.x * 1e-9 + j;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < ILP; ++j) x[j] = x[j] * a + b;       // DMUL then DADD (no contraction)
    }
    double s = 0;
#pragma unroll
    for (int j = 0; j < ILP; ++j) s += x[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int ILP>
static void run(int blocks_per_sm, int threads, int n_sm, double *d)
{
    const int iters = 20000;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k_chain<ILP><<<n_sm * blocks_per_sm, threads>>>(d, 100, 1.0000001, 1e-9);
    cudaEventRecord(e0);
    k_chain<ILP><<<n_sm * blocks_per_sm, threads>>>(d, iters, 1.0000001, 1e-9);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double ops = 2.0 * ILP * iters * (double)threads * blocks_per_sm * n_sm;
    printf("ILP %2d  warps/SM %3d : %8.3f ms  %7.3f Top/s  (%.2f cycles per dependent op pair at 1.965 GHz per warp-chain)\n", ILP,
           blocks_per_sm * threads / 32, ms, ops / ms / 1e9, ms * 1e-3 * 1.965e9 / iters);
}

int main()
{
    int n_sm; cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
    double *d; cudaMalloc(&d, (size_t)n_sm * 64 * 1024 * 8);
    run<1>(1, 32, n_sm, d);      // one warp per SM, one chain: dependent latency of DMUL+DADD
    run<1>(1, 128, n_sm, d);
    run<2>(1, 128, n_sm, d);
    run<4>(1, 128, n_sm, d);
    run<8>(1, 128, n_sm, d);
    run<4>(2, 128, n_sm, d);
    run<4>(3, 128, n_sm, d);
    run<8>(2, 128, n_sm, d);
    run<8>(4, 128, n_sm, d);
    run<8>(8, 128, n_sm, d);
    run<16>(4, 128, n_sm, d);
    return 0;
}
