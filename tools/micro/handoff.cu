// Micro-benchmark: latency of a warp-to-warp hand-off inside one CTA: named barriers vs shared-memory flags vs mbarriers.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void nb_arrive(int id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void nb_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__global__ void pingpong_bar(int n, long long *out, double *sink)
{
    __shared__ double box[2][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double v = lane;
    long long t0 = clock64();
    for (int j = 0; j < n; j++) {
        const int sl = j & 1;
        if (warp == 0) { box[0][lane] = v; __threadfence_block(); nb_arrive(1 + sl); nb_sync(3 + sl); v = box[1][lane] + 1.0; }
        else { nb_sync(1 + sl); const double x = box[0][lane]; box[1][lane] = x * 1.0000001; __threadfence_block(); nb_arrive(3 + sl); }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[0] = (t1 - t0);
    sink[threadIdx.x] = v;
}
__global__ void pingpong_flag(int n, long long *out, double *sink)
{
    __shared__ double box[2][32];
    __shared__ volatile int flag[2][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < 32) { flag[0][lane] = 0; flag[1][lane] = 0; }
    __syncthreads();
    double v = lane;
    long long t0 = clock64();
    for (int j = 1; j <= n; j++) {
        if (warp == 0) { box[0][lane] = v; __threadfence_block(); flag[0][lane] = j; while (flag[1][lane] != j) {} __threadfence_block(); v = box[1][lane] + 1.0; }
        else { while (flag[0][lane] != j) {} __threadfence_block(); const double x = box[0][lane]; box[1][lane] = x * 1.0000001; __threadfence_block(); flag[1][lane] = j; }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[0] = (t1 - t0);
    sink[threadIdx.x] = v;
}
__global__ void chain_fp64(int n, long long *out, double *sink)
{
    double v = threadIdx.x * 1e-3 + 1.0;
    long long t0 = clock64();
    for (int j = 0; j < n; j++) { v = v * 1.0000001 + 1e-9; v = v * 0.9999999 + 1e-9; v = v * 1.0000001 + 1e-9; v = v * 0.9999999 + 1e-9; }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[0] = (t1 - t0);
    sink[threadIdx.x] = v;
}
int main()
{
    long long *d; double *s; long long h;
    cudaMalloc(&d, 8); cudaMalloc(&s, 64 * 8);
    const int n = 100000;
    for (int rep = 0; rep < 2; rep++) {
        pingpong_bar<<<1, 64>>>(n, d, s); cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        printf("named barriers : %.1f cycles per round trip (two hand-offs)\n", (double)h / n);
        pingpong_flag<<<1, 64>>>(n, d, s); cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        printf("smem flags     : %.1f cycles per round trip (two hand-offs)\n", (double)h / n);
        chain_fp64<<<1, 32>>>(n, d, s); cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        printf("dependent DFMA (fmad on: 4 per iter): %.2f cycles per dependent op\n", (double)h / n / 4);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
