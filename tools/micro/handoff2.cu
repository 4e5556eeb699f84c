// Micro-benchmark (next experiments for the K1a pipeline): does the named-barrier hop latency depend on WHERE the two warps
// sit (same SM sub-partition = warp ids equal mod 4, or different ones), and is an mbarrier hand-off any faster?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o handoff2 handoff2.cu && ./handoff2
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ void nb_arrive(int id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void nb_sync(int id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count)); }
__device__ __forceinline__ void mbar_arrive(uint64_t *b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *b, unsigned parity)
{
    asm volatile("{\n.reg .pred p;\nW: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D;\nbra W;\nD:\n}" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}

// warps wa and wb of a 256-thread CTA play ping-pong; the others leave at once
__global__ void pingpong_bar(int wa, int wb, int n, long long *out, double *sink)
{
    __shared__ double box[2][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp != wa && warp != wb) return;
    double v = lane;
    long long t0 = clock64();
    for (int j = 0; j < n; j++) {
        const int sl = j & 1;
        if (warp == wa) { box[0][lane] = v; __threadfence_block(); nb_arrive(1 + sl); nb_sync(3 + sl); v = box[1][lane] + 1.0; }
        else { nb_sync(1 + sl); const double x = box[0][lane]; box[1][lane] = x * 1.0000001; __threadfence_block(); nb_arrive(3 + sl); }
    }
    long long t1 = clock64();
    if (warp == wa && lane == 0) out[0] = (t1 - t0);
    sink[threadIdx.x] = v;
}
__global__ void pingpong_mbar(int wa, int wb, int n, long long *out, double *sink)
{
    __shared__ double box[2][32];
    __shared__ uint64_t bars[2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { mbar_init(&bars[0], 32); mbar_init(&bars[1], 32); }
    __syncthreads();
    if (warp != wa && warp != wb) return;
    double v = lane;
    long long t0 = clock64();
    for (int j = 0; j < n; j++) {
        const unsigned ph = j & 1;
        if (warp == wa) { box[0][lane] = v; mbar_arrive(&bars[0]); mbar_wait(&bars[1], ph); v = box[1][lane] + 1.0; }
        else { mbar_wait(&bars[0], ph); const double x = box[0][lane]; box[1][lane] = x * 1.0000001; mbar_arrive(&bars[1]); }
    }
    long long t1 = clock64();
    if (warp == wa && lane == 0) out[0] = (t1 - t0);
    sink[threadIdx.x] = v;
}
int main()
{
    long long *d; double *s; long long h;
    cudaMalloc(&d, 8); cudaMalloc(&s, 256 * 8);
    const int n = 100000;
    const int pairs[4][2] = {{0, 1}, {0, 4}, {1, 2}, {3, 7}};
    for (int k = 0; k < 4; k++) {
        const int wa = pairs[k][0], wb = pairs[k][1];
        pingpong_bar<<<1, 256>>>(wa, wb, n, d, s); cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        printf("warps %d<->%d (%s sub-partition)  named barriers: %.1f cycles per hop", wa, wb, (wa & 3) == (wb & 3) ? "same" : "different", (double)h / n / 2);
        pingpong_mbar<<<1, 256>>>(wa, wb, n, d, s); cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        printf("   mbarrier: %.1f cycles per hop\n", (double)h / n / 2);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
