// Microbenchmark: attainable random-line gather bandwidth on H100 (what bounds the hash gather?).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o randgather randgather.cu && ./randgather
// Each thread issues ILP independent 16-byte loads per iteration; 8 consecutive lanes cover one
// 128-byte line (LINE=128) or 4 lanes cover 64 bytes (LINE=64), line index = hash(counter).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x;
}

template <int ILP, int LANES_PER_LINE>
__global__ void gather_kernel(const uint4 *__restrict__ tab, uint32_t n_lines, int iters, uint4 *out, uint32_t seed) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t group = tid / LANES_PER_LINE, sub = tid % LANES_PER_LINE;
    uint4 acc = make_uint4(0, 0, 0, 0);
    uint32_t ctr = group * 7919u + seed;
    for (int it = 0; it < iters; ++it) {
        uint4 v[ILP];
#pragma unroll
        for (int i = 0; i < ILP; ++i) {
            uint32_t line = hash32(ctr + i * 0x9e3779b9u + it * 0x85ebca6bu) % n_lines;
            v[i] = __ldg(tab + (size_t)line * 8 + sub);
        }
#pragma unroll
        for (int i = 0; i < ILP; ++i) { acc.x ^= v[i].x; acc.y += v[i].y; acc.z ^= v[i].z; acc.w += v[i].w; }
    }
    if (acc.x == 0x12345678u) out[tid] = acc;
}

template <int ILP, int LPL>
void run(const uint4 *tab, uint32_t n_lines, uint4 *out, int blocks_per_sm, int threads, const char *name) {
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int blocks = sms * blocks_per_sm;
    int iters = 200;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    gather_kernel<ILP, LPL><<<blocks, threads>>>(tab, n_lines, 20, out, 1);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    gather_kernel<ILP, LPL><<<blocks, threads>>>(tab, n_lines, iters, out, 2);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double bytes = (double)blocks * threads * iters * ILP * 16.0;
    printf("%-10s ILP=%2d lanes/line=%d warps/SM=%2d  in-flight/SM=%6.1f KB  %8.1f GB/s  (%.3f ms)\n", name, ILP, LPL,
           blocks_per_sm * threads / 32, blocks_per_sm * threads * ILP * 16.0 / 1024, bytes / ms / 1e6, ms);
}

int main() {
    const size_t bytes = 806ull << 20;
    uint4 *tab, *out;
    cudaMalloc(&tab, bytes); cudaMemset(tab, 1, bytes); cudaMalloc(&out, 64 << 20);
    uint32_t n_lines = bytes / 128;
    printf("table %zu MB, %u lines of 128 B\n", bytes >> 20, n_lines);
    run<1, 8>(tab, n_lines, out, 8, 256, "128B");
    run<2, 8>(tab, n_lines, out, 8, 256, "128B");
    run<4, 8>(tab, n_lines, out, 8, 256, "128B");
    run<8, 8>(tab, n_lines, out, 8, 256, "128B");
    run<16, 8>(tab, n_lines, out, 8, 256, "128B");
    run<8, 8>(tab, n_lines, out, 4, 256, "128B");
    run<8, 8>(tab, n_lines, out, 2, 256, "128B");
    run<4, 8>(tab, n_lines, out, 2, 256, "128B");
    run<8, 4>(tab, n_lines, out, 8, 256, "64B-half");
    run<16, 4>(tab, n_lines, out, 8, 256, "64B-half");
    // smaller tables: L2-resident (64 MB) and the 5 dense levels (68 MB) case
    uint32_t small = (64u << 20) / 128;
    run<8, 8>(tab, small, out, 8, 256, "L2-64MB");
    run<8, 8>(tab, (256u << 20) / 128, out, 8, 256, "256MB");
    return 0;
}
