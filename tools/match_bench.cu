// Cost of match.any.sync (SASS MATCH.ANY) next to SHFL and REDG on sm_90a: the scatter kernels find the lanes that share a dual cell with it.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/match_bench tools/match_bench.cu && ./tools/match_bench
// Prints SM cycles per warp-instruction with all warps of a full grid issuing back to back (throughput), for key patterns with 1 .. 32 distinct
// values per warp, and the same loop with one SHFL.IDX instead.
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void k(int distinct, int iters, unsigned *out, long long *cycles) {
    const int lane = threadIdx.x & 31;
    int key = (lane * distinct) >> 5; // `distinct` different values per warp, equal keys adjacent
    if (MODE == 2) key = lane % distinct; // equal keys interleaved
    unsigned acc = 0;
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < iters; ++i) {
        if (MODE == 1) acc += __shfl_sync(0xffffffffu, key + (int)acc, (lane + 1) & 31);
        else acc += __match_any_sync(0xffffffffu, key + (int)(acc & 0u)) & 1u; // the & 0 keeps a dependency without changing the key
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

int main() {
    const int blocks = 132 * 4, threads = 256, iters = 4096;
    unsigned *out;
    long long *cyc, h[132 * 4];  // four blocks on each of the 132 SMs of an H100 SXM
    cudaMalloc(&out, blocks * threads * sizeof(unsigned));
    cudaMalloc(&cyc, blocks * sizeof(long long));
    auto run = [&](const char *name, int mode, int distinct) {
        for (int rep = 0; rep < 2; ++rep) {
            if (mode == 0) k<0><<<blocks, threads>>>(distinct, iters, out, cyc);
            if (mode == 1) k<1><<<blocks, threads>>>(distinct, iters, out, cyc);
            if (mode == 2) k<2><<<blocks, threads>>>(distinct, iters, out, cyc);
            cudaDeviceSynchronize();
        }
        cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        double s = 0;
        for (int b = 0; b < blocks; ++b) s += (double)h[b];
        // 4 blocks x 8 warps per SM issue concurrently: cycles per warp-instruction per SM = block cycles / iters / 32 warps
        std::printf("%-26s distinct %2d: %7.1f cycles per instruction in one warp's stream, %6.2f SM-cycles per warp-instruction (32 warps per SM)\n", name, distinct,
                    s / blocks / iters, s / blocks / iters / 32.0);
    };
    for (int d : {1, 2, 4, 8, 16, 32}) run("match.any (adjacent keys)", 0, d);
    for (int d : {8, 16}) run("match.any (interleaved)", 2, d);
    run("shfl.idx", 1, 1);
    std::printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
