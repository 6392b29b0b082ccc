// barrier_bench.cu -- what does one "grid-wide sum" cost on an H100?  (tools/gpu_session.sh barrier)
//
// The persistent PCG solver needs two grid-wide reductions per iteration.  With the fluid working set in L2 the solve is bound by
// their latency, so the candidates are timed in isolation (#SM = 132 on an H100 SXM):
//   cg4       cooperative_groups grid.sync() + every block re-reads all partials       (what the solver did in round 1)
//   flat4     monotonic arrival counter (one atomic per block, acquire spin by thread 0) + every block re-reads all partials
//   flat1     the same with #SM blocks of 1024 threads
//   last3/4   one reader: the block that takes the last ticket adds the partials and publishes the total; the others poll that word
//   flat3     flat4 on the column solver's grid of 3 x #SM blocks
//   two4      two-level: blocks sharing an SM-sized group of 4 first meet on a group counter, the last of a group arrives globally;
//             the group's partials are pre-added by that last block, so that #SM instead of 4 x #SM partials are re-read
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o barrier_bench barrier_bench.cu     Run: ./barrier_bench
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>

namespace cg = cooperative_groups;

#define CHECK(x)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (x);                                                                         \
        if (e_ != cudaSuccess) { std::printf("%s failed: %s\n", #x, cudaGetErrorString(e_)); std::exit(1); } \
    } while (0)

__device__ __forceinline__ float warp_sum(float v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release(unsigned *p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float *sh) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) sh[w] = v;
    __syncthreads();
    float r = 0.f;
    if (w == 0) {
        r = lane < THREADS / 32 ? sh[lane] : 0.f;
        r = warp_sum(r);
    }
    return r; // valid in warp 0 (no trailing barrier: the callers synchronise before sh is reused)
}
// every thread of the block gets the fixed-order double sum of partials[0..n)
template <int THREADS>
__device__ __forceinline__ double all_sum(const float *partials, int n, double *shd) {
    double a = 0.0;
    for (int k = threadIdx.x; k < n; k += THREADS) a += (double)__ldcg(partials + k);
    a = warp_sum(a);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) shd[w] = a;
    __syncthreads();
    double r = 0.0;
#pragma unroll
    for (int k = 0; k < THREADS / 32; ++k) r += shd[k]; // every thread adds the warp totals in the same order
    __syncthreads();
    return r;
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS) k_cg(float *partials, int iters, double *out) {
    cg::grid_group grid = cg::this_grid();
    __shared__ float sh[THREADS / 32];
    __shared__ double shd[THREADS / 32];
    double carry = 0.0;
    for (int it = 0; it < iters; ++it) {
        const float bs = block_sum<THREADS>((float)(threadIdx.x & 3) + (float)carry * 1e-30f, sh);
        if (threadIdx.x == 0) partials[(it & 1) * gridDim.x + blockIdx.x] = bs;
        grid.sync();
        carry = all_sum<THREADS>(partials + (it & 1) * gridDim.x, gridDim.x, shd);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = carry;
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS) k_flat(float *partials, unsigned *counter, int iters, double *out) {
    __shared__ float sh[THREADS / 32];
    __shared__ double shd[THREADS / 32];
    double carry = 0.0;
    for (int it = 0; it < iters; ++it) {
        const float bs = block_sum<THREADS>((float)(threadIdx.x & 3) + (float)carry * 1e-30f, sh);
        if (threadIdx.x == 0) {
            partials[(it & 1) * gridDim.x + blockIdx.x] = bs;
            red_release(counter, 1u); // release: the partial above is visible to whoever acquires the count
            const unsigned target = (unsigned)(it + 1) * gridDim.x;
            while (ld_acquire(counter) < target) {}
        }
        __syncthreads();
        carry = all_sum<THREADS>(partials + (it & 1) * gridDim.x, gridDim.x, shd);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = carry;
}

// one reader: the block that takes the last ticket adds all partials and publishes {round, total} with a release store; the others poll
// that word only (the column solver's grid_reduce)
struct LastResult {
    unsigned round;
    float pad;
    double tot;
};
__device__ __forceinline__ void st_release(unsigned *p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
template <int THREADS>
__global__ void __launch_bounds__(THREADS) k_last(float *partials, unsigned *counter, int iters, double *out) {
    __shared__ float sh[THREADS / 32];
    __shared__ double shd[THREADS / 32];
    __shared__ int last;
    __shared__ double result;
    LastResult *res = reinterpret_cast<LastResult *>(counter + 32);
    double carry = 0.0;
    for (int it = 0; it < iters; ++it) {
        const unsigned round = (unsigned)it + 1u;
        const float bs = block_sum<THREADS>((float)(threadIdx.x & 3) + (float)carry * 1e-30f, sh);
        if (threadIdx.x == 0) {
            partials[(it & 1) * gridDim.x + blockIdx.x] = bs;
            __threadfence();
            last = atomicAdd(counter, 1u) == round * gridDim.x - 1u;
            __threadfence();
        }
        __syncthreads();
        if (last) {
            const double t = all_sum<THREADS>(partials + (it & 1) * gridDim.x, gridDim.x, shd);
            if (threadIdx.x == 0) {
                result = t;
                __stcg(&res->tot, t);
                st_release(&res->round, round);
            }
        } else if (threadIdx.x == 0) {
            while (ld_acquire(&res->round) != round) {}
            result = __ldcg(&res->tot);
        }
        __syncthreads();
        carry = result;
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = carry;
}

// groups of G consecutive blocks: the last block of a group to arrive adds the group's partials (fixed order) and arrives globally
template <int THREADS, int G>
__global__ void __launch_bounds__(THREADS) k_two(float *partials, float *group_partials, unsigned *group_counter, unsigned *counter, int iters, double *out) {
    __shared__ float sh[THREADS / 32];
    __shared__ double shd[THREADS / 32];
    const int group = blockIdx.x / G, ngroups = gridDim.x / G;
    double carry = 0.0;
    for (int it = 0; it < iters; ++it) {
        const float bs = block_sum<THREADS>((float)(threadIdx.x & 3) + (float)carry * 1e-30f, sh);
        if (threadIdx.x == 0) {
            partials[blockIdx.x] = bs;
            __threadfence();
            const unsigned arrived = atomicAdd(group_counter + group, 1u);
            if (arrived == (unsigned)(it + 1) * G - 1u) { // last of the group
                __threadfence();
                float g = 0.f;
#pragma unroll
                for (int k = 0; k < G; ++k) g += __ldcg(partials + group * G + k);
                group_partials[(it & 1) * ngroups + group] = g;
                red_release(counter, 1u);
            }
            const unsigned target = (unsigned)(it + 1) * ngroups;
            while (ld_acquire(counter) < target) {}
        }
        __syncthreads();
        carry = all_sum<THREADS>(group_partials + (it & 1) * ngroups, ngroups, shd);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = carry;
}

// thread-block clusters of CS blocks: the cluster's partials meet in block 0's shared memory (DSMEM store + hardware cluster barrier), one
// arrival per cluster on the global counter, gridDim / CS partials to re-read
template <int THREADS, int CS>
__global__ void __launch_bounds__(THREADS) k_cluster(float *cpartials, unsigned *counter, int iters, double *out) {
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ float sh[THREADS / 32];
    __shared__ double shd[THREADS / 32];
    __shared__ float cl_part[2][CS];
    const unsigned rank = cluster.block_rank();
    const int ncl = gridDim.x / CS, cid = blockIdx.x / CS;
    double carry = 0.0;
    for (int it = 0; it < iters; ++it) {
        const float bs = block_sum<THREADS>((float)(threadIdx.x & 3) + (float)carry * 1e-30f, sh);
        if (threadIdx.x == 0) {
            float *dst = cluster.map_shared_rank(&cl_part[it & 1][0], 0);
            dst[rank] = bs;
        }
        cluster.sync();
        if (threadIdx.x == 0) {
            if (rank == 0) {
                float g = 0.f;
#pragma unroll
                for (int k = 0; k < CS; ++k) g += cl_part[it & 1][k];
                cpartials[(it & 1) * ncl + cid] = g;
                red_release(counter, 1u);
            }
            const unsigned target = (unsigned)(it + 1) * ncl;
            while (ld_acquire(counter) < target) {}
        }
        __syncthreads();
        carry = all_sum<THREADS>(cpartials + (it & 1) * ncl, ncl, shd);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = carry;
}

template <int CS>
static bool launch_cluster(int blocks, float *partials, unsigned *counter, int n, double *out) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(blocks);
    cfg.blockDim = dim3(256);
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CS;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeCooperative;
    attr[1].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    cudaError_t e = cudaLaunchKernelEx(&cfg, k_cluster<256, CS>, partials, counter, n, out);
    if (e != cudaSuccess) {
        std::printf("cluster%d: launch failed: %s\n", CS, cudaGetErrorString(e));
        cudaGetLastError();
        return false;
    }
    return true;
}

template <class Launch>
static void time_it(const char *name, int blocks, int threads, int iters, Launch launch) {
    cudaEvent_t e0, e1;
    CHECK(cudaEventCreate(&e0));
    CHECK(cudaEventCreate(&e1));
    launch(20); // warm-up
    CHECK(cudaDeviceSynchronize());
    CHECK(cudaEventRecord(e0));
    launch(iters);
    CHECK(cudaEventRecord(e1));
    CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CHECK(cudaEventElapsedTime(&ms, e0, e1));
    std::printf("%-10s %4d blocks x %4d threads: %7.3f us per grid-wide sum\n", name, blocks, threads, 1e3f * ms / iters);
}

int main() {
    int dev = 0, sms = 0;
    CHECK(cudaGetDevice(&dev));
    CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    float *partials, *gpart;
    unsigned *counters;
    double *out;
    CHECK(cudaMalloc(&partials, 4 * 4096 * sizeof(float)));
    CHECK(cudaMalloc(&gpart, 4 * 4096 * sizeof(float)));
    CHECK(cudaMalloc(&counters, 4096 * sizeof(unsigned)));
    CHECK(cudaMalloc(&out, sizeof(double)));
    const int iters = 2000;
    auto reset = [&] { CHECK(cudaMemset(counters, 0, 4096 * sizeof(unsigned))); };
    for (int per_sm = 3; per_sm <= 4; ++per_sm) { // three blocks per SM: the column solver's grid
        const int blocks = sms * per_sm;
        time_it(per_sm == 3 ? "flat3" : "flat4", blocks, 256, iters, [&](int n) {
            reset();
            unsigned *c = counters;
            void *args[] = {&partials, &c, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_flat<256>, dim3(blocks), dim3(256), args, 0, 0));
        });
        time_it(per_sm == 3 ? "last3" : "last4", blocks, 256, iters, [&](int n) {
            reset();
            unsigned *c = counters;
            void *args[] = {&partials, &c, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_last<256>, dim3(blocks), dim3(256), args, 0, 0));
        });
    }
    {
        const int blocks = sms * 4;
        time_it("cg4", blocks, 256, iters, [&](int n) {
            void *args[] = {&partials, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_cg<256>, dim3(blocks), dim3(256), args, 0, 0));
        });
        time_it("two4", blocks, 256, iters, [&](int n) {
            reset();
            unsigned *gc = counters + 8, *c = counters;
            void *args[] = {&partials, &gpart, &gc, &c, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_two<256, 4>, dim3(blocks), dim3(256), args, 0, 0));
        });
    }
    {
        const int blocks = sms * 4;
        int ncl = 0;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(blocks);
        cfg.blockDim = dim3(256);
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 4;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        if (cudaOccupancyMaxActiveClusters(&ncl, k_cluster<256, 4>, &cfg) == cudaSuccess) std::printf("max co-resident clusters of 4 x 256 threads: %d (need %d)\n", ncl, blocks / 4);
        cudaGetLastError();
        if (ncl >= blocks / 4) {
            bool ok = true;
            time_it("cluster4", blocks, 256, iters, [&](int n) {
                reset();
                if (ok) ok = launch_cluster<4>(blocks, partials, counters, n, out);
            });
        }
        attr[0].val.clusterDim.x = 2;
        if (cudaOccupancyMaxActiveClusters(&ncl, k_cluster<256, 2>, &cfg) == cudaSuccess) std::printf("max co-resident clusters of 2 x 256 threads: %d (need %d)\n", ncl, blocks / 2);
        cudaGetLastError();
        if (ncl >= blocks / 2) {
            bool ok = true;
            time_it("cluster2", blocks, 256, iters, [&](int n) {
                reset();
                if (ok) ok = launch_cluster<2>(blocks, partials, counters, n, out);
            });
        }
    }
    {
        const int blocks = sms;
        time_it("cg1", blocks, 1024, iters, [&](int n) {
            void *args[] = {&partials, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_cg<1024>, dim3(blocks), dim3(1024), args, 0, 0));
        });
        time_it("flat1", blocks, 1024, iters, [&](int n) {
            reset();
            unsigned *c = counters;
            void *args[] = {&partials, &c, &n, &out};
            CHECK(cudaLaunchCooperativeKernel((const void *)k_flat<1024>, dim3(blocks), dim3(1024), args, 0, 0));
        });
    }
    double h = 0;
    CHECK(cudaMemcpy(&h, out, sizeof(double), cudaMemcpyDeviceToHost));
    std::printf("(checksum %g)\n", h);
    return 0;
}
