// grid_reduce.cuh -- the arrival-counter reduction of the persistent solvers (pcg.cu column solver, viscosity_kernels.cu).
#pragma once
#include "common.cuh"

namespace blub {
namespace {

constexpr int PCG_THREADS = 256; // threads per block of every persistent solver
__device__ __forceinline__ int linear_tid() { return threadIdx.y * blockDim.x + threadIdx.x; }

// the guarded divisions that form alpha and beta: a zero system gives zero
constexpr float PCG_EPSILON = 1e-10f; // pressure_reduce.comp:33
__device__ __forceinline__ float guarded_div(float num, float den) { // pressure_reduce.comp:73-80
    return num / (den + (den < 0.0f ? -PCG_EPSILON : PCG_EPSILON));
}

// Grid-wide reduction of the column solver.  With the fluid working set in L2 the solve is bound by the latency of these two
// reductions per iteration, so they are kept lean
// (tools/barrier_bench.cu compares it with cooperative_groups grid.sync() + re-read):
// one shared-memory pass forms the block's sum and maximum, thread 0 publishes them, arrives on a monotonically increasing counter
// (red.release) and spins with ld.acquire until everybody of this round has arrived; then every block re-reads all partials and adds
// them in the same fixed order in fp64: bit-identical scalars in all blocks, deterministic run to run, no broadcast step.
// Partial buffers alternate between the two phases of an iteration, so a fast block never overwrites what a slow one still reads.
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_u32(unsigned *p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
struct ReduceScratch {
    float sh[2 * (PCG_THREADS / 32)];
    double shd[PCG_THREADS / 32];
};
// First half of both forms: the block's sum (and maximum) formed in one shared-memory pass, published by thread 0 into psum / pmax
// [blockIdx.x], which then arrives on the counter for round `round` (counted here).  TICKET = false: release, then wait with acquire until
// everybody of the round has arrived.  TICKET = true: nobody waits; returns true (block-uniform) in the block that arrived last.
template <bool WITH_MAX, bool TICKET>
__device__ __forceinline__ bool publish_and_arrive(unsigned *counter, unsigned &round, float *psum, float *pmax, float acc, float err, ReduceScratch &sc,
                                                   int *sh_last) {
    constexpr int NW = PCG_THREADS / 32;
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5;
    acc = warp_sum(acc);
    if (WITH_MAX) err = warp_max(err);
    if (lane == 0) {
        sc.sh[w] = acc;
        if (WITH_MAX) sc.sh[NW + w] = err;
    }
    __syncthreads();
    round += 1u;
    if (tid == 0) {
        float bs = 0.0f, bm = 0.0f;
#pragma unroll
        for (int k = 0; k < NW; ++k) {
            bs += sc.sh[k];
            if (WITH_MAX) bm = fmaxf(bm, sc.sh[NW + k]);
        }
        psum[blockIdx.x] = bs;
        if (WITH_MAX) pmax[blockIdx.x] = bm;
        if (TICKET) {
            __threadfence(); // release: the partials (and this block's pushes into the neighbours' ghost planes) before the ticket
            const unsigned ticket = atomicAdd(counter, 1u);
            *sh_last = ticket == round * gridDim.x - 1u ? 1 : 0;
            __threadfence(); // acquire (matters in the last block): everybody else's partials are visible from here on
        } else {
            red_release_u32(counter, 1u);
            const unsigned target = round * gridDim.x;
            while (ld_acquire_u32(counter) < target) {}
        }
    }
    __syncthreads();
    return TICKET && *sh_last;
}
// Every thread: the partials of all blocks added in the same fixed order in fp64 (and their maximum).
template <bool WITH_MAX>
__device__ __forceinline__ void read_partials(const float *psum, const float *pmax, ReduceScratch &sc, double &tot, float &gmax) {
    constexpr int NW = PCG_THREADS / 32;
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5;
    double a = 0.0;
    float m = 0.0f;
    for (int k = tid; k < (int)gridDim.x; k += PCG_THREADS) {
        a += (double)__ldcg(psum + k);
        if (WITH_MAX) m = fmaxf(m, __ldcg(pmax + k));
    }
    a = warp_sum(a);
    if (WITH_MAX) m = warp_max(m);
    if (lane == 0) {
        sc.shd[w] = a;
        if (WITH_MAX) sc.sh[w] = m;
    }
    __syncthreads();
    double t = 0.0;
    float mm = 0.0f;
#pragma unroll
    for (int k = 0; k < NW; ++k) { // every thread adds the warp totals in the same order
        t += sc.shd[k];
        if (WITH_MAX) mm = fmaxf(mm, sc.sh[k]);
    }
    tot = t;
    gmax = mm;
}
template <bool WITH_MAX>
__device__ __forceinline__ void grid_reduce(unsigned *counter, unsigned &round, float *psum, float *pmax, float acc, float err, ReduceScratch &sc, double &tot,
                                            float &gmax) {
    publish_and_arrive<WITH_MAX, false>(counter, round, psum, pmax, acc, err, sc, nullptr);
    read_partials<WITH_MAX>(psum, pmax, sc, tot, gmax);
    __syncthreads(); // the scratch is reused by the next reduction
}

// The same reduction for N sums and N maxima in one round (the viscosity solve advances its three components together).  part: 2 * N *
// gridDim.x floats, value j of block b at part[j * gridDim.x + b], sums first; the caller alternates two such buffers between rounds.
template <int N> struct ReduceScratchN {
    float sh[2 * N * (PCG_THREADS / 32)];
    double shd[N * (PCG_THREADS / 32)];
};
template <int N>
__device__ __forceinline__ void grid_reduce_n(unsigned *counter, unsigned &round, float *part, const float (&acc)[N], const float (&err)[N],
                                              ReduceScratchN<N> &sc, double (&tot)[N], float (&gmax)[N]) {
    constexpr int NW = PCG_THREADS / 32;
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5, nb = (int)gridDim.x;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const float a = warp_sum(acc[j]), m = warp_max(err[j]);
        if (lane == 0) {
            sc.sh[j * NW + w] = a;
            sc.sh[(N + j) * NW + w] = m;
        }
    }
    __syncthreads();
    round += 1u;
    if (tid == 0) {
#pragma unroll
        for (int j = 0; j < N; ++j) {
            float bs = 0.0f, bm = 0.0f;
#pragma unroll
            for (int k = 0; k < NW; ++k) {
                bs += sc.sh[j * NW + k];
                bm = fmaxf(bm, sc.sh[(N + j) * NW + k]);
            }
            part[j * nb + blockIdx.x] = bs;
            part[(N + j) * nb + blockIdx.x] = bm;
        }
        red_release_u32(counter, 1u);
        const unsigned target = round * gridDim.x;
        while (ld_acquire_u32(counter) < target) {}
    }
    __syncthreads();
    double a[N];
    float m[N];
#pragma unroll
    for (int j = 0; j < N; ++j) a[j] = 0.0, m[j] = 0.0f;
    for (int k = tid; k < nb; k += PCG_THREADS)
#pragma unroll
        for (int j = 0; j < N; ++j) {
            a[j] += (double)__ldcg(part + j * nb + k);
            m[j] = fmaxf(m[j], __ldcg(part + (N + j) * nb + k));
        }
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const double aw = warp_sum(a[j]);
        const float mw = warp_max(m[j]);
        if (lane == 0) {
            sc.shd[j * NW + w] = aw;
            sc.sh[j * NW + w] = mw;
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < N; ++j) {
        double t = 0.0;
        float mm = 0.0f;
#pragma unroll
        for (int k = 0; k < NW; ++k) { // every thread adds the warp totals in the same order
            t += sc.shd[j * NW + k];
            mm = fmaxf(mm, sc.sh[j * NW + k]);
        }
        tot[j] = t;
        gmax[j] = mm;
    }
    __syncthreads(); // the scratch is reused by the next reduction
}

} // namespace
} // namespace blub
