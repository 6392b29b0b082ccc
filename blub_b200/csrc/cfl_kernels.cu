// cfl_kernels.cu -- CFL-limited substeps (DESIGN.md §8 "CFL-limited substeps").  Not in the reference, whose clock is a fixed 120 Hz.
//
// max_particle_velocity_kernel measures out[c] = max |v_c| over the live particles, v_c = the .w word of velocity row c.  |v| is the float's
// bits with the sign bit cleared; for non-negative floats (and NaN, whose bits are the largest) the unsigned order of the bits is the order of
// the values, so an unsigned max of the bits is exact and does not depend on the order: warp max (__reduce_max_sync), block max in shared
// memory, one atomicMax per block and axis into three words the launch zeroes.  Zero particles give +0; infinity and NaN come out as themselves.
// Every row is read as whole float4s (the .w words sit in the same 32-byte sectors as the rest of the row): 48 bytes per particle.
//
// cfl_substep_ns is the host rule that turns such a measurement into the length of the next substep, in float64 and integer nanoseconds.
#include <algorithm>
#include <cmath>
#include <cstdio>

#include "blub_core.hpp"

namespace blub {

namespace {

constexpr int PT = 256;

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

__device__ __forceinline__ uint32_t abs_bits(float v) { return __float_as_uint(v) & 0x7FFFFFFFu; }

// n: params->num_particles in device-count mode (params != nullptr), else n_host.  Nothing but the three velocity rows is read.
__global__ void __launch_bounds__(PT) max_particle_velocity_kernel(const StepParams *__restrict__ params, uint32_t n_host, const float4 *__restrict__ rx,
                                                                   const float4 *__restrict__ ry, const float4 *__restrict__ rz, uint32_t *__restrict__ out) {
    __shared__ uint32_t part[3][PT / 32];
    const uint32_t n = params ? params->num_particles : n_host;
    uint32_t m0 = 0u, m1 = 0u, m2 = 0u;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < n; i += gridDim.x * PT) {
        // streaming loads: the rows are read once and need not stay in L2
        const float4 a = __ldcs(rx + i), b = __ldcs(ry + i), c = __ldcs(rz + i);
        m0 = max(m0, abs_bits(a.w));
        m1 = max(m1, abs_bits(b.w));
        m2 = max(m2, abs_bits(c.w));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    m0 = __reduce_max_sync(0xFFFFFFFFu, m0);
    m1 = __reduce_max_sync(0xFFFFFFFFu, m1);
    m2 = __reduce_max_sync(0xFFFFFFFFu, m2);
    if (lane == 0) {
        part[0][warp] = m0;
        part[1][warp] = m1;
        part[2][warp] = m2;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        uint32_t m = 0u;
#pragma unroll
        for (int w = 0; w < PT / 32; ++w) m = max(m, part[threadIdx.x][w]);
        if (m) atomicMax(out + threadIdx.x, m); // the words start at +0
    }
}

} // namespace

void launch_max_particle_velocity(cudaStream_t st, const StepParams *params, uint32_t n_host, uint32_t np_upper, float4 *const row[3], uint32_t *out) {
    BLUB_CUDA_CHECK(cudaMemsetAsync(out, 0, 3 * sizeof(uint32_t), st));
    if (np_upper == 0) return;
    // 8 blocks of 256 threads per SM, each thread with three 16-byte loads in flight per iteration
    BLUB_LAUNCH(max_particle_velocity_kernel, std::min(blocks_for(np_upper, PT), device_sm_count() * 8), PT, 0, st, params, n_host, row[0], row[1], row[2],
                out);
}

void check_time_stepping(const BlubTimeStepping &ts) {
    if (!std::isfinite(ts.cfl_number) || !(ts.cfl_number > 0.0f) || ts.cfl_number > 16.0f)
        throw std::invalid_argument("time stepping: cfl_number must be finite and in (0, 16]");
    if (ts.reserved != 0u) throw std::invalid_argument("time stepping: reserved must be 0");
    if (ts.min_dt_ns < 1u || ts.min_dt_ns > ts.max_dt_ns) throw std::invalid_argument("time stepping: 1 <= min_dt_ns <= max_dt_ns is required");
}

uint64_t capillary_limit_ns(float s) {
    const double d_scaled = std::floor(1e9 * std::sqrt(1.0 / (4.0 * M_PI * (double)s)));
    return d_scaled < 18446744073709551616.0 ? (uint64_t)d_scaled : UINT64_MAX;
}

uint64_t cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTimeStepping &ts) {
    check_time_stepping(ts);
    if (remaining_ns == 0) throw std::invalid_argument("cfl substep: remaining_ns must be above 0");
    for (int c = 0; c < 3; ++c)
        if (!std::isfinite(gravity_grid[c])) throw std::invalid_argument("cfl substep: gravity is not finite");
    char v[96];
    std::snprintf(v, sizeof(v), "(%.9g, %.9g, %.9g) cells/s", max_velocity[0], max_velocity[1], max_velocity[2]);
    for (int c = 0; c < 3; ++c)
        if (!std::isfinite(max_velocity[c])) throw UnstableError(std::string("cfl substep: the largest particle velocity per axis ") + v + " is not finite");
    const double u = std::max({std::fabs((double)max_velocity[0]), std::fabs((double)max_velocity[1]), std::fabs((double)max_velocity[2])});
    const double g = std::sqrt((double)gravity_grid[0] * gravity_grid[0] + (double)gravity_grid[1] * gravity_grid[1] + (double)gravity_grid[2] * gravity_grid[2]);
    const double s = u + std::sqrt(5.0 * g); // Bridson's bound on the speed one step of gravity adds, dx = 1
    const double d = s > 0.0 ? (double)ts.cfl_number / s : INFINITY;
    const double d_scaled = d * 1e9;
    uint64_t d_ns = ts.max_dt_ns;
    if (d_scaled < 18446744073709551616.0) d_ns = std::min(d_ns, (uint64_t)std::floor(d_scaled)); // saturating: 2^64 and above is max_dt_ns
    if (d_ns < ts.min_dt_ns) {
        char m[160];
        std::snprintf(m, sizeof(m), ": the CFL step of %llu ns is below min_dt_ns = %llu ns", (unsigned long long)d_ns, (unsigned long long)ts.min_dt_ns);
        throw UnstableError(std::string("cfl substep: at the largest particle velocity per axis ") + v + m);
    }
    if (remaining_ns <= d_ns) return remaining_ns;
    if (remaining_ns - d_ns < d_ns) return remaining_ns - remaining_ns / 2; // R < 2 d: two halves, so that the interval does not end in a sliver
    return d_ns;
}

} // namespace blub
