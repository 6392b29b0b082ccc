// tag_density_kernels.cu -- liquids of different densities (DESIGN.md §8 "Liquids of different densities").  Not in the reference, whose
// liquid has one density.
//
// A table gives the particles of a tag a density relative to rho_ref (tags not in it: 1).  Stage 0, after P2G, turns the particles into cell
// densities and those into the coefficients of the variable-density velocity solve:
//   - tag_density_scatter_kernel: every live particle adds q = rint(rho_tag 2^20) and 1 to the sum and count of its cell, the cell P2G marks
//     FLUID for it (cell_of_position).  Integer sums: the result does not depend on the particle order.  A warp adds each run of lanes that
//     share a cell once (at most 32 q of at most 2^23 each: the run's sum fits 32 bits).
//   - tag_density_finish_kernel: rho_i = float32(S / (n 2^20)), the quotient formed in float64 and rounded once, on FLUID cells (0 elsewhere);
//     sum and count go back to zero.
//   - tag_density_coeff_kernel: per face, beta = float32(2 / (rho_i + rho_j)) between two FLUID cells, float32(1 / rho_i) between a FLUID
//     cell i and an AIR cell, 0 with a SOLID side (the grid's outside is SOLID) or no FLUID side; per FLUID cell the diagonal
//     D = ((((b-x + b+x) + b-y) + b+y) + b-z) + b+z in float32 and the preconditioner factor float32(1 / D^2) (1 where D = 0).
// With every density 1 the coefficients are 1 on the faces the constant-density solve counts, D its diagonal and 1 / D^2 its table.
#include <algorithm>
#include <cmath>

#include "blub_core.hpp"
#include "grid_words.cuh"

namespace blub {

namespace {

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// What a particle adds for its tag: the table's q, or the default of the tags not in it (relative density 1; the fluid's nu).
__device__ __forceinline__ uint32_t untabled_q(const TagDensityBlock &) { return 1u << TAG_DENSITY_FRAC_BITS; }
__device__ __forceinline__ unsigned long long untabled_q(const TagViscosityBlock &b) { return b.q_default; }
// The sum of a peer group's q: one reduce of at most 32 q of at most 2^23 (densities); q <= 2^32 (viscosities) is added in two 16-bit halves.
__device__ __forceinline__ uint32_t group_sum(unsigned peers, uint32_t q) { return __reduce_add_sync(peers, q); }
__device__ __forceinline__ unsigned long long group_sum(unsigned peers, unsigned long long q) {
    const uint32_t lo = __reduce_add_sync(peers, (uint32_t)(q & 0xffffu)), hi = __reduce_add_sync(peers, (uint32_t)(q >> 16));
    return ((unsigned long long)hi << 16) + lo;
}

// n: params->num_particles in device-count mode (device_count != 0), else n_host
template <class Block>
__global__ void __launch_bounds__(PT) tag_density_scatter_kernel(GridDim g, const StepParams *__restrict__ params, int device_count, uint32_t n_host,
                                                                 const float4 *__restrict__ pos, const Block *__restrict__ table,
                                                                 unsigned long long *__restrict__ sum, uint32_t *__restrict__ count) {
    __shared__ Block sh;
    for (int k = threadIdx.x; k < (int)(sizeof(Block) / 4); k += PT)
        reinterpret_cast<uint32_t *>(&sh)[k] = reinterpret_cast<const uint32_t *>(table)[k];
    __syncthreads();
    const uint32_t n = device_count ? params->num_particles : n_host;
    const int lane = threadIdx.x & 31;
    // whole warps iterate together: every lane of a live warp takes part in the match
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < n; i += gridDim.x * PT) {
        const bool valid = i < n;
        int cell = -1;
        decltype(sh.q[0] + 0) q = untabled_q(sh);
        if (valid) {
            const float4 p = pos[i];
            cell = cell_of_position(g, transfer_position(g, p, 1.0f));
            const uint32_t tag = __float_as_uint(p.w);
            for (uint32_t k = 0; k < sh.count; ++k)
                if (sh.tag[k] == tag) q = sh.q[k];
        }
        const unsigned peers = __match_any_sync(0xffffffffu, cell);
        const auto s = group_sum(peers, valid ? q : 0u);
        if (valid && lane == __ffs(peers) - 1) {
            atomicAdd(sum + cell, (unsigned long long)s);
            atomicAdd(count + cell, (uint32_t)__popc(peers));
        }
    }
}

__global__ void __launch_bounds__(PT) tag_density_finish_kernel(GridDim g, const int8_t *__restrict__ marker, unsigned long long *__restrict__ sum,
                                                                uint32_t *__restrict__ count, float *__restrict__ rho) {
    const int i = blockIdx.x * PT + threadIdx.x;
    if (i >= g.n) return;
    const uint32_t c = count[i];
    float r = 0.0f;
    if (marker[i] == CELL_FLUID) // every FLUID cell holds a particle; 1 keeps a marker written from outside the step well defined
        r = c ? (float)((double)sum[i] / ((double)c * (double)(1u << TAG_DENSITY_FRAC_BITS))) : 1.0f;
    rho[i] = r;
    if (c) {
        sum[i] = 0ull;
        count[i] = 0u;
    }
}

// the face between the cells a (lower) and b (upper)
__device__ __forceinline__ float face_beta(int ma, float ra, int mb, float rb) {
    if (ma == CELL_SOLID || mb == CELL_SOLID) return 0.0f;
    if (ma == CELL_FLUID && mb == CELL_FLUID) return (float)(2.0 / ((double)ra + (double)rb));
    if (ma == CELL_FLUID) return (float)(1.0 / (double)ra);
    if (mb == CELL_FLUID) return (float)(1.0 / (double)rb);
    return 0.0f;
}

__global__ void __launch_bounds__(PT) tag_density_coeff_kernel(GridDim g, const int8_t *__restrict__ marker, const float *__restrict__ rho,
                                                               float *__restrict__ bx, float *__restrict__ by, float *__restrict__ bz,
                                                               float *__restrict__ diag, float *__restrict__ inv_diag2) {
    const int i = blockIdx.x * PT + threadIdx.x;
    if (i >= g.n) return;
    const int x = i % g.nx, y = (i / g.nx) % g.ny, z = i / g.sz;
    const int mc = marker[i];
    const float rc = rho[i];
    const bool lo[3] = {x > 0, y > 0, z > 0}, hi[3] = {x + 1 < g.nx, y + 1 < g.ny, z + 1 < g.nz};
    const int stride[3] = {1, g.sy, g.sz};
    float *const out[3] = {bx, by, bz};
    float d = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int jm = i - stride[c], jp = i + stride[c];
        const float bm = lo[c] ? face_beta(marker[jm], rho[jm], mc, rc) : 0.0f;
        const float bp = hi[c] ? face_beta(mc, rc, marker[jp], rho[jp]) : 0.0f;
        out[c][i] = bp;
        d = __fadd_rn(__fadd_rn(d, bm), bp); // -x, +x, -y, +y, -z, +z
    }
    const bool fluid = mc == CELL_FLUID;
    diag[i] = fluid ? d : 0.0f;
    inv_diag2[i] = fluid && d != 0.0f ? (float)(1.0 / ((double)d * (double)d)) : 1.0f;
}

// nu_i = float32(nu_scale S / (n 2^32)), the quotient formed in float64 and rounded once, on FLUID cells; a FLUID cell without a particle
// (a marker written from outside the step) takes the fluid's nu, every other cell 0.  Sum and count go back to zero.
__global__ void __launch_bounds__(PT) tag_viscosity_finish_kernel(GridDim g, const int8_t *__restrict__ marker, const TagViscosityBlock *__restrict__ b,
                                                                  unsigned long long *__restrict__ sum, uint32_t *__restrict__ count, float *__restrict__ nu) {
    const int i = blockIdx.x * PT + threadIdx.x;
    if (i >= g.n) return;
    const uint32_t c = count[i];
    float v = 0.0f;
    if (marker[i] == CELL_FLUID)
        v = c ? (float)(((double)b->nu_scale * (double)sum[i]) / ((double)c * 4294967296.0)) : b->nu_fluid;
    nu[i] = v;
    if (c) {
        sum[i] = 0ull;
        count[i] = 0u;
    }
}

} // namespace

void launch_tag_viscosity_cells(cudaStream_t st, const GridDim &g, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper,
                                const float4 *pos, const int8_t *marker, const TagViscosityWork &w) {
    if (np_upper > 0)
        BLUB_LAUNCH(tag_density_scatter_kernel<TagViscosityBlock>, std::min(blocks_for(np_upper, PT), device_sm_count() * 8), PT, 0, st, g, params,
                    device_count ? 1 : 0, n_host, pos, w.block, w.sum, w.count);
    BLUB_LAUNCH(tag_viscosity_finish_kernel, blocks_for(g.n, PT), PT, 0, st, g, marker, w.block, w.sum, w.count, w.nu);
}

void launch_tag_density(cudaStream_t st, const GridDim &g, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper,
                        const float4 *pos, const int8_t *marker, const TagDensityWork &w) {
    if (np_upper > 0)
        // 8 blocks of 256 threads per SM, a grid-stride loop over the rest
        BLUB_LAUNCH(tag_density_scatter_kernel<TagDensityBlock>, std::min(blocks_for(np_upper, PT), device_sm_count() * 8), PT, 0, st, g, params, device_count ? 1 : 0,
                    n_host, pos, w.block, w.sum, w.count);
    const int cells = blocks_for(g.n, PT);
    BLUB_LAUNCH(tag_density_finish_kernel, cells, PT, 0, st, g, marker, w.sum, w.count, w.rho);
    BLUB_LAUNCH(tag_density_coeff_kernel, cells, PT, 0, st, g, marker, w.rho, w.beta[0], w.beta[1], w.beta[2], w.diag, w.inv_diag2);
}

void check_tag_densities(const BlubTagDensity *table, uint32_t count) {
    if (count > (uint32_t)TAG_DENSITIES_MAX) throw std::invalid_argument("tag densities: at most 16 entries");
    if (count && !table) throw std::invalid_argument("tag densities: NULL table");
    for (uint32_t k = 0; k < count; ++k) {
        const float r = table[k].relative_density;
        if (!std::isfinite(r) || r < 0.5f || r > 2.0f) throw std::invalid_argument("tag densities: a relative density is not finite or lies outside [1/2, 2]");
        for (uint32_t j = 0; j < k; ++j)
            if (table[j].tag == table[k].tag) throw std::invalid_argument("tag densities: a tag is listed twice");
    }
}

TagDensityBlock make_tag_density_block(const BlubTagDensity *table, uint32_t count) {
    TagDensityBlock b{};
    b.count = count;
    for (uint32_t k = 0; k < count; ++k) {
        b.tag[k] = table[k].tag;
        b.q[k] = (uint32_t)std::nearbyint((double)table[k].relative_density * (double)(1u << TAG_DENSITY_FRAC_BITS)); // exact: a power-of-two scale
    }
    return b;
}

} // namespace blub

namespace blub {

void check_tag_viscosities(const BlubTagViscosity *table, uint32_t count) {
    if (count > (uint32_t)TAG_VISCOSITIES_MAX) throw std::invalid_argument("tag viscosities: at most 16 entries");
    if (count && !table) throw std::invalid_argument("tag viscosities: NULL table");
    for (uint32_t k = 0; k < count; ++k) {
        const float v = table[k].kinematic_viscosity;
        if (!std::isfinite(v) || v < 0.0f) throw std::invalid_argument("tag viscosities: a kinematic viscosity is negative or not finite");
        for (uint32_t j = 0; j < k; ++j)
            if (table[j].tag == table[k].tag) throw std::invalid_argument("tag viscosities: a tag is listed twice");
    }
}

float tag_viscosity_scale(const BlubTagViscosity *table, uint32_t count, float fluid_nu) {
    float s = fluid_nu;
    for (uint32_t k = 0; k < count; ++k) s = std::max(s, table[k].kinematic_viscosity);
    return s;
}

TagViscosityBlock make_tag_viscosity_block(const BlubTagViscosity *table, uint32_t count, float fluid_nu) {
    TagViscosityBlock b{};
    b.count = count;
    b.nu_scale = tag_viscosity_scale(table, count, fluid_nu);
    b.nu_fluid = fluid_nu;
    // rint(nu / nu_scale * 2^32): a value below nu_scale 2^-33 adds 0, nu_scale itself 2^32
    auto q = [&](float nu) { return b.nu_scale > 0.0f ? (unsigned long long)std::nearbyint((double)nu / (double)b.nu_scale * 4294967296.0) : 0ull; };
    for (uint32_t k = 0; k < count; ++k) {
        b.tag[k] = table[k].tag;
        b.q[k] = q(table[k].kinematic_viscosity);
    }
    b.q_default = q(fluid_nu);
    return b;
}

} // namespace blub
