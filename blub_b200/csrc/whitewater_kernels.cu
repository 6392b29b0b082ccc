// whitewater_kernels.cu -- spray, foam and bubble particles (sm_90a): the pass at the end of stage 5 (DESIGN.md §8 "Whitewater").
//
// It reads the projected and extrapolated grid velocity, the marker of this step's P2G and the solid volume, and writes nothing but its own
// particles and counters.  Everything runs on the device-resident count (WhitewaterCounters::count) with launches sized by the capacity and
// the grid, so the pass is captured into the step graph:
//   1. whitewater_update_kernel: classify, integrate and test every live particle; the moved particle goes to pos[1] / vel[1] at its own
//      index, its "survives" flag to flags.
//   2. the flow prologue's exclusive scan of the flags, then whitewater_compact_kernel copies the survivors back into pos[0] / vel[0] in
//      their order.
//   3. whitewater_potential_kernel: the particles each FLUID cell of the surface band emits (one draw of the cell's generator for the
//      fraction), 0 elsewhere.  One thread per cell, dense over the grid: a thread whose FLUID bit word is zero writes 0 without reading
//      the marker, the others test their own cell and, for a FLUID cell, its 26 neighbours.
//   4. the exclusive scan of the cell counts, then whitewater_emit_kernel appends the new particles after the survivors in cell order, up
//      to the capacity, and sets the count and the cumulative counters.
// The file is compiled with -fmad=false, and division and square root are IEEE: tests/whitewater_ref.py restates every expression in NumPy
// float32 and agrees bit for bit.  No float atomics, integer scans: every run gives the same bits.
#include <algorithm>

#include "advect.cuh"
#include "xoshiro.hpp"

namespace blub {
namespace {

constexpr uint32_t KIND_SPRAY = BLUB_WHITEWATER_SPRAY, KIND_FOAM = BLUB_WHITEWATER_FOAM, KIND_BUBBLE = BLUB_WHITEWATER_BUBBLE;

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

__device__ __forceinline__ bool fluid_at(const GridDim &g, const int8_t *__restrict__ marker, int x, int y, int z) {
    return x >= 0 && y >= 0 && z >= 0 && x < g.nx && y < g.ny && z < g.nz && marker[lin(g, x, y, z)] == (int8_t)CELL_FLUID;
}

// u(x): advection's MAC trilinear sample
__device__ __forceinline__ void sample_u(const GridDim &g, const float *const U[3], const float x[3], float out[3]) {
    Corners cn;
    float ix[3], iy[3], iz[3];
    mac_corners(g, x, U, cn, ix, iy, iz);
    trilerp3(cn, ix, iy, iz, out);
}

// The kind of a particle at x: a = FLUID cells among the 27 around floor(x) clamped to the grid
__device__ __forceinline__ uint32_t classify(const GridDim &g, const int8_t *__restrict__ marker, const float x[3], const BlubWhitewater &s) {
    const int cx = clampi((int)floorf(x[0]), 0, g.nx - 1), cy = clampi((int)floorf(x[1]), 0, g.ny - 1), cz = clampi((int)floorf(x[2]), 0, g.nz - 1);
    uint32_t a = 0;
    for (int dz = -1; dz <= 1; ++dz)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) a += fluid_at(g, marker, cx + dx, cy + dy, cz + dz) ? 1u : 0u;
    if (a < s.spray_below) return KIND_SPRAY;
    if (marker[lin(g, cx, cy, cz)] == (int8_t)CELL_FLUID && a >= s.bubble_from) return KIND_BUBBLE;
    return KIND_FOAM;
}

__device__ __forceinline__ float ramp(float v, float lo, float hi) { return fminf(fmaxf((v - lo) / (hi - lo), 0.0f), 1.0f); }

__device__ __forceinline__ uint64_t cell_seed(uint32_t step, uint32_t cell) { return (((uint64_t)step << 32) | (uint64_t)cell) ^ WHITEWATER_SEED_KEY; }

__global__ void __launch_bounds__(PT) whitewater_update_kernel(GridDim g, const StepParams *__restrict__ params, const int8_t *__restrict__ marker,
                                                               const float *__restrict__ ux, const float *__restrict__ uy, const float *__restrict__ uz,
                                                               const uint2 *__restrict__ vox, BlubWhitewater s, WhitewaterWork w) {
    const uint32_t n = w.counters->count;
    const float dt = params->dt;
    const float grav[3] = {params->gravity[0], params->gravity[1], params->gravity[2]};
    const float *const U[3] = {ux, uy, uz};
    const int S[3] = {g.nx, g.ny, g.nz};
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i <= w.capacity; i += gridDim.x * PT) {
        uint32_t keep = 0u;
        if (i < n) {
            const float4 p4 = w.pos[0][i], v4 = w.vel[0][i];
            float x[3] = {p4.x, p4.y, p4.z}, v[3] = {v4.x, v4.y, v4.z}, life = p4.w;
            const uint32_t kind = classify(g, marker, x, s);
            if (kind == KIND_SPRAY) {
#pragma unroll
                for (int k = 0; k < 3; ++k) v[k] = v[k] + dt * grav[k];
            } else {
                float u[3];
                sample_u(g, U, x, u);
                if (kind == KIND_BUBBLE) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) v[k] = (v[k] + dt * -(s.buoyancy * grav[k])) + s.drag * (u[k] - v[k]);
                } else {
#pragma unroll
                    for (int k = 0; k < 3; ++k) v[k] = u[k];
                    life = life - dt; // only foam ages
                }
            }
            bool gone = !(life > 0.0f);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                x[k] = x[k] + dt * v[k];
                gone = gone || !(x[k] >= 1.0f && x[k] < (float)S[k] - 1.0f);
            }
            if (!gone) // the cell and the point test advection uses: walls, static solids, moving solids and floating bodies remove whitewater
                gone = marker[lin(g, (int)x[0], (int)x[1], (int)x[2])] == (int8_t)CELL_SOLID || voxel_point_clamp(g, vox, x[0], x[1], x[2]).w > 0.0f;
            keep = gone ? 0u : 1u;
            w.pos[1][i] = make_float4(x[0], x[1], x[2], life);
            w.vel[1][i] = make_float4(v[0], v[1], v[2], __uint_as_float(kind));
        }
        w.flags[i] = keep; // entry capacity stays 0: after the scan it is the number of survivors
    }
}

__global__ void __launch_bounds__(PT) whitewater_compact_kernel(WhitewaterWork w) {
    const uint32_t n = w.counters->count;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < n; i += gridDim.x * PT) {
        const uint32_t at = w.flags[i];
        if (w.flags[i + 1] == at) continue;
        w.pos[0][at] = w.pos[1][i];
        w.vel[0][at] = w.vel[1][i];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { // no thread of this kernel reads survivors
        const uint32_t kept = w.flags[n];
        w.counters->survivors = kept;
        w.counters->removed += n - kept;
    }
}

// The centre velocity of cell (x, y, z): the mean of its two faces per component; the face below cell 0 reads 0
__device__ __forceinline__ void centre_u(const GridDim &g, const float *const U[3], int x, int y, int z, float out[3]) {
    const int c = lin(g, x, y, z);
    out[0] = 0.5f * ((x > 0 ? U[0][c - 1] : 0.0f) + U[0][c]);
    out[1] = 0.5f * ((y > 0 ? U[1][c - g.sy] : 0.0f) + U[1][c]);
    out[2] = 0.5f * ((z > 0 ? U[2][c - g.sz] : 0.0f) + U[2][c]);
}

// The particles FLUID cell (x, y, z) emits: 0 outside the surface band (no draw), else the expected count m rounded by one draw
__device__ uint32_t band_count(const GridDim &g, const StepParams *__restrict__ params, const int8_t *__restrict__ marker, const float *const U[3],
                               const BlubWhitewater &s, int x, int y, int z) {
    if (x == 0 || y == 0 || z == 0 || x == g.nx - 1 || y == g.ny - 1 || z == g.nz - 1) return 0u; // a border cell is never FLUID
    int k = 0, nv[3] = {0, 0, 0};
    for (int dz = -1; dz <= 1; ++dz)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
                if (marker[lin(g, x + dx, y + dy, z + dz)] != (int8_t)CELL_AIR) continue;
                ++k;
                nv[0] += dx;
                nv[1] += dy;
                nv[2] += dz;
            }
    if (k == 0) return 0u;
    float uc[3], xm[3], xp[3], ym[3], yp[3], zm[3], zp[3];
    centre_u(g, U, x, y, z, uc);
    centre_u(g, U, x - 1, y, z, xm);
    centre_u(g, U, x + 1, y, z, xp);
    centre_u(g, U, x, y - 1, z, ym);
    centre_u(g, U, x, y + 1, z, yp);
    centre_u(g, U, x, y, z - 1, zm);
    centre_u(g, U, x, y, z + 1, zp);
    const float wx = (yp[2] - ym[2]) * 0.5f - (zp[1] - zm[1]) * 0.5f;
    const float wy = (zp[0] - zm[0]) * 0.5f - (xp[2] - xm[2]) * 0.5f;
    const float wz = (xp[1] - xm[1]) * 0.5f - (yp[0] - ym[0]) * 0.5f;
    const float curl = sqrtf((wx * wx + wy * wy) + wz * wz);
    const float uu = (uc[0] * uc[0] + uc[1] * uc[1]) + uc[2] * uc[2];
    const float energy = 0.5f * uu;
    const float i_ta = ramp(curl, s.trapped_air_range[0], s.trapped_air_range[1]);
    float i_wc = 0.0f;
    if (nv[0] != 0 || nv[1] != 0 || nv[2] != 0) {
        const float nl = sqrtf((float)(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]));
        const float dot = (uc[0] * (float)nv[0] + uc[1] * (float)nv[1]) + uc[2] * (float)nv[2];
        if (dot >= (0.6f * sqrtf(uu)) * nl) i_wc = ramp((float)k, s.wave_crest_range[0], s.wave_crest_range[1]);
    }
    const float i_k = ramp(energy, s.energy_range[0], s.energy_range[1]);
    const float m = (params->dt * (s.trapped_air_rate * i_ta + s.wave_crest_rate * i_wc)) * i_k;
    Xoshiro256pp rng(cell_seed(params->step_count, lin(g, x, y, z)));
    const float draw = rng.next_f32();
    const float whole = floorf(m);
    const uint32_t base = whole >= (float)s.max_per_cell ? s.max_per_cell : (uint32_t)whole;
    return min(base + (draw < m - whole ? 1u : 0u), s.max_per_cell);
}

__global__ void __launch_bounds__(PT) whitewater_potential_kernel(GridDim g, const StepParams *__restrict__ params, FluidBits bits,
                                                                  const int8_t *__restrict__ marker, const float *__restrict__ ux,
                                                                  const float *__restrict__ uy, const float *__restrict__ uz, BlubWhitewater s,
                                                                  uint32_t *__restrict__ counts) {
    const float *const U[3] = {ux, uy, uz};
    const uint32_t n = (uint32_t)g.n, nx = (uint32_t)g.nx, ny = (uint32_t)g.ny; // fewer than 2^31 cells: 32-bit indices
    for (uint32_t c = blockIdx.x * PT + threadIdx.x; c <= n; c += gridDim.x * PT) {
        uint32_t emit = 0u; // entry n stays 0: after the scan it is the total
        if (c < n) {
            const int x = (int)(c % nx), y = (int)(c / nx % ny), z = (int)(c / nx / ny);
            if (__ldg(bits.words + (z * g.ny + y) * bits.wpr + x / 32) != 0u && marker[c] == (int8_t)CELL_FLUID)
                emit = band_count(g, params, marker, U, s, x, y, z);
        }
        counts[c] = emit;
    }
}

__global__ void __launch_bounds__(PT, 2) whitewater_emit_kernel(GridDim g, const StepParams *__restrict__ params, const int8_t *__restrict__ marker,
                                                             const float *__restrict__ ux, const float *__restrict__ uy, const float *__restrict__ uz,
                                                             BlubWhitewater s, WhitewaterWork w) {
    const uint32_t survivors = w.counters->survivors, total = w.cell_counts[(uint32_t)g.n], room = w.capacity - survivors;
    const uint32_t emitted = total < room ? total : room;
    const float *const U[3] = {ux, uy, uz};
    const uint32_t n = (uint32_t)g.n, nx = (uint32_t)g.nx, ny = (uint32_t)g.ny;
    for (uint32_t c = blockIdx.x * PT + threadIdx.x; c < n; c += gridDim.x * PT) {
        const uint32_t off = w.cell_counts[c], need = w.cell_counts[c + 1] - off;
        if (need == 0u || off >= emitted) continue;
        const int x = (int)(c % nx), y = (int)(c / nx % ny), z = (int)(c / nx / ny);
        Xoshiro256pp rng(cell_seed(params->step_count, c));
        rng.next_f32(); // the fraction's draw
        for (uint32_t j = 0; j < need && off + j < emitted; ++j) {
            float p[3];
            p[0] = (float)x + rng.next_f32();
            p[1] = (float)y + rng.next_f32();
            p[2] = (float)z + rng.next_f32();
            const float life = s.lifetime_lo + rng.next_f32() * (s.lifetime_hi - s.lifetime_lo);
            float v[3];
            sample_u(g, U, p, v);
            const uint32_t kind = classify(g, marker, p, s);
            const uint32_t i = survivors + off + j;
            w.pos[0][i] = make_float4(p[0], p[1], p[2], life);
            w.vel[0][i] = make_float4(v[0], v[1], v[2], __uint_as_float(kind));
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { // no thread of this kernel reads count
        w.counters->count = survivors + emitted;
        w.counters->emitted += emitted;
        w.counters->refused += total - emitted;
    }
}

} // namespace

void launch_whitewater(cudaStream_t st, const GridDim &g, const StepParams *params, const FluidBits &bits, const int8_t *marker, float *const u[3],
                       const uint2 *vox, const BlubWhitewater &s, const WhitewaterWork &w) {
    const int particle_blocks = std::max(std::min(blocks_for((int64_t)w.capacity + 1, PT), device_sm_count() * 16), 1);
    const int cell_blocks = std::max(std::min(blocks_for(g.n + 1, PT), device_sm_count() * 16), 1);
    BLUB_LAUNCH(whitewater_update_kernel, particle_blocks, PT, 0, st, g, params, marker, u[0], u[1], u[2], vox, s, w);
    launch_exclusive_scan(st, w.flags, (int64_t)w.capacity + 1, w.scan_sums);
    BLUB_LAUNCH(whitewater_compact_kernel, particle_blocks, PT, 0, st, w);
    BLUB_LAUNCH(whitewater_potential_kernel, cell_blocks, PT, 0, st, g, params, bits, marker, u[0], u[1], u[2], s, w.cell_counts);
    launch_exclusive_scan(st, w.cell_counts, g.n + 1, w.scan_sums);
    BLUB_LAUNCH(whitewater_emit_kernel, cell_blocks, PT, 0, st, g, params, marker, u[0], u[1], u[2], s, w);
}

} // namespace blub
