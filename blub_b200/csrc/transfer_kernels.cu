// transfer_kernels.cu -- particle <-> grid transfers of the fluid step (sm_90a): cell lists, P2G, density error, binning.
//
// Reference counterparts (relative to the reference's shader/simulation): transfer_clear.comp, transfer_build_linkedlist.comp,
// transfer_gather_velocity.comp, density_projection_gather_error.comp:41-97, particle_binning_*.comp.
//
// Not a port.  The reference threads per-dual-cell linked lists through the particle buffer (atomic exchange: arbitrary order)
// and gathers them with 729-thread groups in lock-step rounds, capped at 12 / 32 entries ("by far the biggest bottleneck",
// README.md:76).  Here:
//
//   * P2G SCATTER (default; the form z-slab ranks always use): one thread per particle; the lanes of a warp that share a dual cell -- found
//     with match.any, adjacent or not -- add their contributions up in groups of four with two shuffle steps, and the lowest lane of a
//     group forms (sum w*value, sum w) of each face as 64-bit fixed-point integers: 10.7 faces per particle instead of 24 (17.8 with runs
//     of adjacent lanes only).  A block walks chunks of 256 consecutive (cell-sorted) particles and adds the faces inside the chunk's
//     window into a shared-memory tile with 32-bit atomics (low / high words), then flushes each touched tile word with ONE global
//     64-bit reduction; faces outside the window go to the global volume directly.  ~6 global reductions per particle instead of ~21, and
//     sums that do not depend on the arrival order of the atomics or on the split between tile and global path (deterministic).
//     A sparse finish pass normalises and puts the accumulators back to zero (no memsets, no dense pass).  The density scatter is tiled
//     the same way.
//   * CELL LISTS (gather form and binning): a counting sort of particle INDICES by primal cell -- count (one integer atomic per particle),
//     exclusive scan, fill, and a canonicalisation (rank counting) that puts every cell's slice into ascending particle index.  The
//     lists are therefore a pure function of the particle array: the same input gives the same lists, run after run, whatever
//     order the atomics arrived in.
//   * P2G GATHER (deterministic, selectable: BLUB_P2G=gather): one thread per primal cell walks its own list and keeps the
//     (sum w*value, sum w) of the 18 faces a cell's particles can reach in REGISTERS; blocks march along y so that the y-combination of
//     those partial sums happens in registers too, x-neighbours are combined with warp shuffles, z-neighbours through shared memory --
//     all in a fixed order.  No atomics, normalisation / gravity / solid rule fused into the epilogue, bit-identical run to run; slower
//     than the scatter at every phase of a dam break (instruction bound), hence not the default.
//   * the marker volume and a 1-bit-per-cell FLUID mask: from the particles' cells (scatter form) or the cell counts (gather form); a cell
//     is FLUID iff a particle lies in it (transfer_build_linkedlist.comp:17-19) unless it is a border / solid cell
//     (transfer_set_boundary_marker.comp).
#include <cstdlib>
#include <cstring>

#include "advect.cuh"
#include "fluid_kernels.hpp"

namespace blub {
namespace {

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }
// particle kernels: at most 128 blocks per SM (small enough for a negligible tail, few enough to launch quickly), a grid-stride loop over the rest
inline int particle_blocks(uint32_t np_upper) { return min(blocks_for(np_upper, PT), device_sm_count() * 128); }

// ------------------------------------------------------------------------------------------------ cell lists
// count: cell_count[cell] += 1; the returned value is the particle's (arbitrary) slot inside the cell
__device__ __forceinline__ void cell_count_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos, float lo,
                                                        uint32_t *__restrict__ cell_count, uint2 *__restrict__ cell_slot) {
    if (i >= params->num_particles) return;
    const int cell = cell_of_position(g, transfer_position(g, pos[i], lo));
    cell_slot[i] = make_uint2((uint32_t)cell, atomicAdd(cell_count + cell, 1u));
}
__global__ void __launch_bounds__(PT) cell_count_kernel(GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos, float lo,
                                                        uint32_t *__restrict__ cell_count, uint2 *__restrict__ cell_slot) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < np_; i += gridDim.x * PT) cell_count_kernel_one(i, g, params, pos, lo, cell_count, cell_slot);
}

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8; // 2048 cells per block
// phase 1: per-block totals
__global__ void __launch_bounds__(SCAN_THREADS) scan_block_sums_kernel(const uint32_t *__restrict__ in, int64_t n, uint32_t *__restrict__ sums) {
    __shared__ uint32_t sh[SCAN_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_THREADS * SCAN_ITEMS + (int64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t acc = 0;
    if (base + SCAN_ITEMS <= n) {
        const uint4 a = *reinterpret_cast<const uint4 *>(in + base), b = *reinterpret_cast<const uint4 *>(in + base + 4);
        acc = (a.x + a.y) + (a.z + a.w) + (b.x + b.y) + (b.z + b.w);
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k)
            if (base + k < n) acc += in[base + k];
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int k = 0; k < SCAN_THREADS / 32; ++k) t += sh[k];
        sums[blockIdx.x] = t;
    }
}
// phase 2: exclusive scan of the block totals by one block (deterministic block order, unlike the reference's atomic
// arrival order, particle_binning_prefixsum.comp:53-56)
__global__ void __launch_bounds__(1024) scan_sums_kernel(uint32_t *__restrict__ sums, int nblocks) {
    __shared__ uint32_t sh[32];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < nblocks; base += 1024) {
        const int idx = base + threadIdx.x;
        const uint32_t v = idx < nblocks ? sums[idx] : 0u;
        uint32_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) sh[w] = incl;
        __syncthreads();
        if (w == 0) {
            uint32_t s = sh[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += t;
            }
            sh[lane] = s; // inclusive scan of the warp totals
        }
        __syncthreads();
        const uint32_t before = carry + (w > 0 ? sh[w - 1] : 0u);
        if (idx < nblocks) sums[idx] = before + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + incl;
        __syncthreads();
    }
}
// phase 3: exclusive scan inside each block + block base, written in place
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(uint32_t *__restrict__ data, int64_t n, const uint32_t *__restrict__ sums) {
    __shared__ uint32_t sh[SCAN_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_THREADS * SCAN_ITEMS + (int64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], acc = 0;
    const bool full = base + SCAN_ITEMS <= n;
    if (full) {
        const uint4 a = *reinterpret_cast<const uint4 *>(data + base), b = *reinterpret_cast<const uint4 *>(data + base + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) v[k] = base + k < n ? data[base + k] : 0u;
    }
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) acc += v[k];
    uint32_t incl = acc;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) sh[w] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (int k = 0; k < w; ++k) wbase += sh[k];
    uint32_t run = sums[blockIdx.x] + wbase + incl - acc;
    uint32_t o[SCAN_ITEMS];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        o[k] = run;
        run += v[k];
    }
    if (full) {
        *reinterpret_cast<uint4 *>(data + base) = make_uint4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<uint4 *>(data + base + 4) = make_uint4(o[4], o[5], o[6], o[7]);
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k)
            if (base + k < n) data[base + k] = o[k];
    }
}

// fill: arrival[cell_start[cell] + slot] = particle index (the slot is whatever the count atomic returned: arbitrary inside a cell)
__device__ __forceinline__ void cell_fill_kernel_one(uint32_t i, const StepParams *__restrict__ params, const uint2 *__restrict__ cell_slot,
                                                       const uint32_t *__restrict__ cell_start, uint32_t *__restrict__ arrival) {
    if (i >= params->num_particles) return;
    const uint2 cs = cell_slot[i];
    arrival[cell_start[cs.x] + cs.y] = i;
}
__global__ void __launch_bounds__(PT) cell_fill_kernel(const StepParams *__restrict__ params, const uint2 *__restrict__ cell_slot,
                                                       const uint32_t *__restrict__ cell_start, uint32_t *__restrict__ arrival) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < np_; i += gridDim.x * PT) cell_fill_kernel_one(i, params, cell_slot, cell_start, arrival);
}

// canonicalise: ascending particle index inside every cell, by rank counting -- entry j of cell c goes to position
// cell_start[c] + #{entries of c smaller than it}.  One thread per list entry, k loads each from one or two cache lines.
// After this the lists no longer depend on the arrival order of the count atomics.
// CROWDED cells (more than CROWD_T particles: a wave piling up against a wall puts thousands of particles into single cells --
// thousands at step 56 of the 256^3 dam break -- where the reference simply stops reading its lists after 12
// entries) are appended to the crowded-cell list instead and put into the same order by a whole block each (crowded_canonicalize_kernel):
// one thread per entry would walk thousands of entries there.  Their P2G sums are formed by a whole warp in exact integer arithmetic
// (p2g_crowded_kernel).
constexpr uint32_t CROWD_T = 32;
__device__ __forceinline__ void cell_canonicalize_kernel_one(uint32_t j, const StepParams *__restrict__ params, const uint2 *__restrict__ cell_slot,
                                                               const uint32_t *__restrict__ cell_start, const uint32_t *__restrict__ arrival,
                                                               uint32_t *__restrict__ order, CrowdedCells crowd) {
    if (j >= params->num_particles) return;
    const uint32_t v = arrival[j];
    const uint32_t cell = cell_slot[v].x;
    const uint32_t s = cell_start[cell], e = cell_start[cell + 1];
    uint32_t rank = j - s;
    if (e - s <= CROWD_T) {
        rank = 0;
        for (uint32_t t = s; t < e; ++t) rank += arrival[t] < v ? 1u : 0u;
    } else if (j == s) {
        const uint32_t slot = atomicAdd(crowd.count, 1u); // table slots are handed out in arrival order: the table CONTENT does not depend on it
        crowd.cells[slot] = cell;
        crowd.slot_of_cell[cell] = slot;
    }
    order[s + rank] = v;
}
__global__ void __launch_bounds__(PT) cell_canonicalize_kernel(const StepParams *__restrict__ params, const uint2 *__restrict__ cell_slot,
                                                               const uint32_t *__restrict__ cell_start, const uint32_t *__restrict__ arrival,
                                                               uint32_t *__restrict__ order, CrowdedCells crowd) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t j = blockIdx.x * PT + threadIdx.x; (j & ~31u) < np_; j += gridDim.x * PT) cell_canonicalize_kernel_one(j, params, cell_slot, cell_start, arrival, order, crowd);
}

// Ascending particle index inside every crowded cell: one block per cell.  A slice of up to CROWD_SORT_SMEM entries is sorted in shared
// memory by a bitonic network (O(k log^2 k) compare-exchanges spread over the block); a larger one (none seen in the scenes here) falls back
// to rank counting over global memory.  The binning permutes the particles by these lists, so their order must not depend on the
// arrival order of the count atomics either.
constexpr uint32_t CROWD_SORT_SMEM = 8192; // entries (32 KB)
__global__ void __launch_bounds__(PT) crowded_canonicalize_kernel(const uint32_t *__restrict__ cell_start, const uint32_t *__restrict__ arrival,
                                                                  uint32_t *__restrict__ order, CrowdedCells crowd) {
    __shared__ uint32_t sh[CROWD_SORT_SMEM];
    const uint32_t ncrowded = *crowd.count;
    for (uint32_t slot = blockIdx.x; slot < ncrowded; slot += gridDim.x) {
        const uint32_t cell = crowd.cells[slot];
        const uint32_t s = cell_start[cell], k = cell_start[cell + 1] - s;
        const uint32_t *src = arrival + s;
        if (k <= CROWD_SORT_SMEM) { // block-uniform
            uint32_t m = 2;
            while (m < k) m <<= 1;
            for (uint32_t t = threadIdx.x; t < m; t += PT) sh[t] = t < k ? src[t] : 0xffffffffu; // padding sorts last
            __syncthreads();
            for (uint32_t size = 2; size <= m; size <<= 1)
                for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                    for (uint32_t t = threadIdx.x; t < (m >> 1); t += PT) {
                        const uint32_t a = 2 * t - (t & (stride - 1)), b = a + stride;
                        const uint32_t x = sh[a], y = sh[b];
                        if ((x > y) == ((a & size) == 0)) { sh[a] = y; sh[b] = x; }
                    }
                    __syncthreads();
                }
            for (uint32_t t = threadIdx.x; t < k; t += PT) order[s + t] = sh[t];
            __syncthreads(); // the slice in shared memory is read to the end before the next cell overwrites it
        } else {
            for (uint32_t j = threadIdx.x; j < k; j += PT) {
                const uint32_t v = src[j];
                uint32_t rank = 0;
                for (uint32_t t = 0; t < k; ++t) rank += src[t] < v ? 1u : 0u;
                order[s + rank] = v;
            }
        }
    }
}

// Which cells of a 32-cell word the boundary rule makes SOLID: border cells and solid voxels (transfer_set_boundary_marker.comp:11-20)
__device__ __forceinline__ unsigned solid_rule_mask(const GridDim &g, const uint2 *__restrict__ vox, int xw, int y, int z, int cells) {
    const int row = lin(g, 0, y, z), x0 = xw * 32;
    if (y == 0 || y == g.ny - 1 || z <= g.z_wall_lo || z >= g.z_wall_hi) return 0xffffffffu;
    unsigned solid = 0u;
    if (x0 == 0) solid |= 1u;
    if (x0 + cells == g.nx) solid |= 1u << (cells - 1);
    if (vox != nullptr) {
        for (int k = 0; k < cells; ++k)
            if (load_voxel(vox, row + x0 + k).w != 0.0f) solid |= 1u << k;
    }
    return solid;
}

// marker <- f(cell lists): a cell is FLUID iff a particle lies in it (transfer_build_linkedlist.comp:17-19) unless the boundary rule
// makes it SOLID; everything else is AIR (transfer_clear.comp).  One thread per 32-cell word of a row; also writes the FLUID bit mask.
__global__ void __launch_bounds__(PT) marker_from_lists_kernel(GridDim g, FluidBits bits, const uint32_t *__restrict__ cell_start, int8_t *__restrict__ marker,
                                                               const uint2 *__restrict__ vox, uint32_t *__restrict__ particle_words) {
    const int w = blockIdx.x * PT + threadIdx.x;
    if (w >= bits.wpr * g.ny * g.nz) return;
    const int xw = w % bits.wpr, rowi = w / bits.wpr, y = rowi % g.ny, z = rowi / g.ny;
    const int cells = min(32, g.nx - xw * 32);
    const int i0 = lin(g, xw * 32, y, z);
    const uint32_t *cs = cell_start + i0;
    unsigned fluid = 0;
    uint32_t prev = cs[0];
    for (int k4 = 0; k4 < cells; k4 += 4) { // cells is a multiple of 8
        const uint32_t a = cs[k4 + 1], b = cs[k4 + 2], c = cs[k4 + 3], d = cs[k4 + 4];
        fluid |= (a != prev ? 1u : 0u) << k4;
        fluid |= (b != a ? 1u : 0u) << (k4 + 1);
        fluid |= (c != b ? 1u : 0u) << (k4 + 2);
        fluid |= (d != c ? 1u : 0u) << (k4 + 3);
        prev = d;
    }
    const unsigned solid = solid_rule_mask(g, vox, xw, y, z, cells);
    if (particle_words) particle_words[w] = fluid; // cells that hold a particle, whatever the boundary rule makes of them
    fluid &= ~solid;
    for (int k8 = 0; k8 < cells; k8 += 8) { // rows start on multiples of 8 cells: 8-byte stores
        unsigned long long m = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const unsigned bit = 1u << (k8 + k);
            const int v = (solid & bit) ? CELL_SOLID : ((fluid & bit) ? CELL_FLUID : CELL_AIR);
            m |= (unsigned long long)(uint8_t)(int8_t)v << (8 * k);
        }
        *reinterpret_cast<unsigned long long *>(marker + i0 + k8) = m;
    }
    bits.words[w] = fluid;
}

// marker <- boundary rule applied to an existing marker volume (transfer_set_boundary_marker.comp:11-20; every other cell keeps its
// value), + the FLUID bit mask of the result
__global__ void __launch_bounds__(PT) marker_finalize_kernel(GridDim g, FluidBits bits, int8_t *__restrict__ marker, const uint2 *__restrict__ vox,
                                                             uint32_t *__restrict__ particle_words) {
    const int w = blockIdx.x * PT + threadIdx.x;
    if (w >= bits.wpr * g.ny * g.nz) return;
    const int xw = w % bits.wpr, rowi = w / bits.wpr, y = rowi % g.ny, z = rowi / g.ny;
    const int cells = min(32, g.nx - xw * 32);
    int8_t *m = marker + lin(g, xw * 32, y, z);
    const unsigned solid = solid_rule_mask(g, vox, xw, y, z, cells);
    unsigned fluid = 0;
    for (int k8 = 0; k8 < cells; k8 += 8) {
        unsigned long long v = *reinterpret_cast<const unsigned long long *>(m + k8);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if ((int8_t)((v >> (8 * k)) & 0xffull) == (int8_t)CELL_FLUID) fluid |= 1u << (k8 + k);
        const unsigned s8 = (solid >> k8) & 0xffu;
        if (s8) {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (s8 & (1u << k)) v &= ~(0xffull << (8 * k)); // CELL_SOLID == 0
            *reinterpret_cast<unsigned long long *>(m + k8) = v;
        }
    }
    if (particle_words) particle_words[w] = fluid; // cells that were marked FLUID by a particle, whatever the boundary rule makes of them
    bits.words[w] = fluid & ~solid;
}

// FLUID bit mask of a marker volume that is already final (uploaded through the test taps)
__global__ void __launch_bounds__(PT) fluid_bits_kernel(GridDim g, FluidBits bits, const int8_t *__restrict__ marker) {
    const int w = blockIdx.x * PT + threadIdx.x;
    if (w >= bits.wpr * g.ny * g.nz) return;
    const int xw = w % bits.wpr, rowi = w / bits.wpr, y = rowi % g.ny, z = rowi / g.ny;
    const int cells = min(32, g.nx - xw * 32);
    const int8_t *m = marker + lin(g, xw * 32, y, z);
    unsigned fluid = 0;
    for (int k8 = 0; k8 < cells; k8 += 8) {
        const unsigned long long v = *reinterpret_cast<const unsigned long long *>(m + k8);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if ((int8_t)((v >> (8 * k)) & 0xffull) == (int8_t)CELL_FLUID) fluid |= 1u << (k8 + k);
    }
    bits.words[w] = fluid;
}

// ------------------------------------------------------------------------------------------------ P2G, gather form
// Face of cell (i,j,k) for component c samples at q = (i,j,k) + 0.5 + 0.5 e_c; a particle p contributes with
//   weight = prod_d sat(1 - |q_d - p_d|),  value = row_c . (q - p, 1)                  (transfer_gather_velocity.comp:23-31)
// A particle of primal cell C reaches, per dimension d, the faces C_d - 1, C_d (d == c: offset 1.0) or C_d - 1, C_d, C_d + 1
// (d != c: offset 0.5; one of the three always gets weight exactly 0) -- 18 faces, exactly the (face, particle) pairs with
// non-zero weight that the reference's gather visits (:39-97; no 12-entry cap, SURVEY B3).
//
// Work decomposition: block = 32 x-consecutive cells (lanes) x (GW + 2) z rows (warps), marching along y over GLY + 2 cell
// rows.  Thread (lane, warp) owns the cell column (x0 - 1 + lane, *, z0 - 1 + warp).  While it walks the list of its cell in
// row y it accumulates acc[fy][fx][fz] for face rows y - 1, y (, y + 1); after row y, face row y - 1 is complete in y and is
// combined across x (shuffles: lane L's face gets lane L+1's "x - 1" slot and lane L-1's "x + 1" slot) and z (shared memory),
// normalised and stored.  The outermost lanes / warps / rows of a block are halo: computed, never stored.
constexpr int GW = 6;     // z rows stored by a block (warps = GW + 2)
constexpr int GLY = 32;   // face rows stored by a block
constexpr int GXS = 30;   // faces along x stored by a block (lanes 1..30)
constexpr int GCAP = 384; // particles a warp stages per cell row (7 floats each); the rest of a longer row is read from global memory
constexpr int GATHER_THREADS = 32 * (GW + 2);
constexpr int GATHER_STAGE_FLOATS = 7 * GCAP;
constexpr int GATHER_SMEM_BYTES = (GW + 2) * GATHER_STAGE_FLOATS * 4 + 2 * 3 * (GW + 2) * 32 * 8;

template <int AXIS>
__global__ void __launch_bounds__(GATHER_THREADS, 2) p2g_gather_kernel(GridDim g, const StepParams *__restrict__ params, const uint32_t *__restrict__ cell_start,
                                                                       const uint32_t *__restrict__ order, const float4 *__restrict__ pos,
                                                                       const float4 *__restrict__ rowc, const int8_t *__restrict__ marker, float *__restrict__ u,
                                                                       CrowdedCells crowd) {
    constexpr int NFX = AXIS == 0 ? 2 : 3, NFY = AXIS == 1 ? 2 : 3, NFZ = AXIS == 2 ? 2 : 3;
    constexpr float OX = AXIS == 0 ? 1.0f : 0.5f, OY = AXIS == 1 ? 1.0f : 0.5f, OZ = AXIS == 2 ? 1.0f : 0.5f;
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, wz = threadIdx.x >> 5;
    float *stage = smem + wz * GATHER_STAGE_FLOATS;                                      // this warp's staging area: x | y | z | r0..r3, GCAP each
    float2 *q_all = reinterpret_cast<float2 *>(smem + (GW + 2) * GATHER_STAGE_FLOATS); // [2][3][GW + 2][32]
    const int x0 = blockIdx.x * GXS, y0 = blockIdx.y * GLY, z0 = blockIdx.z * GW;
    const int cx = x0 - 1 + lane, cz = z0 - 1 + wz;
    const bool col_valid = cx >= 0 && cx < g.nx && cz >= 0 && cz < g.nz;
    // the lanes of this warp that have a cell: [lane_lo, lane_hi]
    const int lane_lo = x0 == 0 ? 1 : 0, lane_hi = min(31, g.nx - x0);
    const bool warp_valid = cz >= 0 && cz < g.nz && lane_lo <= lane_hi;

    // quick exit: no particle anywhere in the block's cells (lists of a row of x-consecutive cells are one contiguous range)
    {
        int any = 0;
        if (warp_valid) {
            for (int yy = lane; yy < GLY + 2; yy += 32) {
                const int y = y0 - 1 + yy;
                if (y < 0 || y >= g.ny) continue;
                const int c0 = lin(g, x0 - 1 + lane_lo, y, cz);
                any |= cell_start[c0 + (lane_hi - lane_lo + 1)] != cell_start[c0] ? 1 : 0;
            }
        }
        if (!__syncthreads_or(any)) return;
    }

    float2 acc[NFY][NFX][NFZ];
#pragma unroll
    for (int a = 0; a < NFY; ++a)
#pragma unroll
        for (int b = 0; b < NFX; ++b)
#pragma unroll
            for (int c = 0; c < NFZ; ++c) acc[a][b][c] = make_float2(0.f, 0.f);

    const float gdt = params->gravity_dt[AXIS];
    const float fcx = (float)cx, fcz = (float)cz;
    const int y_end = min(y0 + GLY, g.ny); // face rows [y0, y_end) are stored
    for (int y = y0 - 1; y <= y0 + GLY; ++y) {
        if (warp_valid && y >= 0 && y < g.ny) {
            const int ci = lin(g, min(max(cx, 0), g.nx - 1), y, cz);
            uint32_t cs = 0, ce = 0;
            if (col_valid) { cs = cell_start[ci]; ce = cell_start[ci + 1]; }
            const uint32_t S = __shfl_sync(0xffffffffu, cs, lane_lo), E = __shfl_sync(0xffffffffu, ce, lane_hi);
            if (E != S) {
                // stage the row's particles (list order) into shared memory: coalesced index loads, one gather per particle
                const uint32_t staged = min(E - S, (uint32_t)GCAP);
                for (uint32_t j = lane; j < staged; j += 32) {
                    const uint32_t idx = order[S + j];
                    const float3 p = transfer_position(g, pos[idx], 1.0f);
                    const float4 r = rowc[idx];
                    stage[j] = p.x; stage[GCAP + j] = p.y; stage[2 * GCAP + j] = p.z;
                    stage[3 * GCAP + j] = r.x; stage[4 * GCAP + j] = r.y; stage[5 * GCAP + j] = r.z; stage[6 * GCAP + j] = r.w;
                }
                __syncwarp();
                uint32_t cnt = ce - cs;
                if (cnt > CROWD_T) { // crowded cell: its 18 face sums were formed by p2g_crowded_kernel
                    const float2 *tab = crowd.sums + (size_t)crowd.slot_of_cell[ci] * 18;
#pragma unroll
                    for (int fy = 0; fy < NFY; ++fy)
#pragma unroll
                        for (int fx = 0; fx < NFX; ++fx)
#pragma unroll
                            for (int fz = 0; fz < NFZ; ++fz) {
                                const float2 tsum = tab[(fy * NFX + fx) * NFZ + fz];
                                acc[fy][fx][fz].x += tsum.x;
                                acc[fy][fx][fz].y += tsum.y;
                            }
                    cnt = 0;
                }
                const uint32_t kmax = __reduce_max_sync(0xffffffffu, cnt);
                const float fcy = (float)y;
                for (uint32_t k = 0; k < kmax; ++k) {
                    if (k < cnt) {
                        const uint32_t slot = cs - S + k;
                        float px, py, pz, r0, r1, r2, r3;
                        if (slot < (uint32_t)GCAP) {
                            px = stage[slot]; py = stage[GCAP + slot]; pz = stage[2 * GCAP + slot];
                            r0 = stage[3 * GCAP + slot]; r1 = stage[4 * GCAP + slot]; r2 = stage[5 * GCAP + slot]; r3 = stage[6 * GCAP + slot];
                        } else { // a row with more than GCAP particles: the tail comes straight from global memory
                            const uint32_t idx = order[cs + k];
                            const float3 p = transfer_position(g, pos[idx], 1.0f);
                            const float4 r = rowc[idx];
                            px = p.x; py = p.y; pz = p.z; r0 = r.x; r1 = r.y; r2 = r.z; r3 = r.w;
                        }
                        float tx[NFX], ty[NFY], tz[NFZ], wx[NFX], wy[NFY], wzv[NFZ], vz[NFZ];
#pragma unroll
                        for (int f = 0; f < NFX; ++f) { tx[f] = ((fcx + (float)(f - 1)) + OX) - px; wx[f] = saturatef(1.0f - fabsf(tx[f])); }
#pragma unroll
                        for (int f = 0; f < NFY; ++f) { ty[f] = ((fcy + (float)(f - 1)) + OY) - py; wy[f] = saturatef(1.0f - fabsf(ty[f])); }
#pragma unroll
                        for (int f = 0; f < NFZ; ++f) {
                            tz[f] = ((fcz + (float)(f - 1)) + OZ) - pz;
                            wzv[f] = saturatef(1.0f - fabsf(tz[f]));
                            vz[f] = fmaf(r2, tz[f], r3);
                        }
#pragma unroll
                        for (int fy = 0; fy < NFY; ++fy)
#pragma unroll
                            for (int fx = 0; fx < NFX; ++fx) {
                                const float wxy = wx[fx] * wy[fy];
                                const float vxy = fmaf(r1, ty[fy], r0 * tx[fx]);
#pragma unroll
                                for (int fz = 0; fz < NFZ; ++fz) {
                                    const float w = wxy * wzv[fz];
                                    const float v = vxy + vz[fz]; // (r0 tx + r1 ty) + (r2 tz + r3)
                                    acc[fy][fx][fz].x = fmaf(w, v, acc[fy][fx][fz].x);
                                    acc[fy][fx][fz].y += w;
                                }
                            }
                    }
                }
                __syncwarp(); // the staging area is reused by the next row
            }
        }
        // ---- face row y - 1 is complete in y: combine across x and z, normalise, store
        const int yr = y - 1;
        if (yr >= y0 && yr < y_end) { // block-uniform
            float2 *q = q_all + ((yr & 1) * 3) * (GW + 2) * 32;
            // x: face of lane L = [x+1 slot of lane L-1] + [own x slot] + [x-1 slot of lane L+1]   (fixed order)
#pragma unroll
            for (int fz = 0; fz < NFZ; ++fz) {
                float2 s;
                if (AXIS == 0) { // slots: 0 = face cx - 1, 1 = face cx
                    const float2 up = acc[0][0][fz];
                    s.x = acc[0][1][fz].x + __shfl_down_sync(0xffffffffu, up.x, 1);
                    s.y = acc[0][1][fz].y + __shfl_down_sync(0xffffffffu, up.y, 1);
                } else {         // slots: 0 = face cx - 1, 1 = face cx, 2 = face cx + 1
                    const float2 lo = acc[0][NFX - 1][fz], hi = acc[0][0][fz];
                    s.x = (__shfl_up_sync(0xffffffffu, lo.x, 1) + acc[0][1][fz].x) + __shfl_down_sync(0xffffffffu, hi.x, 1);
                    s.y = (__shfl_up_sync(0xffffffffu, lo.y, 1) + acc[0][1][fz].y) + __shfl_down_sync(0xffffffffu, hi.y, 1);
                }
                q[(fz * (GW + 2) + wz) * 32 + lane] = s;
            }
            __syncthreads();
            if (wz >= 1 && wz <= GW && lane >= 1 && lane <= GXS && cx < g.nx && cz < g.nz) {
                // z: face of warp W = [z+1 slot of warp W-1] + [own z slot] + [z-1 slot of warp W+1]   (fixed order)
                float2 s;
                if (AXIS == 2) { // slots: 0 = face cz - 1, 1 = face cz
                    const float2 a = q[(1 * (GW + 2) + wz) * 32 + lane], b = q[(0 * (GW + 2) + wz + 1) * 32 + lane];
                    s = make_float2(a.x + b.x, a.y + b.y);
                } else {
                    const float2 a = q[(2 * (GW + 2) + wz - 1) * 32 + lane], b = q[(1 * (GW + 2) + wz) * 32 + lane], c = q[(0 * (GW + 2) + wz + 1) * 32 + lane];
                    s = make_float2((a.x + b.x) + c.x, (a.y + b.y) + c.y);
                }
                // normalisation + global forces + "don't flow into solid": transfer_gather_velocity.comp:116-127.  Faces that touch
                // no FLUID cell are written 0 (the reference leaves them stale; never observable, SURVEY B6).
                const int i = lin(g, cx, yr, cz);
                const int ma = marker[i], mb = marker[i + (AXIS == 0 ? 1 : (AXIS == 1 ? g.sy : g.sz))];
                float out = 0.0f;
                if ((ma == CELL_FLUID || mb == CELL_FLUID) && ma != CELL_SOLID && mb != CELL_SOLID) {
                    float v = s.x;
                    if (s.y > 0.0f) v /= s.y;
                    out = v + gdt;
                }
                u[i] = out;
            }
        }
        // shift the accumulators: face row y becomes "y - 1" of the next cell row
#pragma unroll
        for (int fx = 0; fx < NFX; ++fx)
#pragma unroll
            for (int fz = 0; fz < NFZ; ++fz) {
#pragma unroll
                for (int fy = 0; fy + 1 < NFY; ++fy) acc[fy][fx][fz] = acc[fy + 1][fx][fz];
                acc[NFY - 1][fx][fz] = make_float2(0.f, 0.f);
            }
    }
}

// The (sum w*value, sum w) of the 18 faces of every CROWDED cell, one warp per cell: the lanes take the cell's particles round robin,
// convert every contribution to 40.24 fixed point and add integers -- exact, hence independent of the order of the particles and of
// the split across lanes -- then the warp total goes back to float.  |w * value| < 2^39 and a cell would need more than 10^9
// particles to overflow; the quantisation (2^-24 per contribution) is below the float rounding of the sums it replaces.
template <int AXIS>
__global__ void __launch_bounds__(PT) p2g_crowded_kernel(GridDim g, const uint32_t *__restrict__ cell_start, const uint32_t *__restrict__ order,
                                                         const float4 *__restrict__ pos, const float4 *__restrict__ rowc, CrowdedCells crowd) {
    constexpr int NFX = AXIS == 0 ? 2 : 3, NFY = AXIS == 1 ? 2 : 3, NFZ = AXIS == 2 ? 2 : 3;
    constexpr float OX = AXIS == 0 ? 1.0f : 0.5f, OY = AXIS == 1 ? 1.0f : 0.5f, OZ = AXIS == 2 ? 1.0f : 0.5f;
    constexpr float FIX = 16777216.0f; // 2^24
    const int lane = threadIdx.x & 31;
    const uint32_t n = *crowd.count;
    for (uint32_t ci = blockIdx.x * (PT / 32) + (threadIdx.x >> 5); ci < n; ci += gridDim.x * (PT / 32)) {
        const uint32_t cell = crowd.cells[ci];
        const uint32_t tq = cell / (uint32_t)g.nx;
        const float fcx = (float)(cell - tq * (uint32_t)g.nx), fcy = (float)(tq % (uint32_t)g.ny), fcz = (float)(tq / (uint32_t)g.ny);
        const uint32_t cs = cell_start[cell], ce = cell_start[cell + 1];
        long long acc[NFY][NFX][NFZ][2];
#pragma unroll
        for (int a = 0; a < NFY; ++a)
#pragma unroll
            for (int b = 0; b < NFX; ++b)
#pragma unroll
                for (int c = 0; c < NFZ; ++c) acc[a][b][c][0] = acc[a][b][c][1] = 0;
        for (uint32_t k = cs + lane; k < ce; k += 32) {
            const uint32_t idx = order[k];
            const float3 p = transfer_position(g, pos[idx], 1.0f);
            const float4 r = rowc[idx];
            float tx[NFX], ty[NFY], tz[NFZ], wx[NFX], wy[NFY], wzv[NFZ], vz[NFZ];
#pragma unroll
            for (int f = 0; f < NFX; ++f) { tx[f] = ((fcx + (float)(f - 1)) + OX) - p.x; wx[f] = saturatef(1.0f - fabsf(tx[f])); }
#pragma unroll
            for (int f = 0; f < NFY; ++f) { ty[f] = ((fcy + (float)(f - 1)) + OY) - p.y; wy[f] = saturatef(1.0f - fabsf(ty[f])); }
#pragma unroll
            for (int f = 0; f < NFZ; ++f) {
                tz[f] = ((fcz + (float)(f - 1)) + OZ) - p.z;
                wzv[f] = saturatef(1.0f - fabsf(tz[f]));
                vz[f] = fmaf(r.z, tz[f], r.w);
            }
#pragma unroll
            for (int fy = 0; fy < NFY; ++fy)
#pragma unroll
                for (int fx = 0; fx < NFX; ++fx) {
                    const float wxy = wx[fx] * wy[fy];
                    const float vxy = fmaf(r.y, ty[fy], r.x * tx[fx]);
#pragma unroll
                    for (int fz = 0; fz < NFZ; ++fz) {
                        const float w = wxy * wzv[fz];
                        const float v = vxy + vz[fz];
                        acc[fy][fx][fz][0] += __float2ll_rn((w * v) * FIX);
                        acc[fy][fx][fz][1] += __float2ll_rn(w * FIX);
                    }
                }
        }
        float2 *out = crowd.sums + (size_t)ci * 18;
#pragma unroll
        for (int fy = 0; fy < NFY; ++fy)
#pragma unroll
            for (int fx = 0; fx < NFX; ++fx)
#pragma unroll
                for (int fz = 0; fz < NFZ; ++fz) {
                    long long a0 = acc[fy][fx][fz][0], a1 = acc[fy][fx][fz][1];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
                        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
                    }
                    if (lane == 0) out[(fy * NFX + fx) * NFZ + fz] = make_float2(__ll2float_rn(a0) * (1.0f / FIX), __ll2float_rn(a1) * (1.0f / FIX));
                }
    }
}

// ------------------------------------------------------------------------------------------------ P2G, scatter form
// One thread per particle.  For component c the particle lies in dual cell d = trunc(pos - off_c), off_c = 0.5 except 1.0 on
// axis c (transfer_build_linkedlist.comp:21-23), and contributes to the eight faces d + {0,1}^3.  (sum w*value, sum w) of a
// face are interleaved as one float2.  Runs of adjacent lanes with the same dual cell (cell-sorted particles hit the SAME eight
// faces) first add their contributions up with shuffles (segmented reduction in groups of four lanes); only the first lane of a group issues
// reductions: two 64-bit fixed-point integer adds per (group, face), fewer than per (particle, face).
// Runs are cut into groups of at most four lanes: two shuffle steps instead of five.  A full log2(32) reduction costs 240 shuffles per
// particle, while runs are short -- a dual cell
// holds 8 particles on average and a cell-sorted warp holds them in 2-4 separate runs; a longer run simply issues one reduction per
// group of four.  Warps in which every lane is its own run (the usual case once the particle order has decayed) skip the shuffles.
// Since r2 session 18 this is the comparison path (BLUB_SCATTER_AGG=adjacent); the default is matched_group_sum below.
template <int NV>
__device__ __forceinline__ bool segmented_run_sum(int key, float (&v)[NV]) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int prev = __shfl_up_sync(full, key, 1);
    const bool start = lane == 0 || prev != key;
    const unsigned starts = __ballot_sync(full, start);
    if (starts == full) return true;                                            // warp-uniform: nothing to add up
    const unsigned upto = starts & (lane == 31 ? full : ((2u << lane) - 1u));   // run starts in the lanes up to this one
    const int pos = lane - (31 - __clz(upto));                                  // position inside the run
    const unsigned above = lane == 31 ? 0u : (starts & ~((2u << lane) - 1u));   // run starts in the lanes above this one
    const int end = above ? __ffs(above) - 1 : 32;                              // first lane that is not part of this lane's run
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        const bool take = (pos & 3) + o < 4 && lane + o < end;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const float t = __shfl_down_sync(full, v[k], o);
            if (take) v[k] += t;
        }
    }
    return (pos & 3) == 0; // the first lane of every group of four issues the reductions
}

// The same reduction over ALL lanes of the warp that share a dual cell, adjacent or not (match.any).  A cell-sorted warp holds the particles
// of about four primal cells; a dual cell of component c collects the particles of one half of a primal cell (c = x) or of the facing halves of
// two x-adjacent primal cells (c = y, z), which sit in the warp but not next to each other: adjacent runs save 17-25 % of the reductions, the
// peer groups 55 % (24 -> 10.7 per particle on the dam break, 8 -> 3.7-4.4 for the density; tools/red_stats.py, oracle positions), and they
// keep doing so while the particle order decays between two re-sorts.  Peer groups are cut into groups of four by rank, the tree is the one
// above: (v0 + v1) + (v2 + v3) in ascending lane order, the group's lowest lane issues the reductions.
template <int NV>
__device__ __forceinline__ bool matched_group_sum(int key, float (&v)[NV]) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(full, key);
    if (__all_sync(full, peers == (1u << lane))) return true;                    // warp-uniform: every lane is alone
    const int rank = __popc(peers & ((1u << lane) - 1u));                        // position among the lanes with this key
    const unsigned above = lane == 31 ? 0u : (peers & ~((2u << lane) - 1u));
    const int n1 = above ? __ffs(above) - 1 : -1;                                // the peer of rank + 1, if any
    const int n2 = __shfl_sync(full, n1, n1 >= 0 ? n1 : lane);                   // the peer of rank + 2 (a lane without a next peer reads its own -1)
    const bool take1 = (rank & 1) == 0 && n1 >= 0, take2 = (rank & 3) == 0 && n2 >= 0;
    const int s1 = n1 >= 0 ? n1 : lane, s2 = n2 >= 0 ? n2 : lane;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const float t = __shfl_sync(full, v[k], s1);
        if (take1) v[k] += t;
    }
    if (__any_sync(full, take2)) { // warp-uniform: no group of this warp has a third member (the usual case for the x component)
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const float t = __shfl_sync(full, v[k], s2);
            if (take2) v[k] += t;
        }
    }
    return (rank & 3) == 0; // the lowest lane of every group of four issues the reductions
}
template <bool MATCH, int NV>
__device__ __forceinline__ bool warp_group_sum(int key, float (&v)[NV]) {
    return MATCH ? matched_group_sum<NV>(key, v) : segmented_run_sum<NV>(key, v);
}

// ---- block-private accumulator tiles of the scatters
// A block walks chunks of PT consecutive particles (warp k of a chunk still owns particles 32k .. 32k + 31, so the warp peer groups and
// the integers formed per group and face are those of a plain one-thread-per-particle launch).  Particles are re-sorted into x-fastest
// primal-cell order every few steps, so a chunk covers a short run of x-adjacent cells in one or two rows and its faces fall into a small
// box: the group heads add the faces that lie inside the chunk's box (its WINDOW) into a shared-memory tile, and after the chunk every
// non-zero tile word goes out as ONE global 64-bit reduction -- 5.7 global reductions per particle instead of 19-21 on a sorted dam
// break, 8.8 instead of 25 after the order has decayed (tools/red_stats.py).  Faces outside the window (a far-off particle, a decayed or
// unsorted order) take the global path directly, decided per face: slower, never wrong.
//
// The tile words are 32-bit: a 64-bit shared atomicAdd compiles to a CAS loop on sm_90a, a 32-bit one to a native ATOMS.ADD.  A 64-bit
// sum is kept as a low word and a high word; the add that wraps the low word carries into the high one, so (hi << 32) | lo is the sum
// modulo 2^64 whatever the order of arrival -- and the global sums, integer adds modulo 2^64 too, come out bit for bit as without tile.
struct TileWindow {
    int ox, oy, oz; // face (x, y, z) of tile entry 0
    int ex, ey, ez; // extent; ex * ey * ez <= the tile's capacity (ex may be 0: no tile)
};
// tile_add_lo adds the low word of q and returns what the high word still needs: the high half of q plus the carry out of the low word.
// The scatters' fast paths issue the low-word adds of several faces back to back and only then the high-word adds, so that the round
// trips overlap; they add zeros rather than branch around them (q == 0 leaves both words as they are).
__device__ __forceinline__ uint32_t tile_add_lo(uint32_t *lo, long long q) {
    const uint32_t ql = (uint32_t)q;
    const uint32_t old = atomicAdd(lo, ql);
    return (uint32_t)((unsigned long long)q >> 32) + (old + ql < old ? 1u : 0u);
}
__device__ __forceinline__ void tile_add(uint32_t *lo, uint32_t *hi, long long q) {
    const uint32_t h = tile_add_lo(lo, q);
    if (h != 0u) atomicAdd(hi, h);
}
__device__ __forceinline__ long long tile_word(const uint32_t *lo, const uint32_t *hi) {
    return (long long)(((unsigned long long)*hi << 32) | *lo);
}
// Zeroes the first `size` entries of PLANES word planes of CAP entries with 128-bit stores (the tile is 16-byte aligned and CAP % 4 == 0,
// so the range rounded up to 4 entries stays inside each plane; no face adds to the entries past `size`).  The flushes keep 32-bit loads:
// lane = entry keeps a warp's global reductions on adjacent cells.
template <int PLANES, int CAP>
__device__ __forceinline__ void tile_zero(uint32_t *tile, int size) {
    static_assert(CAP % 4 == 0, "128-bit tile stores");
    for (int t = 4 * threadIdx.x; t < size; t += 4 * PT)
#pragma unroll
        for (int k = 0; k < PLANES; ++k) *reinterpret_cast<uint4 *>(tile + k * CAP + t) = make_uint4(0u, 0u, 0u, 0u);
}
// The window of the chunk starting at particle b, from the primal cells of its particles (every thread of the block calls this, `cell`
// of its own particle, `valid` whether it has one).  It covers the faces [min - 1, max + 1] of those cells in every dimension, which
// holds every face they reach; a box of more than CAP faces is cut -- z first, then y (neither below 3 faces), then x -- around the
// cell of the chunk's middle particle, so that one far-off particle does not push the others out.  Ends with __syncthreads().
template <int CAP>
__device__ __forceinline__ TileWindow scatter_window(uint32_t b, uint32_t np, bool valid, int3 cell, int (*scratch)[8], TileWindow *shared_win) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int big = 0x3fffffff;
    const int mnx = __reduce_min_sync(0xffffffffu, valid ? cell.x : big), mxx = __reduce_max_sync(0xffffffffu, valid ? cell.x : -big);
    const int mny = __reduce_min_sync(0xffffffffu, valid ? cell.y : big), mxy = __reduce_max_sync(0xffffffffu, valid ? cell.y : -big);
    const int mnz = __reduce_min_sync(0xffffffffu, valid ? cell.z : big), mxz = __reduce_max_sync(0xffffffffu, valid ? cell.z : -big);
    if (lane == 0) {
        scratch[warp][0] = mnx; scratch[warp][1] = mny; scratch[warp][2] = mnz;
        scratch[warp][3] = mxx; scratch[warp][4] = mxy; scratch[warp][5] = mxz;
    }
    const uint32_t n = min(np - b, (uint32_t)PT); // b < np
    if (threadIdx.x == n / 2) { scratch[PT / 32][0] = cell.x; scratch[PT / 32][1] = cell.y; scratch[PT / 32][2] = cell.z; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int lo[3], hi[3], e[3];
        for (int d = 0; d < 3; ++d) {
            lo[d] = big; hi[d] = -big;
            for (int w = 0; w < PT / 32; ++w) { lo[d] = min(lo[d], scratch[w][d]); hi[d] = max(hi[d], scratch[w][3 + d]); }
            lo[d] -= 1; hi[d] += 1;
            e[d] = hi[d] - lo[d] + 1;
        }
        e[2] = min(e[2], max(3, CAP / (e[0] * e[1])));
        e[1] = min(e[1], max(3, CAP / (e[0] * e[2])));
        e[0] = min(e[0], CAP / (e[1] * e[2]));
        int o[3];
        for (int d = 0; d < 3; ++d) o[d] = min(max(scratch[PT / 32][d] - e[d] / 2, lo[d]), hi[d] - e[d] + 1);
        *shared_win = TileWindow{o[0], o[1], o[2], e[0], e[1], e[2]};
    }
    __syncthreads();
    return *shared_win;
}
// tile entry of face (x, y, z), or -1 outside the window
__device__ __forceinline__ int tile_entry(const TileWindow &w, int x, int y, int z) {
    const int rx = x - w.ox, ry = y - w.oy, rz = z - w.oz;
    return ((unsigned)rx < (unsigned)w.ex && (unsigned)ry < (unsigned)w.ey && (unsigned)rz < (unsigned)w.ez) ? (rz * w.ey + ry) * w.ex + rx : -1;
}
// tile entry of face (x, y, z) if the whole box of faces x..x+1, y..y+1, z..z+1 lies inside the window (its eight entries are then this one
// plus 0, 1, ex, ex + 1, ex * ey, ...), or -1
__device__ __forceinline__ int tile_box_entry(const TileWindow &w, int x, int y, int z) {
    const int rx = x - w.ox, ry = y - w.oy, rz = z - w.oz;
    return (rx >= 0 && ry >= 0 && rz >= 0 && rx + 1 < w.ex && ry + 1 < w.ey && rz + 1 < w.ez) ? (rz * w.ey + ry) * w.ex + rx : -1;
}
// global cell index of tile entry t
__device__ __forceinline__ int tile_cell(const GridDim &g, const TileWindow &w, int t) {
    const int q = t / w.ex;
    return lin(g, w.ox + (t - q * w.ex), w.oy + q % w.ey, w.oz + q / w.ey);
}

// P2G tile: per face 3 components x {sum w * value, sum w} x {low, high} words, word planes of P2G_TILE entries
constexpr int P2G_TILE = 1184;
constexpr int P2G_TILE_BYTES = 12 * P2G_TILE * 4; // 56,832 B: with the 1 KB the hardware reserves per block, 4 blocks fit into 228 KB
constexpr int DENSITY_TILE = 2048;                // density tile: {low, high} word planes (16 KB)
constexpr int P2G_CARRY_BATCH = 4;                // P2G faces whose low-word adds (value and weight) are issued before their carries

// ---- brick schedule of the density and P2G scatters (built at every re-sort, DESIGN.md §3.2)
// After a re-sort the particles are in x-fastest cell order, so a chunk of 256 consecutive particles covers one short run of a cell row and
// every cell row is flushed once by each of the chunks of the 3 x 3 cell rows around it.  The schedule groups the aligned warps (particles
// 32w .. 32w + 31) by the BRICK of SCHED_BX x SCHED_BY x SCHED_BZ cells that holds the cell of their first particle, and cuts each brick's
// warps (ascending) into work items of at most SCHED_K warps.  A block runs a work item's warps through one tile -- its window set from
// where the item's particles are at the time of the scatter (item_window) -- and flushes it once.  A
// warp still holds the particles it holds in a plain launch, so every peer group and every integer it forms is the same, and the sums come
// out bit for bit the same whatever warps share a tile: the schedule only decides how much goes the tile way.  Coverage is all that
// correctness rests on: the items hold warps [0, brick_warps[nbricks]) once each, the 256-particle chunks take the rest.
constexpr int SCHED_BX = 28, SCHED_BY = 4, SCHED_BZ = 4; // cells per brick
constexpr int P2G_MIN_ITEM_WAVES = 8;                     // P2G walks the work items only when they fill this many waves of 4 blocks per SM
constexpr uint32_t SCHED_K = 64;                         // warps per work item at most: a long tail and too few items for a small fluid cost more
// the cells of a brick (+-1) and room for warps that start near its high x edge and reach over it
static_assert((SCHED_BX + 4) * (SCHED_BY + 2) * (SCHED_BZ + 2) <= DENSITY_TILE, "a brick's window fits the density tile");

__device__ __forceinline__ uint32_t warps_before(uint32_t particle) { return (particle >> 5) + ((particle & 31u) != 0u ? 1u : 0u); }
__device__ __forceinline__ int3 brick_origin(const GridDim &g, int b) {
    const int nbx = (g.nx + SCHED_BX - 1) / SCHED_BX, nby = (g.ny + SCHED_BY - 1) / SCHED_BY;
    return make_int3(b % nbx * SCHED_BX, b / nbx % nby * SCHED_BY, b / nbx / nby * SCHED_BZ);
}
// The warps whose first particle lies in the x-run [x0, x0 + SCHED_BX) of row (y, z): [warps_before(start of the run), warps_before(its end)).
// Over all runs of all bricks these ranges cover [0, warps_before(np)) once each.
__device__ __forceinline__ uint2 run_warps(const GridDim &g, const uint32_t *__restrict__ cell_start, int x0, int y, int z) {
    const int c0 = lin(g, x0, y, z);
    return make_uint2(warps_before(cell_start[c0]), warps_before(cell_start[c0 + min(SCHED_BX, g.nx - x0)]));
}
// one thread per brick: its warp and work item counts (the entries at nbricks, the totals after the scans, are set to 0 here)
__global__ void __launch_bounds__(PT) schedule_count_kernel(GridDim g, const uint32_t *__restrict__ cell_start, ScatterSchedule s) {
    const int b = blockIdx.x * PT + threadIdx.x;
    if (b == 0) s.brick_warps[s.nbricks] = s.brick_items[s.nbricks] = 0u;
    if (b >= s.nbricks) return;
    const int3 o = brick_origin(g, b);
    uint32_t warps = 0;
    for (int z = o.z; z < min(o.z + SCHED_BZ, g.nz); ++z)
        for (int y = o.y; y < min(o.y + SCHED_BY, g.ny); ++y) {
            const uint2 r = run_warps(g, cell_start, o.x, y, z);
            warps += r.y - r.x;
        }
    s.brick_warps[b] = warps;
    s.brick_items[b] = (warps + SCHED_K - 1) / SCHED_K;
}
// one warp per brick (after the scans): its warps in ascending order, and the first warp and the brick of each of its work items
__global__ void __launch_bounds__(PT) schedule_fill_kernel(GridDim g, const uint32_t *__restrict__ cell_start, ScatterSchedule s) {
    const int b = (blockIdx.x * PT + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= s.nbricks) return; // warp-uniform
    const int3 o = brick_origin(g, b);
    const uint32_t first = s.brick_warps[b], item0 = s.brick_items[b], nitems = s.brick_items[b + 1] - item0;
    for (uint32_t k = lane; k < nitems; k += 32) {
        s.item_start[item0 + k] = first + k * SCHED_K;
        s.item_brick[item0 + k] = (uint32_t)b;
        s.item_box[2 * (item0 + k)] = make_int4(1, 1, 1, 0); // empty until the density scatter has seen the item
        s.item_box[2 * (item0 + k) + 1] = make_int4(0, 0, 0, 0);
    }
    uint32_t out = first;
    for (int z = o.z; z < min(o.z + SCHED_BZ, g.nz); ++z)
        for (int y = o.y; y < min(o.y + SCHED_BY, g.ny); ++y) {
            const uint2 r = run_warps(g, cell_start, o.x, y, z);
            for (uint32_t w = r.x + lane; w < r.y; w += 32) s.warps[out + (w - r.x)] = w;
            out += r.y - r.x;
        }
}
// The work items of the schedule (none while it is invalid or absent); `tail` = the first particle it does not cover
__device__ __forceinline__ uint32_t schedule_items(const ScatterSchedule &s, uint32_t &tail) {
    tail = 0u;
    if (s.valid == nullptr || *s.valid == 0u) return 0u;
    tail = 32u * s.brick_warps[s.nbricks];
    return s.brick_items[s.nbricks];
}
// The tile window of work item `it` from the box of its particles' primal cells, [lo, hi] (lo > hi: none of them is left, no tile): the
// faces [lo - 1, hi + 1] in every dimension; a box of more than CAP entries is cut -- z first, then y (neither below the brick's rows + 2),
// then x -- around the middle of the item's brick.
template <int CAP>
__device__ __forceinline__ TileWindow box_window(const GridDim &g, const ScatterSchedule &s, uint32_t it, int4 lo_cell, int4 hi_cell) {
    if (lo_cell.x > hi_cell.x || lo_cell.y > hi_cell.y || lo_cell.z > hi_cell.z) return TileWindow{0, 0, 0, 0, 0, 0};
    const int lo[3] = {lo_cell.x - 1, lo_cell.y - 1, lo_cell.z - 1}, hi[3] = {hi_cell.x + 1, hi_cell.y + 1, hi_cell.z + 1};
    int e[3] = {hi[0] - lo[0] + 1, hi[1] - lo[1] + 1, hi[2] - lo[2] + 1};
    e[2] = min(e[2], max(SCHED_BZ + 2, CAP / (e[0] * e[1])));
    e[1] = min(e[1], max(SCHED_BY + 2, CAP / (e[0] * e[2])));
    e[0] = min(e[0], CAP / (e[1] * e[2]));
    const int3 b = brick_origin(g, (int)s.item_brick[it]);
    const int mid[3] = {b.x + SCHED_BX / 2, b.y + SCHED_BY / 2, b.z + SCHED_BZ / 2};
    int o[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) o[d] = min(max(mid[d] - e[d] / 2, lo[d]), hi[d] - e[d] + 1);
    return TileWindow{o[0], o[1], o[2], e[0], e[1], e[2]};
}
// The box of primal cells a work item's particles are in, one thread's share: `p` a position as the scatter sees it (transfer_position)
constexpr int BOX_EMPTY = 0x3fffffff;
__device__ __forceinline__ void extend_box(const GridDim &g, const float3 &p, int mn[3], int mx[3]) {
    const int c[3] = {min((int)p.x, g.nx - 1), min((int)p.y, g.ny - 1), min((int)p.z, g.nz - 1)};
#pragma unroll
    for (int d = 0; d < 3; ++d) { mn[d] = min(mn[d], c[d]); mx[d] = max(mx[d], c[d]); }
}
// The tile window of work item `it` from the threads' shares of its cell box (extend_box), which is also kept in s.item_box.  Every thread
// of the block calls this; it ends with __syncthreads().
template <int CAP>
__device__ __forceinline__ TileWindow item_box_window(const GridDim &g, const ScatterSchedule &s, uint32_t it, int mn[3], int mx[3], int (*scratch)[8],
                                                      TileWindow *shared_win) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        mn[d] = __reduce_min_sync(0xffffffffu, mn[d]);
        mx[d] = __reduce_max_sync(0xffffffffu, mx[d]);
    }
    if (lane == 0)
#pragma unroll
        for (int d = 0; d < 3; ++d) { scratch[warp][d] = mn[d]; scratch[warp][3 + d] = mx[d]; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int lo[3], hi[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            lo[d] = BOX_EMPTY; hi[d] = -BOX_EMPTY;
            for (int w = 0; w < PT / 32; ++w) { lo[d] = min(lo[d], scratch[w][d]); hi[d] = max(hi[d], scratch[w][3 + d]); }
        }
        const int4 l = make_int4(lo[0], lo[1], lo[2], 0), h = make_int4(hi[0], hi[1], hi[2], 0);
        s.item_box[2 * it] = l;
        s.item_box[2 * it + 1] = h;
        *shared_win = box_window<CAP>(g, s, it, l, h);
    }
    __syncthreads();
    return *shared_win;
}
// The window of work item `it` (its warps are s.warps[w0 .. w1)) for the density scatter, from the primal cells its particles are in NOW:
// particles drift away from the brick they were sorted into, and a window fixed at the re-sort loses them within a few steps.  The box of
// those cells is also kept in s.item_box: the next step's P2G scatter takes its window from it (the density correction in between moves
// particles by a fraction of a cell; a face that leaves the window takes the global path).  Every thread of the block calls this; it ends
// with __syncthreads().
template <int CAP>
__device__ __forceinline__ TileWindow item_window(const GridDim &g, const ScatterSchedule &s, uint32_t it, uint32_t w0, uint32_t w1, uint32_t np,
                                                  const float4 *__restrict__ pos, float clamp_lo, int (*scratch)[8], TileWindow *shared_win) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int mn[3] = {BOX_EMPTY, BOX_EMPTY, BOX_EMPTY}, mx[3] = {-BOX_EMPTY, -BOX_EMPTY, -BOX_EMPTY};
    for (uint32_t k = w0 + warp; k < w1; k += PT / 32) { // warp-uniform
        const uint32_t i = 32u * s.warps[k] + lane;
        if (i < np) extend_box(g, transfer_position(g, pos[i], clamp_lo), mn, mx);
    }
    return item_box_window<CAP>(g, s, it, mn, mx, scratch, shared_win);
}

template <bool MARK, bool MATCH>
__device__ __forceinline__ void p2g_scatter_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params, const float3 p,
                                                         const float4 *__restrict__ rowx, const float4 *__restrict__ rowy,
                                                         const float4 *__restrict__ rowz, longlong2 *__restrict__ nwx, longlong2 *__restrict__ nwy,
                                                         longlong2 *__restrict__ nwz, int8_t *__restrict__ marker, const TileWindow &win,
                                                         uint32_t *__restrict__ tile) {
    const uint32_t np = params->num_particles;
    if ((i & ~31u) >= np) return;  // whole warp beyond the last particle (z-slab ranks launch over their capacity)
    const bool valid = i < np;     // no per-lane early return: every lane of a live warp takes part in the shuffles
    if (MARK && valid) marker[cell_of_position(g, p)] = (int8_t)CELL_FLUID; // transfer_build_linkedlist.comp:17-19
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    // one copy of the component body, not three: unrolled (and inlined twice, by the item and the chunk path) the loop makes the kernel
    // about 8,000 instructions, and the scatter runs measurably slower out of the instruction caches
#pragma unroll 1
    for (int c = 0; c < 3; ++c) {
        const float4 *const row = c == 0 ? rowx : c == 1 ? rowy : rowz;
        longlong2 *const nwc = c == 0 ? nwx : c == 1 ? nwy : nwz;
        const float ox = c == 0 ? 1.0f : 0.5f, oy = c == 1 ? 1.0f : 0.5f, oz = c == 2 ? 1.0f : 0.5f;
        const int dx = (int)(p.x - ox), dy = (int)(p.y - oy), dz = (int)(p.z - oz);
        const float qx = (float)dx + ox, qy = (float)dy + oy, qz = (float)dz + oz; // sample point of face (dx,dy,dz)
        const float4 r = valid ? row[i] : zero;
        const float tx[2] = {qx - p.x, qx + 1.0f - p.x}, ty[2] = {qy - p.y, qy + 1.0f - p.y}, tz[2] = {qz - p.z, qz + 1.0f - p.z};
        const float wxs[2] = {saturatef(1.0f - fabsf(tx[0])), saturatef(1.0f - fabsf(tx[1]))};
        const float wys[2] = {saturatef(1.0f - fabsf(ty[0])), saturatef(1.0f - fabsf(ty[1]))};
        const float wzs[2] = {saturatef(1.0f - fabsf(tz[0])), saturatef(1.0f - fabsf(tz[1]))};
        const int base = lin(g, dx, dy, dz);
        float acc[16]; // (sum w * value, sum w) of the eight faces
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ox_ = k & 1, oy_ = (k >> 1) & 1, oz_ = k >> 2;
            const float w = valid ? wxs[ox_] * wys[oy_] * wzs[oz_] : 0.0f;
            const float v = r.x * tx[ox_] + r.y * ty[oy_] + r.z * tz[oz_] + r.w;
            acc[2 * k] = w > 0.0f ? w * v : 0.0f;
            acc[2 * k + 1] = w > 0.0f ? w : 0.0f;
        }
        const bool live = warp_group_sum<MATCH, 16>(valid ? base : -1 - (int)(threadIdx.x & 31), acc) && valid; // a head issues the adds
        const int e0 = tile_box_entry(win, dx, dy, dz);
        if (__all_sync(0xffffffffu, e0 >= 0 || !live)) { // warp-uniform: every head's eight faces go to the tile
            // the same sums as below without a branch per face, P2G_CARRY_BATCH faces at a time: their low-word adds (value and weight)
            // first, then the high words they carry into.  A weight that rounds to 0 leaves its value out, as below: both add 0.
            if (live) {
                uint32_t *const t = tile + 4 * c * P2G_TILE + e0; // planes: value low, value high, weight low, weight high
                const int sy = win.ex, sz = win.ex * win.ey;
#pragma unroll
                for (int k0 = 0; k0 < 8; k0 += P2G_CARRY_BATCH) {
                    uint32_t hv[P2G_CARRY_BATCH], hw[P2G_CARRY_BATCH];
#pragma unroll
                    for (int j = 0; j < P2G_CARRY_BATCH; ++j) {
                        const int k = k0 + j, o = (k & 1) + ((k >> 1) & 1) * sy + (k >> 2) * sz;
                        const long long wq = to_fixed<FIXED_WEIGHT_BITS>(acc[2 * k + 1]);
                        const long long num = wq > 0 ? to_fixed<FIXED_VALUE_BITS>(acc[2 * k]) : 0;
                        hv[j] = tile_add_lo(t + o, num);
                        hw[j] = tile_add_lo(t + 2 * P2G_TILE + o, wq > 0 ? wq : 0);
                    }
#pragma unroll
                    for (int j = 0; j < P2G_CARRY_BATCH; ++j) {
                        const int k = k0 + j, o = (k & 1) + ((k >> 1) & 1) * sy + (k >> 2) * sz;
                        atomicAdd(t + P2G_TILE + o, hv[j]);
                        atomicAdd(t + 3 * P2G_TILE + o, hw[j]);
                    }
                }
            }
        } else if (live) {
            uint32_t *const t = tile + 4 * c * P2G_TILE;
#pragma unroll
            for (int k = 0; k < 8; ++k)
            {
                // a contribution whose weight rounds to 0 is left out entirely (value too), so a face with weight 0 also has value 0
                const long long wq = to_fixed<FIXED_WEIGHT_BITS>(acc[2 * k + 1]);
                if (wq > 0) {
                    const long long num = to_fixed<FIXED_VALUE_BITS>(acc[2 * k]);
                    const int e = tile_entry(win, dx + (k & 1), dy + ((k >> 1) & 1), dz + (k >> 2));
                    if (e >= 0) {
                        if (num != 0) tile_add(t + e, t + P2G_TILE + e, num);
                        tile_add(t + 2 * P2G_TILE + e, t + 3 * P2G_TILE + e, wq);
                    } else {
                        longlong2 *const f = nwc + base + (k & 1) + ((k >> 1) & 1) * g.sy + (k >> 2) * g.sz;
                        if (num != 0) fixed_add(&f->x, num);
                        fixed_add(&f->y, wq);
                    }
                }
            }
        }
    }
}
// 4 resident blocks per SM (64 registers, no spills for sm_90a; P2G_TILE_BYTES of dynamic shared memory); a 5 / 6-block bound
// (48 / 40 registers) spills
template <bool MARK, bool MATCH>
__global__ void __launch_bounds__(PT, 4) p2g_scatter_kernel(GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos,
                                                         const float4 *__restrict__ rowx, const float4 *__restrict__ rowy,
                                                         const float4 *__restrict__ rowz, longlong2 *__restrict__ nwx, longlong2 *__restrict__ nwy,
                                                         longlong2 *__restrict__ nwz, int8_t *__restrict__ marker, ScatterSchedule sched,
                                                         uint32_t min_items) {
    extern __shared__ __align__(16) uint32_t tile[]; // [12][P2G_TILE]
    __shared__ int scratch[PT / 32 + 1][8];
    __shared__ TileWindow shared_win;
    longlong2 *const nw[3] = {nwx, nwy, nwz};
    const uint32_t np_ = params->num_particles;
    // the work items of the brick schedule, their windows from the cell boxes the last density scatter left (item_window): one zeroing and
    // one flush per item, its warps 8 at a time.  Fewer than min_items items (a small fluid) would leave SMs idle at 4 blocks per SM while
    // each block walks up to 8 rounds of warps: the chunks then take every particle.
    uint32_t tail;
    uint32_t items = schedule_items(sched, tail);
    if (items < min_items) items = tail = 0u;
    for (uint32_t it = blockIdx.x; it < items; it += gridDim.x) { // block-uniform
        if (threadIdx.x == 0) shared_win = box_window<P2G_TILE>(g, sched, it, sched.item_box[2 * it], sched.item_box[2 * it + 1]);
        __syncthreads();
        const TileWindow win = shared_win;
        const int size = win.ex * win.ey * win.ez;
        tile_zero<12, P2G_TILE>(tile, size);
        __syncthreads();
        const uint32_t w0 = sched.item_start[it], w1 = it + 1 < items ? sched.item_start[it + 1] : tail / 32u;
        for (uint32_t k = w0 + (threadIdx.x >> 5); k < w1; k += PT / 32) { // warp-uniform
            const uint32_t i = 32u * sched.warps[k] + (threadIdx.x & 31);
            const float3 p = transfer_position(g, i < np_ ? pos[i] : make_float4(1.5f, 1.5f, 1.5f, 0.0f), 1.0f);
            p2g_scatter_kernel_one<MARK, MATCH>(i, g, params, p, rowx, rowy, rowz, nwx, nwy, nwz, marker, win, tile);
        }
        __syncthreads();
        for (int t = threadIdx.x; t < size; t += PT) {
            int cell_index = -1;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const uint32_t *const tc = tile + 4 * c * P2G_TILE + t;
                const long long num = tile_word(tc, tc + P2G_TILE), wq = tile_word(tc + 2 * P2G_TILE, tc + 3 * P2G_TILE);
                if (num == 0 && wq == 0) continue;
                if (cell_index < 0) cell_index = tile_cell(g, win, t);
                if (num != 0) fixed_add(&nw[c][cell_index].x, num);
                if (wq != 0) fixed_add(&nw[c][cell_index].y, wq);
            }
        }
        __syncthreads(); // the tile and shared_win are read to the end before the next item
    }
    // chunks of PT particles from the first one the schedule does not cover (all of them without schedule); a bounded grid strides over
    // them: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    for (uint32_t b = tail + blockIdx.x * PT; b < np_; b += gridDim.x * PT) { // block-uniform
        const uint32_t i = b + threadIdx.x;
        const bool valid = i < np_;
        const float3 p = transfer_position(g, valid ? pos[i] : make_float4(1.5f, 1.5f, 1.5f, 0.0f), 1.0f);
        const int3 cell = make_int3(min((int)p.x, g.nx - 1), min((int)p.y, g.ny - 1), min((int)p.z, g.nz - 1));
        const TileWindow win = scatter_window<P2G_TILE>(b, np_, valid, cell, scratch, &shared_win);
        const int size = win.ex * win.ey * win.ez;
        tile_zero<12, P2G_TILE>(tile, size);
        __syncthreads();
        p2g_scatter_kernel_one<MARK, MATCH>(i, g, params, p, rowx, rowy, rowz, nwx, nwy, nwz, marker, win, tile);
        __syncthreads();
        // flush: one global reduction per non-zero word; the next chunk's window is set up behind a barrier (scatter_window)
        for (int t = threadIdx.x; t < size; t += PT) {
            int cell_index = -1;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const uint32_t *const tc = tile + 4 * c * P2G_TILE + t;
                const long long num = tile_word(tc, tc + P2G_TILE), wq = tile_word(tc + 2 * P2G_TILE, tc + 3 * P2G_TILE);
                if (num == 0 && wq == 0) continue;
                if (cell_index < 0) cell_index = tile_cell(g, win, t);
                if (num != 0) fixed_add(&nw[c][cell_index].x, num);
                if (wq != 0) fixed_add(&nw[c][cell_index].y, wq);
            }
        }
    }
}

// Normalisation + global forces + "don't flow into solid" for the scatter form: transfer_gather_velocity.comp:116-127 -- and the
// accumulators are put back to zero on the way, so that no memset is needed: a particle of cell C only ever touches accumulators of
// cells C-1 .. C+1 (in every dimension), so the cells to visit are the one-cell dilation of the cells that hold particles
// (particle_words, written by marker_finalize_kernel).  One warp per 32 words of 32 cells: the lanes first work out which of their
// words are touched at all (almost none away from the fluid), then the warp walks the touched words with lane = cell (coalesced).
// Faces away from the fluid keep their previous value, as in the reference (SURVEY B6).
__device__ __forceinline__ unsigned pbits(const GridDim &g, const uint32_t *__restrict__ pw, int wpr, int xw, int y, int z) {
    if (xw < 0 || xw >= wpr || y < 0 || y >= g.ny || z < 0 || z >= g.nz) return 0u;
    return __ldg(pw + (z * g.ny + y) * wpr + xw);
}
// the cells of word w (xw, y, z) within one cell of a cell in particle_words; 0 for a thread beyond the last word
__device__ __forceinline__ unsigned particle_dilation(const GridDim &g, const uint32_t *__restrict__ particle_words, int wpr, int w, int &xw, int &y, int &z) {
    unsigned touched = 0;
    if (w < wpr * g.ny * g.nz) {
        xw = w % wpr;
        const int rowi = w / wpr;
        y = rowi % g.ny;
        z = rowi / g.ny;
#pragma unroll
        for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy) {
                const unsigned b = pbits(g, particle_words, wpr, xw, y + dy, z + dz);
                touched |= b | (b << 1) | (b >> 1) | (pbits(g, particle_words, wpr, xw - 1, y + dy, z + dz) >> 31) | (pbits(g, particle_words, wpr, xw + 1, y + dy, z + dz) << 31);
            }
        const int cells = min(32, g.nx - xw * 32);
        if (cells < 32) touched &= (1u << cells) - 1u;
    }
    return touched;
}
__global__ void __launch_bounds__(PT) p2g_normalize_kernel(GridDim g, int wpr, const uint32_t *__restrict__ particle_words, const StepParams *__restrict__ params,
                                                           const int8_t *__restrict__ marker, float *__restrict__ ux, float *__restrict__ uy,
                                                           float *__restrict__ uz, longlong2 *__restrict__ nwx, longlong2 *__restrict__ nwy,
                                                           longlong2 *__restrict__ nwz) {
    const int w = blockIdx.x * PT + threadIdx.x, lane = threadIdx.x & 31;
    int xw = 0, y = 0, z = 0;
    const unsigned touched = particle_dilation(g, particle_words, wpr, w, xw, y, z);
    unsigned todo = __ballot_sync(0xffffffffu, touched != 0u);
    float *const u[3] = {ux, uy, uz};
    longlong2 *const nw[3] = {nwx, nwy, nwz};
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const unsigned tw = __shfl_sync(0xffffffffu, touched, src);
        const int sxw = __shfl_sync(0xffffffffu, xw, src), sy = __shfl_sync(0xffffffffu, y, src), sz = __shfl_sync(0xffffffffu, z, src);
        if (!((tw >> lane) & 1u)) continue;
        const int i = lin(g, sxw * 32 + lane, sy, sz);
        const int ma = marker[i];
        const int mb[3] = {marker[i + 1], marker[i + g.sy], marker[i + g.sz]};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const longlong2 a = nw[c][i];
            if (a.x != 0 || a.y != 0) nw[c][i] = make_longlong2(0, 0);
            float out = 0.0f;
            if (ma == CELL_FLUID || mb[c] == CELL_FLUID) {
                if (ma != CELL_SOLID && mb[c] != CELL_SOLID) {
                    const double num = from_fixed<FIXED_VALUE_BITS>(a.x), den = from_fixed<FIXED_WEIGHT_BITS>(a.y);
                    const float v = a.y > 0 ? (float)(num / den) : 0.0f; // weight 0: no contribution reached this face
                    out = v + params->gravity_dt[c];
                }
            }
            u[c][i] = out;
        }
    }
}

// ------------------------------------------------------------------------------------------------ density projection
// Scatter counterpart of density_projection_gather_error.comp:41-97: dual cell d = trunc(pos - 0.5), cell centres d + {0,1}^3;
// warp-aggregated and tiled like the P2G scatter.
template <bool MATCH>
__device__ __forceinline__ void density_scatter_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params, const float3 p,
                                                             long long *__restrict__ density, const TileWindow &win, uint32_t *__restrict__ tile,
                                                             bool keep = true) {
    const uint32_t np = params->num_particles;
    if ((i & ~31u) >= np) return; // whole warp beyond the last particle
    const bool valid = i < np && keep; // a particle that is not kept still joins the warp's peer groups, with a key of its own
    const int dx = (int)(p.x - 0.5f), dy = (int)(p.y - 0.5f), dz = (int)(p.z - 0.5f);
    const float qx = (float)dx + 0.5f, qy = (float)dy + 0.5f, qz = (float)dz + 0.5f;
    const float wx[2] = {saturatef(1.0f - fabsf(qx - p.x)), saturatef(1.0f - fabsf(qx + 1.0f - p.x))};
    const float wy[2] = {saturatef(1.0f - fabsf(qy - p.y)), saturatef(1.0f - fabsf(qy + 1.0f - p.y))};
    const float wz[2] = {saturatef(1.0f - fabsf(qz - p.z)), saturatef(1.0f - fabsf(qz + 1.0f - p.z))};
    const int base = lin(g, dx, dy, dz);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = valid ? wx[k & 1] * wy[(k >> 1) & 1] * wz[k >> 2] : 0.0f;
    const bool live = warp_group_sum<MATCH, 8>(valid ? base : -1 - (int)(threadIdx.x & 31), acc) && valid; // a head issues the adds
    const int e0 = tile_box_entry(win, dx, dy, dz);
    if (__all_sync(0xffffffffu, e0 >= 0 || !live)) { // warp-uniform: every head's eight cells go to the tile; low words first, as in P2G
        if (live) {
            uint32_t *const t = tile + e0;
            const int sy = win.ex, sz = win.ex * win.ey;
            uint32_t h[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) h[k] = tile_add_lo(t + (k & 1) + ((k >> 1) & 1) * sy + (k >> 2) * sz, acc[k] > 0.0f ? to_fixed<FIXED_WEIGHT_BITS>(acc[k]) : 0);
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(t + DENSITY_TILE + (k & 1) + ((k >> 1) & 1) * sy + (k >> 2) * sz, h[k]);
        }
    } else if (live) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (acc[k] > 0.0f) {
                const long long q = to_fixed<FIXED_WEIGHT_BITS>(acc[k]);
                const int e = tile_entry(win, dx + (k & 1), dy + ((k >> 1) & 1), dz + (k >> 2));
                if (e >= 0) tile_add(tile + e, tile + DENSITY_TILE + e, q);
                else fixed_add(density + base + (k & 1) + ((k >> 1) & 1) * g.sy + (k >> 2) * g.sz, q);
            }
    }
}
// The whole scatter: the particles `keep(position)` accepts add their weights (every particle of the fused and unfiltered scatters)
template <bool MATCH, class Keep>
__device__ __forceinline__ void density_scatter_all(GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos,
                                                    long long *__restrict__ density, const ScatterSchedule &sched, Keep keep) {
    __shared__ __align__(16) uint32_t tile[2 * DENSITY_TILE]; // low words, high words
    __shared__ int scratch[PT / 32 + 1][8];
    __shared__ TileWindow shared_win;
    const uint32_t np_ = params->num_particles;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // the work items of the brick schedule: one window, one zeroing and one flush per item, its warps 8 at a time
    uint32_t tail;
    const uint32_t items = schedule_items(sched, tail);
    for (uint32_t it = blockIdx.x; it < items; it += gridDim.x) { // block-uniform
        const uint32_t w0 = sched.item_start[it], w1 = it + 1 < items ? sched.item_start[it + 1] : tail / 32u;
        const TileWindow win = item_window<DENSITY_TILE>(g, sched, it, w0, w1, np_, pos, 0.5f, scratch, &shared_win);
        const int size = win.ex * win.ey * win.ez;
        tile_zero<2, DENSITY_TILE>(tile, size);
        __syncthreads();
        for (uint32_t k = w0 + warp; k < w1; k += PT / 32) { // warp-uniform
            const uint32_t i = 32u * sched.warps[k] + lane;
            const float4 q = i < np_ ? pos[i] : make_float4(1.5f, 1.5f, 1.5f, 0.0f);
            density_scatter_kernel_one<MATCH>(i, g, params, transfer_position(g, q, 0.5f), density, win, tile, keep(q));
        }
        __syncthreads();
        for (int t = threadIdx.x; t < size; t += PT) { // flush, as in p2g_scatter_kernel
            const long long q = tile_word(tile + t, tile + DENSITY_TILE + t);
            if (q != 0) fixed_add(density + tile_cell(g, win, t), q);
        }
        // the next item's window is set up behind a barrier (item_window); the first chunk's too (scatter_window)
    }
    // chunks of PT particles from the first one the schedule does not cover (all of them without schedule); a bounded grid strides over
    // them: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    for (uint32_t b = tail + blockIdx.x * PT; b < np_; b += gridDim.x * PT) { // block-uniform
        const uint32_t i = b + threadIdx.x;
        const bool valid = i < np_;
        const float4 q = valid ? pos[i] : make_float4(1.5f, 1.5f, 1.5f, 0.0f);
        const float3 p = transfer_position(g, q, 0.5f);
        const int3 cell = make_int3(min((int)p.x, g.nx - 1), min((int)p.y, g.ny - 1), min((int)p.z, g.nz - 1));
        const TileWindow win = scatter_window<DENSITY_TILE>(b, np_, valid, cell, scratch, &shared_win);
        const int size = win.ex * win.ey * win.ez;
        tile_zero<2, DENSITY_TILE>(tile, size);
        __syncthreads();
        density_scatter_kernel_one<MATCH>(i, g, params, p, density, win, tile, keep(q));
        __syncthreads();
        for (int t = threadIdx.x; t < size; t += PT) {
            const long long q = tile_word(tile + t, tile + DENSITY_TILE + t);
            if (q != 0) fixed_add(density + tile_cell(g, win, t), q);
        }
    }
}
template <bool MATCH>
__global__ void __launch_bounds__(PT) density_scatter_kernel(GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos,
                                                             long long *__restrict__ density, ScatterSchedule sched) {
    density_scatter_all<MATCH>(g, params, pos, density, sched, [](const float4 &) { return true; });
}
// The interfacial tension's phase-B splat: only the particles whose tag (the fourth word's bits) is in the set add their weights.  The others
// still take part in the windows and the warp's peer matching, but with a key of their own, so a kept particle's peer group holds only kept
// particles: where both phases share a cell within a warp, the group sums (and their fixed-point roundings) differ from the all-particle
// splat's.  The phase field takes any pair of splats (DESIGN.md §8 "Interfacial tension").
template <bool MATCH>
__global__ void __launch_bounds__(PT) phase_scatter_kernel(GridDim g, const StepParams *__restrict__ params, const float4 *__restrict__ pos,
                                                           long long *__restrict__ density, ScatterSchedule sched,
                                                           const InterfacialTensionBlock *__restrict__ blk) {
    __shared__ uint32_t set[INTERFACE_TAGS_MAX];
    const uint32_t count = blk->count;
    if (threadIdx.x < INTERFACE_TAGS_MAX) set[threadIdx.x] = blk->tag[threadIdx.x];
    __syncthreads();
    density_scatter_all<MATCH>(g, params, pos, density, sched, [&](const float4 &q) {
        const uint32_t t = __float_as_uint(q.w);
        bool in = false;
#pragma unroll
        for (int k = 0; k < INTERFACE_TAGS_MAX; ++k) in |= k < (int)count && set[k] == t;
        return in;
    });
}

// Stage 7 with the density scatter of stage 9 fused in behind it (one GPU): every particle is advected by advect_kernel_one and its new
// position goes on to density_scatter_kernel_one from the block's registers and shared memory, never from the position array.  The work order
// is density_scatter_kernel's -- the schedule's work items, 8 of an item's warps at a time, then 256-particle chunks for the rest -- so
// every warp holds the particles it holds there and forms the same peer groups and integers.  An item's warps are advected first, their
// positions kept in `moved`; the item's window (and s.item_box) come from them, then the tile is zeroed, scattered into and flushed.  One
// block's tile atomics overlap another's advection traffic on the same SM, and the positions are not read a second time.  The density
// volume must be all zero on entry (HybridFluid::density_zero_).
template <bool MATCH>
__global__ void __launch_bounds__(PT) advect_density_kernel(GridDim g, const StepParams *__restrict__ params, float4 *__restrict__ pos,
                                                            float4 *__restrict__ rowx, float4 *__restrict__ rowy, float4 *__restrict__ rowz,
                                                            const float *__restrict__ ux, const float *__restrict__ uy, const float *__restrict__ uz,
                                                            const uint2 *__restrict__ vox, int8_t *__restrict__ marker, long long *__restrict__ density,
                                                            ScatterSchedule sched) {
    __shared__ __align__(16) uint32_t tile[2 * DENSITY_TILE]; // low words, high words
    __shared__ float3 moved[SCHED_K * 32];                     // the new positions of an item's particles, as the scatter sees them
    __shared__ int scratch[PT / 32 + 1][8];
    __shared__ TileWindow shared_win;
    const uint32_t np_ = params->num_particles;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t tail;
    const uint32_t items = schedule_items(sched, tail);
    for (uint32_t it = blockIdx.x; it < items; it += gridDim.x) { // block-uniform
        const uint32_t w0 = sched.item_start[it], w1 = it + 1 < items ? sched.item_start[it + 1] : tail / 32u;
        int mn[3] = {BOX_EMPTY, BOX_EMPTY, BOX_EMPTY}, mx[3] = {-BOX_EMPTY, -BOX_EMPTY, -BOX_EMPTY};
        for (uint32_t k = w0 + warp; k < w1; k += PT / 32) { // warp-uniform
            const uint32_t i = 32u * sched.warps[k] + lane;
            const float3 p = transfer_position(g, advect_kernel_one<false>(i, g, params, pos, rowx, rowy, rowz, ux, uy, uz, vox, marker, MigrateOut{}), 0.5f);
            moved[(k - w0) * 32 + lane] = p;
            if (i < np_) extend_box(g, p, mn, mx);
        }
        const TileWindow win = item_box_window<DENSITY_TILE>(g, sched, it, mn, mx, scratch, &shared_win);
        const int size = win.ex * win.ey * win.ez;
        tile_zero<2, DENSITY_TILE>(tile, size);
        __syncthreads();
        for (uint32_t k = w0 + warp; k < w1; k += PT / 32) // warp-uniform; each warp reads back only what it wrote
            density_scatter_kernel_one<MATCH>(32u * sched.warps[k] + lane, g, params, moved[(k - w0) * 32 + lane], density, win, tile);
        __syncthreads();
        for (int t = threadIdx.x; t < size; t += PT) {
            const long long q = tile_word(tile + t, tile + DENSITY_TILE + t);
            if (q != 0) fixed_add(density + tile_cell(g, win, t), q);
        }
    }
    for (uint32_t b = tail + blockIdx.x * PT; b < np_; b += gridDim.x * PT) { // block-uniform
        const uint32_t i = b + threadIdx.x;
        const float3 p = transfer_position(g, advect_kernel_one<false>(i, g, params, pos, rowx, rowy, rowz, ux, uy, uz, vox, marker, MigrateOut{}), 0.5f);
        const int3 cell = make_int3(min((int)p.x, g.nx - 1), min((int)p.y, g.ny - 1), min((int)p.z, g.nz - 1));
        const TileWindow win = scatter_window<DENSITY_TILE>(b, np_, i < np_, cell, scratch, &shared_win);
        const int size = win.ex * win.ey * win.ez;
        tile_zero<2, DENSITY_TILE>(tile, size);
        __syncthreads();
        density_scatter_kernel_one<MATCH>(i, g, params, p, density, win, tile);
        __syncthreads();
        for (int t = threadIdx.x; t < size; t += PT) {
            const long long q = tile_word(tile + t, tile + DENSITY_TILE + t);
            if (q != 0) fixed_add(density + tile_cell(g, win, t), q);
        }
    }
}

// density_projection_gather_error.comp:99-199: the right-hand side of FLUID cell i from its density sum q
__device__ __forceinline__ float density_rhs_of(const GridDim &g, const StepParams *__restrict__ params, const int8_t *__restrict__ marker, int64_t i,
                                                long long q) {
    float d = (float)from_fixed<FIXED_WEIGHT_BITS>(q);
    const int m[6] = {marker[i + 1], marker[i + g.sy], marker[i + g.sz], marker[i - 1], marker[i - g.sy], marker[i - g.sz]};
    bool any_air = false;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        if (m[k] == CELL_SOLID) d += 0.5625f;
        any_air = any_air || (m[k] == CELL_AIR);
    }
    if (any_air) d = fmaxf(8.0f, d);
    d = 1.0f - d / 8.0f;
    d = fminf(fmaxf(d, -0.5f), 0.5f);
    d /= params->dt;
    return d;
}
__global__ void __launch_bounds__(PT) density_rhs_kernel(GridDim g, const StepParams *__restrict__ params,
                                                         const int8_t *__restrict__ marker, const long long *__restrict__ density,
                                                         float *__restrict__ rhs) {
    const int64_t i = (int64_t)blockIdx.x * PT + threadIdx.x;
    if (i >= g.n) return;
    if (marker[i] != CELL_FLUID) return;
    rhs[i] = density_rhs_of(g, params, marker, i, density[i]);
}
// The sparse finish after advect_density_kernel: the particles of stage 7 marked the cells in particle_words (stage 8), and each of them
// added only to the cells within one cell of its own.  So the dilation of those cells holds every non-zero density word and every FLUID cell:
// the warp walks it as p2g_normalize_kernel does, writes the right-hand side of the FLUID cells and puts the words back to zero.
__global__ void __launch_bounds__(PT) density_finish_sparse_kernel(GridDim g, int wpr, const uint32_t *__restrict__ particle_words,
                                                                   const StepParams *__restrict__ params, const int8_t *__restrict__ marker,
                                                                   long long *__restrict__ density, float *__restrict__ rhs) {
    const int w = blockIdx.x * PT + threadIdx.x, lane = threadIdx.x & 31;
    int xw = 0, y = 0, z = 0;
    const unsigned touched = particle_dilation(g, particle_words, wpr, w, xw, y, z);
    unsigned todo = __ballot_sync(0xffffffffu, touched != 0u);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const unsigned tw = __shfl_sync(0xffffffffu, touched, src);
        const int sxw = __shfl_sync(0xffffffffu, xw, src), sy = __shfl_sync(0xffffffffu, y, src), sz = __shfl_sync(0xffffffffu, z, src);
        if (!((tw >> lane) & 1u)) continue;
        const int i = lin(g, sxw * 32 + lane, sy, sz);
        const long long q = density[i];
        if (q != 0) density[i] = 0;
        if (marker[i] == CELL_FLUID) rhs[i] = density_rhs_of(g, params, marker, i, q);
    }
}

// ------------------------------------------------------------------------------------------------ binning
// particle_binning_rewrite_particles.comp: the cell lists ARE the sorted order -- dst[j] = src[order[j]] (x-fastest cell order,
// ascending previous index inside a cell: deterministic; the reference's atomic ranks are not, and its inclusive - index
// addressing loses a particle, SURVEY B2).  The whole float4 moves: its fourth word is the particle's tag (raw bits, never arithmetic).
__device__ __forceinline__ void binning_permute_kernel_one(uint32_t j, const StepParams *__restrict__ params, const uint32_t *__restrict__ order,
                                                             const float4 *__restrict__ src, float4 *__restrict__ dst) {
    if (j >= params->num_particles) return;
    dst[j] = src[order[j]];
}
__global__ void __launch_bounds__(PT) binning_permute_kernel(const StepParams *__restrict__ params, const uint32_t *__restrict__ order,
                                                             const float4 *__restrict__ src, float4 *__restrict__ dst) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t j = blockIdx.x * PT + threadIdx.x; (j & ~31u) < np_; j += gridDim.x * PT) binning_permute_kernel_one(j, params, order, src, dst);
}

} // namespace

// ------------------------------------------------------------------------------------------------ launchers
int binning_scan_blocks(const GridDim &g) { return blocks_for(g.n + 1, SCAN_THREADS * SCAN_ITEMS); }

int exclusive_scan_blocks(int64_t n) { return blocks_for(n, SCAN_THREADS * SCAN_ITEMS); }

void launch_exclusive_scan(cudaStream_t st, uint32_t *data, int64_t n, uint32_t *block_sums) {
    const int nb = exclusive_scan_blocks(n);
    BLUB_LAUNCH(scan_block_sums_kernel, nb, SCAN_THREADS, 0, st, data, n, block_sums);
    BLUB_LAUNCH(scan_sums_kernel, 1, 1024, 0, st, block_sums, nb);
    BLUB_LAUNCH(scan_apply_kernel, nb, SCAN_THREADS, 0, st, data, n, block_sums);
}

void launch_cell_lists(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, float clamp_lo, const CellLists &l) {
    const int64_t n1 = g.n + 1; // cell_start[n] = number of particles
    const int nb = binning_scan_blocks(g);
    BLUB_CUDA_CHECK(cudaMemsetAsync(l.cell_start, 0, (size_t)n1 * sizeof(uint32_t), st));
    if (np_upper > 0) BLUB_LAUNCH(cell_count_kernel, particle_blocks(np_upper), PT, 0, st, g, params, pos, clamp_lo, l.cell_start, l.cell_slot);
    BLUB_LAUNCH(scan_block_sums_kernel, nb, SCAN_THREADS, 0, st, l.cell_start, n1, l.block_sums);
    BLUB_LAUNCH(scan_sums_kernel, 1, 1024, 0, st, l.block_sums, nb);
    BLUB_LAUNCH(scan_apply_kernel, nb, SCAN_THREADS, 0, st, l.cell_start, n1, l.block_sums);
    if (np_upper == 0) return;
    BLUB_LAUNCH(cell_fill_kernel, particle_blocks(np_upper), PT, 0, st, params, l.cell_slot, l.cell_start, l.arrival);
    BLUB_CUDA_CHECK(cudaMemsetAsync(l.crowd.count, 0, sizeof(uint32_t), st));
    BLUB_LAUNCH(cell_canonicalize_kernel, particle_blocks(np_upper), PT, 0, st, params, l.cell_slot, l.cell_start, l.arrival, l.order, l.crowd);
    BLUB_LAUNCH(crowded_canonicalize_kernel, 2 * device_sm_count(), PT, 0, st, l.cell_start, l.arrival, l.order, l.crowd); // 2 blocks per SM
}

void launch_marker_from_lists(cudaStream_t st, const GridDim &g, const CellLists &l, int8_t *marker, const uint2 *vox, const FluidBits &bits,
                              uint32_t *particle_words) {
    BLUB_LAUNCH(marker_from_lists_kernel, blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT), PT, 0, st, g, bits, l.cell_start, marker, vox, particle_words);
}

void launch_boundary_marker(cudaStream_t st, const GridDim &g, int8_t *marker, const uint2 *vox, const FluidBits &bits, uint32_t *particle_words) {
    BLUB_LAUNCH(marker_finalize_kernel, blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT), PT, 0, st, g, bits, marker, vox, particle_words);
}

void launch_fluid_bits(cudaStream_t st, const GridDim &g, const int8_t *marker, const FluidBits &bits) {
    BLUB_LAUNCH(fluid_bits_kernel, blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT), PT, 0, st, g, bits, marker);
}

// opt in to > 48 KB of dynamic shared memory; per device, so every HybridFluid constructor calls it after cudaSetDevice
void configure_transfer_kernels() {
    BLUB_CUDA_CHECK(cudaFuncSetAttribute(p2g_gather_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, GATHER_SMEM_BYTES));
    BLUB_CUDA_CHECK(cudaFuncSetAttribute(p2g_gather_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, GATHER_SMEM_BYTES));
    BLUB_CUDA_CHECK(cudaFuncSetAttribute(p2g_gather_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GATHER_SMEM_BYTES));
    // the P2G scatter tile: the whole shared-memory carveout, so that 4 blocks of P2G_TILE_BYTES are resident per SM
    for (const auto kernel : {p2g_scatter_kernel<true, true>, p2g_scatter_kernel<true, false>}) {
        BLUB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, P2G_TILE_BYTES));
        BLUB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
}


void launch_p2g_gather(cudaStream_t st, const GridDim &g, const StepParams *params, const CellLists &l, const float4 *pos, float4 *const row[3],
                       const int8_t *marker, float *const u[3]) {
    // 2 blocks of 8 warps per SM walk the crowded-cell list (usually empty: the kernel then costs a launch)
    const int CROWD_BLOCKS = 2 * device_sm_count();
    const dim3 grid((g.nx + GXS - 1) / GXS, (g.ny + GLY - 1) / GLY, (g.nz + GW - 1) / GW);
    // Faces no block stores (blocks without particles return at once) keep their previous value, as in the reference, which only
    // writes faces that touch a FLUID cell (transfer_gather_velocity.comp:41-47, SURVEY B6): nothing reads them before
    // divergence_remove rewrites every face.
    BLUB_LAUNCH(p2g_crowded_kernel<0>, CROWD_BLOCKS, PT, 0, st, g, l.cell_start, l.order, pos, row[0], l.crowd);
    BLUB_LAUNCH(p2g_gather_kernel<0>, grid, GATHER_THREADS, GATHER_SMEM_BYTES, st, g, params, l.cell_start, l.order, pos, row[0], marker, u[0], l.crowd);
    BLUB_LAUNCH(p2g_crowded_kernel<1>, CROWD_BLOCKS, PT, 0, st, g, l.cell_start, l.order, pos, row[1], l.crowd);
    BLUB_LAUNCH(p2g_gather_kernel<1>, grid, GATHER_THREADS, GATHER_SMEM_BYTES, st, g, params, l.cell_start, l.order, pos, row[1], marker, u[1], l.crowd);
    BLUB_LAUNCH(p2g_crowded_kernel<2>, CROWD_BLOCKS, PT, 0, st, g, l.cell_start, l.order, pos, row[2], l.crowd);
    BLUB_LAUNCH(p2g_gather_kernel<2>, grid, GATHER_THREADS, GATHER_SMEM_BYTES, st, g, params, l.cell_start, l.order, pos, row[2], marker, u[2], l.crowd);
}

// Which warp aggregation the scatter kernels use: peer groups found with match.any (default) or runs of adjacent lanes (the comparison
// path: BLUB_SCATTER_AGG=adjacent, read once).
static bool scatter_groups_by_match() {
    static const bool by_match = [] {
        const char *e = std::getenv("BLUB_SCATTER_AGG");
        return !(e && std::strcmp(e, "adjacent") == 0);
    }();
    return by_match;
}

// Whether re-sorts build the brick schedule of the scatters: BLUB_SCATTER_SCHEDULE=off (read once) keeps both on the 256-particle
// chunks, the reference the schedule is tested against.
bool scatter_schedule_enabled() {
    static const bool on = [] {
        const char *e = std::getenv("BLUB_SCATTER_SCHEDULE");
        return !(e && std::strcmp(e, "off") == 0);
    }();
    return on;
}

// How many waves of 4 blocks per SM the work items must fill before P2G walks them: P2G_MIN_ITEM_WAVES, or BLUB_P2G_ITEM_WAVES=N (0..8,
// read once; a test hook: 0 walks the items whenever the schedule is valid, so that small grids reach the item path).
static uint32_t p2g_item_waves() {
    static const uint32_t waves = [] {
        const char *e = std::getenv("BLUB_P2G_ITEM_WAVES");
        if (e && e[0] >= '0' && e[0] <= '0' + P2G_MIN_ITEM_WAVES && e[1] == '\0') return (uint32_t)(e[0] - '0');
        return (uint32_t)P2G_MIN_ITEM_WAVES;
    }();
    return waves;
}

int scatter_schedule_bricks(const GridDim &g) {
    return ((g.nx + SCHED_BX - 1) / SCHED_BX) * ((g.ny + SCHED_BY - 1) / SCHED_BY) * ((g.nz + SCHED_BZ - 1) / SCHED_BZ);
}
uint32_t scatter_schedule_max_items(const GridDim &g, uint32_t max_warps) { return (uint32_t)scatter_schedule_bricks(g) + max_warps / SCHED_K + 1; }

void launch_scatter_schedule(cudaStream_t st, const GridDim &g, const CellLists &l, const ScatterSchedule &s) {
    const int nb = s.nbricks;
    BLUB_LAUNCH(schedule_count_kernel, blocks_for(nb, PT), PT, 0, st, g, l.cell_start, s);
    launch_exclusive_scan(st, s.brick_warps, (int64_t)nb + 1, l.block_sums);
    launch_exclusive_scan(st, s.brick_items, (int64_t)nb + 1, l.block_sums);
    BLUB_LAUNCH(schedule_fill_kernel, blocks_for((int64_t)nb * 32, PT), PT, 0, st, g, l.cell_start, s);
    BLUB_CUDA_CHECK(cudaMemsetAsync(s.valid, 1, sizeof(uint32_t), st)); // non-zero: valid
}

void launch_p2g_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, float4 *const row[3],
                        longlong2 *const nw[3], int8_t *marker, bool clear_accumulators, const ScatterSchedule &sched) {
    // transfer_clear.comp: marker <- AIR.  The (num, weight) volumes (they replace the linked-list head volume) are all zero here on one GPU:
    // they are allocated zeroed and launch_p2g_finish puts back to zero what the scatter touched.  A z-slab rank also receives partial sums
    // from its neighbours in the overlap planes, some of them from particles whose cells it never sees: it clears the volumes the plain way.
    BLUB_CUDA_CHECK(cudaMemsetAsync(marker, 0xFF, (size_t)g.n, st));
    if (clear_accumulators)
        for (int c = 0; c < 3; ++c) BLUB_CUDA_CHECK(cudaMemsetAsync(nw[c], 0, (size_t)g.n * sizeof(longlong2), st));
    if (np_upper == 0) return;
    const auto kernel = scatter_groups_by_match() ? p2g_scatter_kernel<true, true> : p2g_scatter_kernel<true, false>;
    BLUB_LAUNCH(kernel, particle_blocks(np_upper), PT, P2G_TILE_BYTES, st, g, params, pos, row[0], row[1], row[2], nw[0], nw[1], nw[2], marker, sched,
                p2g_item_waves() * 4u * (uint32_t)device_sm_count());
}

void launch_p2g_finish(cudaStream_t st, const GridDim &g, const StepParams *params, float *const u[3], longlong2 *const nw[3], int8_t *marker,
                       const uint2 *vox, const FluidBits &bits, uint32_t *particle_words) {
    launch_boundary_marker(st, g, marker, vox, bits, particle_words);
    BLUB_LAUNCH(p2g_normalize_kernel, blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT), PT, 0, st, g, bits.wpr, particle_words, params, marker, u[0], u[1], u[2], nw[0],
                nw[1], nw[2]);
}

void launch_density_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, long long *density,
                            const ScatterSchedule &sched) {
    BLUB_CUDA_CHECK(cudaMemsetAsync(density, 0, (size_t)g.n * sizeof(long long), st));
    if (np_upper == 0) return;
    const auto kernel = scatter_groups_by_match() ? density_scatter_kernel<true> : density_scatter_kernel<false>;
    BLUB_LAUNCH(kernel, particle_blocks(np_upper), PT, 0, st, g, params, pos, density, sched);
}

void launch_phase_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, long long *density,
                          const ScatterSchedule &sched, const InterfacialTensionBlock *blk) {
    BLUB_CUDA_CHECK(cudaMemsetAsync(density, 0, (size_t)g.n * sizeof(long long), st));
    if (np_upper == 0) return;
    const auto kernel = scatter_groups_by_match() ? phase_scatter_kernel<true> : phase_scatter_kernel<false>;
    BLUB_LAUNCH(kernel, particle_blocks(np_upper), PT, 0, st, g, params, pos, density, sched, blk);
}

void launch_density_finish(cudaStream_t st, const GridDim &g, const StepParams *params, const int8_t *marker, const long long *density, float *rhs) {
    BLUB_LAUNCH(density_rhs_kernel, blocks_for(g.n, PT), PT, 0, st, g, params, marker, density, rhs);
}

void launch_density_rhs(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos,
                        const int8_t *marker, long long *density, float *rhs, const ScatterSchedule &sched) {
    launch_density_scatter(st, g, params, np_upper, pos, density, sched);
    launch_density_finish(st, g, params, marker, density, rhs);
}

void launch_advect_density(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                           float *const u[3], const uint2 *vox, int8_t *marker, long long *density, const ScatterSchedule &sched) {
    if (np_upper == 0) return;
    const auto kernel = scatter_groups_by_match() ? advect_density_kernel<true> : advect_density_kernel<false>;
    BLUB_LAUNCH(kernel, particle_blocks(np_upper), PT, 0, st, g, params, pos, row[0], row[1], row[2], u[0], u[1], u[2], vox, marker, density, sched);
}

void launch_density_finish_sparse(cudaStream_t st, const GridDim &g, const StepParams *params, const int8_t *marker, const FluidBits &bits,
                                  const uint32_t *particle_words, long long *density, float *rhs) {
    BLUB_LAUNCH(density_finish_sparse_kernel, blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT), PT, 0, st, g, bits.wpr, particle_words, params, marker, density, rhs);
}

void launch_binning(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *src, float4 *dst, const CellLists &l) {
    if (np_upper == 0) return;
    launch_cell_lists(st, g, params, np_upper, src, 0.0f, l);
    BLUB_LAUNCH(binning_permute_kernel, particle_blocks(np_upper), PT, 0, st, params, l.order, src, dst);
}

} // namespace blub
