// load_kernels.cu -- solid load probes (DESIGN.md §8 "Solid load probes").  Not in the reference.
//
// Right after the velocity solve (end of stage 2) every probe box is walked once: each SOLID cell inside it looks at its six neighbours, and
// every FLUID one inside the grid makes a wetted face.  The face force is q = -p_vel * inv_dt (pressure / density; the solver's volume
// holds -p * dt / density) along the face axis, pointing from the fluid cell into the solid one; the torque is (face centre - pivot) x force, so each
// of its two non-zero components is the single float32 product r_b * q with a sign.  Both are turned into int64 fixed point (2^16 and 2^8)
// and added with integer atomics: the record is exact and does not depend on the launch order.
#include <algorithm>

#include "fluid_kernels.hpp"
#include "solid_faces.cuh"

namespace blub {

namespace {

constexpr int PT = 256;

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// The step's slot of every probe: step number set, sums zero.  Runs in front of solid_load_kernel.
__global__ void load_slot_clear_kernel(const StepParams *__restrict__ params, int num_probes, BlubSolidLoad *__restrict__ ring) {
    const int p = threadIdx.x;
    if (p >= num_probes) return;
    const uint32_t step = params->step_count;
    BlubSolidLoad &r = ring[(size_t)p * LOAD_HISTORY_LENGTH + step % LOAD_HISTORY_LENGTH];
    r.step = step;
    r.wetted_faces = 0u;
    for (int k = 0; k < 3; ++k) r.force_fx[k] = r.torque_fx[k] = 0;
}

// blockIdx.y = probe; the blocks of x stride over the probe box's cells, x fastest.  Each thread adds up its faces in registers
// (add_wetted_faces), the block reduces them (block_load_sum) and issues one global atomic per non-zero field.
__global__ void __launch_bounds__(PT) solid_load_kernel(GridDim g, const StepParams *__restrict__ params, const LoadProbeBox *__restrict__ probes,
                                                        const int8_t *__restrict__ marker, const float *__restrict__ p_vel, BlubSolidLoad *__restrict__ ring) {
    __shared__ unsigned long long part[PT / 32][LOAD_FIELDS];
    const LoadProbeBox b = probes[blockIdx.y];
    // a thread takes 4 cells of a row at a time (x aligned to 4: nx is a multiple of 8 and the marker volume starts 256-byte aligned), one
    // 32-bit marker load for all four
    const int qx0 = b.lo[0] >> 2;
    const uint32_t ex = (uint32_t)(((b.hi[0] + 3) >> 2) - qx0), ey = (uint32_t)(b.hi[1] - b.lo[1]);
    const uint32_t quads = ex * ey * (uint32_t)(b.hi[2] - b.lo[2]);
    if (blockIdx.x * PT >= quads) return; // the whole block: the grid is sized for the largest box
    const float inv_dt = params->inv_dt;
    long long acc[6] = {0, 0, 0, 0, 0, 0};
    unsigned long long faces = 0;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < quads; i += gridDim.x * PT) {
        const uint32_t t = i / ex;
        const int x0 = (qx0 + (int)(i - t * ex)) << 2, y = b.lo[1] + (int)(t % ey), z = b.lo[2] + (int)(t / ey);
        const int64_t s0 = (int64_t)x0 + (int64_t)y * g.sy + (int64_t)z * g.sz;
        const uint32_t word = *reinterpret_cast<const uint32_t *>(marker + s0);
        uint32_t solid = __vcmpeq4(word, 0u); // 0xFF in every byte whose cell is SOLID
        if (!solid) continue;
#pragma unroll 1
        for (int j = 0; j < 4; ++j) {
            if (!((solid >> (8 * j)) & 1u) || x0 + j < b.lo[0] || x0 + j >= b.hi[0]) continue;
            const int c[3] = {x0 + j, y, z};
            faces += add_wetted_faces(g, marker, p_vel, inv_dt, c, s0 + j, b.pivot, acc);
        }
    }
    const unsigned long long sum = block_load_sum<PT>(acc, faces, part);
    if (sum == 0) return;
    BlubSolidLoad &rec = ring[(size_t)blockIdx.y * LOAD_HISTORY_LENGTH + params->step_count % LOAD_HISTORY_LENGTH];
    if (threadIdx.x < 3) atomicAdd(reinterpret_cast<unsigned long long *>(&rec.force_fx[threadIdx.x]), sum);
    else if (threadIdx.x < 6) atomicAdd(reinterpret_cast<unsigned long long *>(&rec.torque_fx[threadIdx.x - 3]), sum);
    else atomicAdd(&rec.wetted_faces, (uint32_t)sum);
}

} // namespace

void launch_solid_loads(cudaStream_t st, const GridDim &g, const StepParams *params, int num_probes, uint32_t max_cells, const LoadProbeBox *probes,
                        const int8_t *marker, const float *p_vel, BlubSolidLoad *ring) {
    if (num_probes <= 0) return;
    BLUB_LAUNCH(load_slot_clear_kernel, 1, 32, 0, st, params, num_probes, ring);
    // a box has at most as many 4-cell quads as cells
    const dim3 grid((unsigned)std::min(blocks_for(max_cells, PT), device_sm_count() * 8), (unsigned)num_probes);
    BLUB_LAUNCH(solid_load_kernel, grid, PT, 0, st, g, params, probes, marker, p_vel, ring);
}

} // namespace blub
