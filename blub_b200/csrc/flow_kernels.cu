// flow_kernels.cu -- fluid sources and drains (sm_90a): the flow prologue at the start of stage 0, before P2G.
//
// All of it runs on the device-resident particle count (StepParams::num_particles) inside the captured step, with no host synchronisation:
//   1. flow_count_kernel: one pass over the particles.  A particle whose cell lies in a drain box is counted per FLOW_CHUNK chunk and the
//      lowest such index is kept (warp-aggregated integer atomics); a particle in a source cell is counted for that cell and gets the source velocity
//      (rows (0, 0, 0, v_c)) at once -- sources and drains never overlap, so this is the velocity it has after the drain too.
//   2. drains: exclusive scan of the chunk counts, then flow_compact_kernel writes the survivors from the first drained index on into the
//      spare arrays in their order (block-wide ballot scan inside a chunk), and flow_copy_back_kernel copies that suffix back.  Both return
//      at once when no particle was drained: such a step does not move the particle arrays.
//   3. sources: flow_need_kernel turns the counts into the number of particles each source cell gets, an exclusive scan orders them by
//      (source, cell x fastest, slot), and flow_emit_kernel appends them after the survivors up to the capacity and sets the new count and
//      the cumulative counters.
// The jitter of an emitted particle is a function of (step, cell, slot): Xoshiro256pp seeded with step << 32 | cell, 8 slots x 3 draws; it carries
// the tag of its source.
//
// Particle tags share the drains' cell rule and live here too: paint_tags_kernel sets the tag of the particles whose cell lies in a box, and
// tag_census_kernel adds up count, positions, velocities and cell bounds per tag.  A tag is the raw bits of the fourth word of a position:
// every path copies it, none puts it through float arithmetic.
#include <algorithm>
#include <climits>

#include "fluid_kernels.hpp"
#include "xoshiro.hpp"

namespace blub {
namespace {

constexpr int PT = 256;
constexpr uint32_t NONE = 0xFFFFFFFFu;
static_assert(FLOW_CHUNK % PT == 0, "a chunk is a whole number of block rounds");

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// the cell the binning assigns (transfer_position with clamp_lo = 0, then cell_of_position, transfer_kernels.cu); the velocity transfer clamps
// at 1.0 instead, which differs only for particles in [0, 1) handed in from outside: a simulated particle stays in [1.001, dim - 1.001]
__device__ __forceinline__ int3 flow_cell(const GridDim &g, const float4 &p) {
    const float x = fminf(fmaxf(p.x, 0.0f), (float)g.nx - 1.0f), y = fminf(fmaxf(p.y, 0.0f), (float)g.ny - 1.0f),
                z = fminf(fmaxf(p.z, 0.0f), (float)g.nz - 1.0f);
    return make_int3(min((int)x, g.nx - 1), min((int)y, g.ny - 1), min((int)z, g.nz - 1));
}
__device__ __forceinline__ bool in_box(const FlowBox &b, int3 c) {
    return c.x >= b.lo[0] && c.x < b.hi[0] && c.y >= b.lo[1] && c.y < b.hi[1] && c.z >= b.lo[2] && c.z < b.hi[2];
}
__device__ __forceinline__ bool drained(const FlowSet &fs, int3 c) {
    for (int d = 0; d < fs.num_drains; ++d)
        if (in_box(fs.drain[d], c)) return true;
    return false;
}

__global__ void __launch_bounds__(PT) flow_count_kernel(GridDim g, const StepParams *__restrict__ params, FlowSet fs, const float4 *__restrict__ pos,
                                                        float4 *__restrict__ rx, float4 *__restrict__ ry, float4 *__restrict__ rz, FlowScratch s) {
    const uint32_t n = params->num_particles;
    if (blockIdx.x == 0 && threadIdx.x == 0) s.scalars[2] = n;
    const int lane = threadIdx.x & 31;
    // whole warps walk the loop (a warp's 32 consecutive indices lie in one FLOW_CHUNK chunk): the drain atomics are warp-aggregated, one
    // add to the chunk count, one to the step total and one min per warp that drains anything
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < n; i += gridDim.x * PT) {
        const bool live = i < n;
        const int3 c = live ? flow_cell(g, pos[i]) : make_int3(0, 0, 0);
        const bool gone = live && drained(fs, c);
        const uint32_t ballot = __ballot_sync(0xffffffffu, gone);
        if (ballot && lane == 0) {
            atomicAdd(s.chunk_drained + i / FLOW_CHUNK, (uint32_t)__popc(ballot));
            atomicAdd(s.scalars + 1, (uint32_t)__popc(ballot));
            atomicMin(s.scalars, i + (uint32_t)(__ffs(ballot) - 1));
        }
        if (!live || gone) continue;
        for (int k = 0; k < fs.num_sources; ++k) {
            const FlowBox &b = fs.source[k];
            if (!in_box(b, c)) continue;
            const uint32_t ex = (uint32_t)(b.hi[0] - b.lo[0]), ey = (uint32_t)(b.hi[1] - b.lo[1]);
            const uint32_t local = ((uint32_t)(c.z - b.lo[2]) * ey + (uint32_t)(c.y - b.lo[1])) * ex + (uint32_t)(c.x - b.lo[0]);
            atomicAdd(s.source_count + fs.source_base[k] + local, 1u);
            rx[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][0]);
            ry[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][1]);
            rz[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][2]);
            break;
        }
    }
}

// Stable compaction of the survivors from the first drained index on into the spare arrays.  Chunk c keeps its survivors in order, starting
// at c * FLOW_CHUNK - (drained in the chunks before c); inside a chunk a block-wide ballot scan numbers them.
__global__ void __launch_bounds__(PT) flow_compact_kernel(GridDim g, FlowSet fs, const float4 *__restrict__ pos, const float4 *__restrict__ rx,
                                                          const float4 *__restrict__ ry, const float4 *__restrict__ rz, float4 *__restrict__ pos2,
                                                          float4 *__restrict__ rx2, float4 *__restrict__ ry2, float4 *__restrict__ rz2, FlowScratch s) {
    const uint32_t first = s.scalars[0];
    if (first == NONE) return;
    const uint32_t n = s.scalars[2];
    __shared__ uint32_t warp_total[PT / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (uint32_t c = first / FLOW_CHUNK + blockIdx.x; c < s.num_chunks; c += gridDim.x) {
        const uint32_t base = c * FLOW_CHUNK;
        if (base >= n) break;
        uint32_t out = base - s.chunk_drained[c];
        for (uint32_t r = 0; r < FLOW_CHUNK; r += PT) {
            const uint32_t i = base + r + threadIdx.x;
            const bool keep = i < n && !drained(fs, flow_cell(g, pos[i]));
            const uint32_t ballot = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) warp_total[w] = __popc(ballot);
            __syncthreads();
            uint32_t before = 0, total = 0;
            for (int k = 0; k < PT / 32; ++k) {
                before += k < w ? warp_total[k] : 0u;
                total += warp_total[k];
            }
            const uint32_t dst = out + before + __popc(ballot & ((1u << lane) - 1u));
            if (keep && i >= first) { // survivors before the first drained index stay where they are
                pos2[dst] = pos[i];
                rx2[dst] = rx[i];
                ry2[dst] = ry[i];
                rz2[dst] = rz[i];
            }
            out += total;
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(PT) flow_copy_back_kernel(FlowScratch s, float4 *__restrict__ pos, float4 *__restrict__ rx, float4 *__restrict__ ry,
                                                            float4 *__restrict__ rz, const float4 *__restrict__ pos2, const float4 *__restrict__ rx2,
                                                            const float4 *__restrict__ ry2, const float4 *__restrict__ rz2, uint32_t *schedule_valid) {
    const uint32_t first = s.scalars[0];
    if (first == NONE) return;
    // the survivors moved to lower indices: the scatter schedule no longer describes the order (it stays correct, but its windows miss)
    if (schedule_valid != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *schedule_valid = 0u;
    const uint32_t m = s.scalars[2] - s.scalars[1];
    for (uint32_t i = first + blockIdx.x * PT + threadIdx.x; i < m; i += gridDim.x * PT) {
        pos[i] = pos2[i];
        rx[i] = rx2[i];
        ry[i] = ry2[i];
        rz[i] = rz2[i];
    }
}

__device__ __forceinline__ int source_of(const FlowSet &fs, uint32_t j) {
    int k = 0;
    while (k + 1 < fs.num_sources && j >= fs.source_base[k + 1]) ++k;
    return k;
}
__device__ __forceinline__ int3 source_cell(const FlowSet &fs, int k, uint32_t j) {
    const FlowBox &b = fs.source[k];
    const uint32_t ex = (uint32_t)(b.hi[0] - b.lo[0]), ey = (uint32_t)(b.hi[1] - b.lo[1]), local = j - fs.source_base[k];
    return make_int3(b.lo[0] + (int)(local % ex), b.lo[1] + (int)(local / ex % ey), b.lo[2] + (int)(local / ex / ey));
}

// particles a source cell gets: top up to 8 when it holds fewer than 4, unless it is solid or a border cell
__global__ void __launch_bounds__(PT) flow_need_kernel(GridDim g, FlowSet fs, const uint2 *__restrict__ vox, FlowScratch s) {
    for (uint32_t j = blockIdx.x * PT + threadIdx.x; j < s.source_cells; j += gridDim.x * PT) {
        const int3 c = source_cell(fs, source_of(fs, j), j);
        const bool border = c.x == 0 || c.y == 0 || c.z == 0 || c.x == g.nx - 1 || c.y == g.ny - 1 || c.z == g.nz - 1;
        const bool solid = load_voxel(vox, ((int64_t)c.z * g.ny + c.y) * g.nx + c.x).w != 0.0f;
        const uint32_t count = s.source_count[j];
        s.emit_offsets[j] = count < 4 && !solid && !border ? 8u - count : 0u;
    }
}

__global__ void __launch_bounds__(PT) flow_emit_kernel(GridDim g, StepParams *__restrict__ params, uint32_t capacity, FlowSet fs, float4 *__restrict__ pos,
                                                       float4 *__restrict__ rx, float4 *__restrict__ ry, float4 *__restrict__ rz, FlowScratch s) {
    const uint32_t survivors = s.scalars[2] - s.scalars[1];
    const uint32_t total = s.source_cells ? s.emit_offsets[s.source_cells] : 0u, room = capacity - survivors;
    const uint32_t emitted = total < room ? total : room;
    const uint64_t step = (uint64_t)params->step_count << 32;
    for (uint32_t j = blockIdx.x * PT + threadIdx.x; j < s.source_cells; j += gridDim.x * PT) {
        const uint32_t off = s.emit_offsets[j], need = s.emit_offsets[j + 1] - off;
        if (need == 0) continue;
        const int k = source_of(fs, j);
        const int3 c = source_cell(fs, k, j);
        const float cell[3] = {(float)c.x, (float)c.y, (float)c.z};
        Xoshiro256pp rng(step | (uint64_t)(((int64_t)c.z * g.ny + c.y) * g.nx + c.x));
        const uint32_t count = 8u - need;
        for (uint32_t slot = 0; slot < 8u; ++slot) {
            float p[3];
            const float strat[3] = {(float)(slot % 2u), (float)(slot / 2u % 2u), (float)(slot / 4u % 2u)};
            for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(cell[a], __fadd_rn(__fmul_rn(strat[a], 0.5f), __fmul_rn(rng.next_f32(), 0.5f))); // add_cube
            const uint32_t e = off + slot - count; // this cell's slots count..7 in order
            if (slot < count || e >= emitted) continue;
            const uint32_t i = survivors + e;
            pos[i] = make_float4(p[0], p[1], p[2], __uint_as_float(fs.tag[k])); // the source's tag, as bits
            rx[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][0]);
            ry[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][1]);
            rz[i] = make_float4(0.0f, 0.0f, 0.0f, fs.velocity[k][2]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { // no thread of this kernel reads params->num_particles
        params->num_particles = survivors + emitted;
        s.counters[0] += emitted;
        s.counters[1] += s.scalars[1];
        s.counters[2] += total - emitted;
    }
}

// ---- particle tags ----
__device__ __forceinline__ uint32_t live_count(const StepParams *params, uint32_t n_host) { return params ? params->num_particles : n_host; }

__global__ void __launch_bounds__(PT) paint_tags_kernel(GridDim g, const StepParams *__restrict__ params, uint32_t n_host, FlowBox box, uint32_t tag,
                                                        float4 *__restrict__ pos) {
    const uint32_t n = live_count(params, n_host);
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < n; i += gridDim.x * PT)
        if (in_box(box, flow_cell(g, pos[i]))) pos[i].w = __uint_as_float(tag); // only the fourth word is stored
}

// 2^16 fixed point: the product with a power of two is exact, __float2ll_rn rounds it to nearest even; integer sums do not depend on the order
__device__ __forceinline__ unsigned long long census_fixed(float v) {
    return (unsigned long long)__float2ll_rn(v * (float)(1 << BLUB_TAG_CENSUS_FRAC_BITS));
}

// Per tag in [first, first + num_tags): count, sums of positions and velocities (v_c = row c .w) and the cell bounds.  Each block adds up its
// particles in a private shared-memory table, a warp whose 32 particles share one tag with one table update; then the block flushes its
// non-empty entries with one global atomic per field.
__global__ void __launch_bounds__(PT) tag_census_kernel(GridDim g, const StepParams *__restrict__ params, uint32_t n_host, uint32_t first, uint32_t num_tags,
                                                        const float4 *__restrict__ pos, const float4 *__restrict__ rx, const float4 *__restrict__ ry,
                                                        const float4 *__restrict__ rz, BlubTagCensus *__restrict__ out) {
    __shared__ unsigned long long sum[6][TAG_CENSUS_MAX]; // position x, y, z, velocity x, y, z
    __shared__ int lo[3][TAG_CENSUS_MAX], hi[3][TAG_CENSUS_MAX];
    __shared__ uint32_t count[TAG_CENSUS_MAX];
    for (uint32_t t = threadIdx.x; t < num_tags; t += PT) {
        count[t] = 0u;
        for (int k = 0; k < 6; ++k) sum[k][t] = 0ull;
        for (int k = 0; k < 3; ++k) {
            lo[k][t] = INT_MAX;
            hi[k][t] = INT_MIN;
        }
    }
    __syncthreads();
    const uint32_t n = live_count(params, n_host);
    const int lane = threadIdx.x & 31;
    // whole warps walk the loop, as in flow_count_kernel
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < n; i += gridDim.x * PT) {
        const bool live = i < n;
        const float4 p = live ? pos[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        const uint32_t key = live ? __float_as_uint(p.w) - first : NONE; // tags below `first` wrap to large keys
        const bool in = key < num_tags;
        if (!__any_sync(0xffffffffu, in)) continue;
        const float4 vx = in ? rx[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f), vy = in ? ry[i] : vx, vz = in ? rz[i] : vx;
        const int3 c = flow_cell(g, p);
        unsigned long long q[6] = {census_fixed(p.x), census_fixed(p.y), census_fixed(p.z), census_fixed(vx.w), census_fixed(vy.w), census_fixed(vz.w)};
        int cmin[3] = {c.x, c.y, c.z}, cmax[3] = {c.x, c.y, c.z};
        uint32_t particles = 1u;
        if (__all_sync(0xffffffffu, key == __shfl_sync(0xffffffffu, key, 0))) { // the whole warp has one tag in range
            particles = 32u;
#pragma unroll
            for (int k = 0; k < 6; ++k)
                for (int o = 16; o > 0; o >>= 1) q[k] += __shfl_xor_sync(0xffffffffu, q[k], o);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                cmin[k] = __reduce_min_sync(0xffffffffu, cmin[k]);
                cmax[k] = __reduce_max_sync(0xffffffffu, cmax[k]);
            }
            if (lane != 0) continue;
        } else if (!in) {
            continue;
        }
        atomicAdd(count + key, particles);
#pragma unroll
        for (int k = 0; k < 6; ++k) atomicAdd(&sum[k][key], q[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            atomicMin(&lo[k][key], cmin[k]);
            atomicMax(&hi[k][key], cmax[k]);
        }
    }
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < num_tags; t += PT) {
        if (count[t] == 0u) continue;
        BlubTagCensus &o = out[t];
        atomicAdd(reinterpret_cast<unsigned long long *>(&o.count), (unsigned long long)count[t]);
        for (int k = 0; k < 3; ++k) {
            atomicAdd(reinterpret_cast<unsigned long long *>(&o.position_sum_fx[k]), sum[k][t]);
            atomicAdd(reinterpret_cast<unsigned long long *>(&o.velocity_sum_fx[k]), sum[3 + k][t]);
            atomicMin(&o.cell_min[k], lo[k][t]);
            atomicMax(&o.cell_max[k], hi[k][t]);
        }
    }
}

} // namespace

void launch_flow_prologue(cudaStream_t st, const GridDim &g, StepParams *params, uint32_t capacity, const FlowSet &fs, const FlowScratch &s, float4 *pos,
                          float4 *pos_spare, float4 *const row[3], float4 *const row_spare[3], const uint2 *vox, uint32_t *schedule_valid) {
    const int particle_blocks = std::min(blocks_for(capacity, PT), device_sm_count() * 16); // bounded grid-stride loops over the device count
    BLUB_CUDA_CHECK(cudaMemsetAsync(s.scalars, 0xFF, sizeof(uint32_t), st));
    BLUB_CUDA_CHECK(cudaMemsetAsync(s.scalars + 1, 0, sizeof(uint32_t), st));
    if (fs.num_drains) BLUB_CUDA_CHECK(cudaMemsetAsync(s.chunk_drained, 0, (size_t)s.num_chunks * sizeof(uint32_t), st));
    if (s.source_cells) BLUB_CUDA_CHECK(cudaMemsetAsync(s.source_count, 0, (size_t)s.source_cells * sizeof(uint32_t), st));
    BLUB_LAUNCH(flow_count_kernel, std::max(particle_blocks, 1), PT, 0, st, g, params, fs, pos, row[0], row[1], row[2], s);
    if (fs.num_drains) {
        launch_exclusive_scan(st, s.chunk_drained, s.num_chunks, s.scan_sums);
        BLUB_LAUNCH(flow_compact_kernel, std::max(std::min((int)s.num_chunks, device_sm_count() * 8), 1), PT, 0, st, g, fs, pos, row[0], row[1], row[2],
                    pos_spare, row_spare[0], row_spare[1], row_spare[2], s);
        BLUB_LAUNCH(flow_copy_back_kernel, std::max(particle_blocks, 1), PT, 0, st, s, pos, row[0], row[1], row[2], pos_spare, row_spare[0], row_spare[1],
                    row_spare[2], schedule_valid);
    }
    if (s.source_cells) {
        const int cell_blocks = std::min(blocks_for(s.source_cells, PT), device_sm_count() * 8);
        BLUB_LAUNCH(flow_need_kernel, cell_blocks, PT, 0, st, g, fs, vox, s);
        BLUB_CUDA_CHECK(cudaMemsetAsync(s.emit_offsets + s.source_cells, 0, sizeof(uint32_t), st));
        launch_exclusive_scan(st, s.emit_offsets, (int64_t)s.source_cells + 1, s.scan_sums);
        BLUB_LAUNCH(flow_emit_kernel, cell_blocks, PT, 0, st, g, params, capacity, fs, pos, row[0], row[1], row[2], s);
    } else {
        BLUB_LAUNCH(flow_emit_kernel, 1, PT, 0, st, g, params, capacity, fs, pos, row[0], row[1], row[2], s); // count and counters only
    }
}

void launch_paint_tags(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t n_host, uint32_t np_upper, const FlowBox &box, uint32_t tag,
                       float4 *pos) {
    if (np_upper == 0) return;
    BLUB_LAUNCH(paint_tags_kernel, std::min(blocks_for(np_upper, PT), device_sm_count() * 16), PT, 0, st, g, params, n_host, box, tag, pos);
}

void launch_tag_census(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t n_host, uint32_t np_upper, uint32_t first, uint32_t num_tags,
                       const float4 *pos, float4 *const row[3], BlubTagCensus *out) {
    if (np_upper == 0) return;
    // 8 blocks of 256 threads and 19 KB per SM: every block flushes at most num_tags entries
    BLUB_LAUNCH(tag_census_kernel, std::min(blocks_for(np_upper, PT), device_sm_count() * 8), PT, 0, st, g, params, n_host, first, num_tags, pos, row[0],
                row[1], row[2], out);
}

} // namespace blub
