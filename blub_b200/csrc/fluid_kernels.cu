// fluid_kernels.cu -- grid passes and grid -> particle kernels of the fluid step (sm_90a); the particle -> grid transfers
// live in transfer_kernels.cu, the pressure solve in pcg.cu.
//
// Reference counterparts (relative to the reference's shader/simulation): divergence_compute.comp, divergence_remove.comp,
// extrapolate_velocity.comp, advect_particles.comp, density_projection_{position_change,correct_particles}.comp.
#include <cstdlib>
#include <cstring>

#include "fluid_kernels.hpp"
#include "advect.cuh"

namespace blub {
namespace {

// ------------------------------------------------------------------------------------------------ grid passes

// divergence_compute.comp:28-86 (only FLUID cells get a right-hand side; the solver zeroes the rest)
__global__ void __launch_bounds__(PT) divergence_compute_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ marker,
                                                                const float *__restrict__ ux, const float *__restrict__ uy,
                                                                const float *__restrict__ uz, const uint2 *__restrict__ vox,
                                                                float *__restrict__ rhs) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? fbits(g, b, p.xw, p.y, p.z) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z);
        const float px = ux[i], py = uy[i], pz = uz[i];
        const float nx = ux[i - 1], ny = uy[i - g.sy], nz = uz[i - g.sz];
        float d = px - nx;
        d += py - ny;
        d += pz - nz;
        if (marker[i - 1] == CELL_SOLID) d += nx - load_voxel(vox, i - 1).x;
        if (marker[i - g.sy] == CELL_SOLID) d += ny - load_voxel(vox, i - g.sy).y;
        if (marker[i - g.sz] == CELL_SOLID) d += nz - load_voxel(vox, i - g.sz).z;
        if (marker[i + 1] == CELL_SOLID) d -= px - load_voxel(vox, i + 1).x;
        if (marker[i + g.sy] == CELL_SOLID) d -= py - load_voxel(vox, i + g.sy).y;
        if (marker[i + g.sz] == CELL_SOLID) d -= pz - load_voxel(vox, i + g.sz).z;
        rhs[i] = d;
    });
}

// divergence_remove.comp:19-49, on the cells within one cell of the fluid and (pw: particle words, with a solid volume) within two
// cells of a SOLID cell that holds a particle.  bx, by, bz (liquids of different densities; nullptr: constant density): the face
// coefficients, u = u* - beta (p_i - p_j) on the faces with a FLUID side and no SOLID side.
__global__ void __launch_bounds__(PT) divergence_remove_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ marker,
                                                               const float *__restrict__ p, const uint2 *__restrict__ vox,
                                                               const uint32_t *__restrict__ pw, float *__restrict__ ux, float *__restrict__ uy,
                                                               float *__restrict__ uz, const float *__restrict__ bx, const float *__restrict__ by,
                                                               const float *__restrict__ bz) {
    const WordPos wp = word_of_thread(g, b);
    const unsigned todo = wp.inside ? (near_fluid_word(g, b, wp) | (pw != nullptr ? near_stray_word<2>(g, b, pw, wp) : 0u)) : 0u;
    warp_walk(g, todo, wp, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z);
        const int mc = marker[i];
        const float pc = mc == CELL_FLUID ? p[i] : 0.0f;
        float *const u[3] = {ux, uy, uz};
        const float *const beta[3] = {bx, by, bz};
        const int nb[3] = {i + 1, i + g.sy, i + g.sz};
        const bool inb[3] = {x + 1 < g.nx, y + 1 < g.ny, z + 1 < g.nz};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int mn = inb[c] ? marker[nb[c]] : CELL_SOLID;
            float v = 0.0f;
            if (mc == CELL_FLUID || mn == CELL_FLUID) {
                if (mc == CELL_SOLID) {
                    const Voxel s = load_voxel(vox, i);
                    v = c == 0 ? s.x : (c == 1 ? s.y : s.z);
                } else if (mn == CELL_SOLID) {
                    Voxel s = {0, 0, 0, 0};
                    if (inb[c]) s = load_voxel(vox, nb[c]);
                    v = c == 0 ? s.x : (c == 1 ? s.y : s.z);
                } else {
                    const float pn = mn == CELL_FLUID ? p[nb[c]] : 0.0f;
                    if (bx) v = __fsub_rn(u[c][i], __fmul_rn(beta[c][i], __fsub_rn(pc, pn)));
                    else v = u[c][i] - (pc - pn);
                }
            }
            u[c][i] = v;
        }
    });
}

// density_projection_position_change.comp:18-51 (writes the displacement field INTO the velocity volumes), on the cells within one
// cell of the fluid and (pw: particle words, with a solid volume) within one cell of a SOLID cell that holds a particle
__global__ void __launch_bounds__(PT) position_change_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params,
                                                             const int8_t *__restrict__ marker, const float *__restrict__ p,
                                                             const uint32_t *__restrict__ pw, float *__restrict__ ux, float *__restrict__ uy,
                                                             float *__restrict__ uz) {
    const WordPos wp = word_of_thread(g, b);
    const unsigned todo = wp.inside ? (near_fluid_word(g, b, wp) | (pw != nullptr ? near_stray_word<1>(g, b, pw, wp) : 0u)) : 0u;
    const float dt = params->dt;
    warp_walk(g, todo, wp, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z);
        const int mc = marker[i];
        const float pc = mc == CELL_FLUID ? p[i] : 0.0f;
        float *const u[3] = {ux, uy, uz};
        const int nb[3] = {i + 1, i + g.sy, i + g.sz};
        const bool inb[3] = {x + 1 < g.nx, y + 1 < g.ny, z + 1 < g.nz};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int mn = inb[c] ? marker[nb[c]] : CELL_SOLID;
            const float pn = mn == CELL_FLUID ? p[nb[c]] : 0.0f;
            float d = (pn - pc) * dt;
            if (mc == CELL_SOLID || mn == CELL_SOLID) d = 0.0f;
            u[c][i] = d;
        }
    });
}

// extrapolate_velocity.comp:26-90.  In place: only invalid faces are written, only valid faces are read.
// A face of component c is VALID when its cell or the cell's +c neighbour is FLUID (:5-10); an invalid face takes the average of
// the valid ones among its 8 in-plane neighbours (:26-90, first in-plane axis fastest, as in the shader's contribution lists).
// The owner thread of a word forms the validity words of the 3 x 3 in-plane neighbourhood with shifts and ORs and from them the mask
// of cells that get a value; the warp then walks those words, every lane testing its own bit of the eight neighbour words (handed over
// by shuffles).  Same neighbours, same order, same arithmetic as a per-cell pass over the marker volume.
// validity word of component c for the word (xw, y, z): bit k = the face of cell 32 xw + k is valid
__device__ __forceinline__ unsigned valid_word(const GridDim &g, const FluidBits &b, int c, int xw, int y, int z) {
    const unsigned f = fbits(g, b, xw, y, z);
    if (c == 0) return f | (f >> 1) | (fbits(g, b, xw + 1, y, z) << 31);
    if (c == 1) return f | fbits(g, b, xw, y + 1, z);
    return f | fbits(g, b, xw, y, z + 1);
}
template <int C>
__device__ __forceinline__ void extrapolate_component(const GridDim &g, const FluidBits &b, const WordPos &p, bool near, float *__restrict__ u) {
    // nb[ob + 1][oa + 1]: validity of the in-plane neighbour (oa along the first in-plane axis, ob along the second), as a word aligned
    // with this thread's cells
    unsigned nb[3][3];
#pragma unroll
    for (int ob = 0; ob < 3; ++ob)
#pragma unroll
        for (int oa = 0; oa < 3; ++oa) nb[ob][oa] = 0u;
    if (near) {
        if (C == 0) { // in-plane axes y (fast), z
#pragma unroll
            for (int ob = -1; ob <= 1; ++ob)
#pragma unroll
                for (int oa = -1; oa <= 1; ++oa) nb[ob + 1][oa + 1] = valid_word(g, b, 0, p.xw, p.y + oa, p.z + ob);
        } else {      // in-plane axes x (fast) and z (C == 1) or y (C == 2)
#pragma unroll
            for (int ob = -1; ob <= 1; ++ob) {
                const int yy = C == 1 ? p.y : p.y + ob, zz = C == 1 ? p.z + ob : p.z;
                const unsigned m = valid_word(g, b, C, p.xw, yy, zz), l = valid_word(g, b, C, p.xw - 1, yy, zz), r = valid_word(g, b, C, p.xw + 1, yy, zz);
                nb[ob + 1][0] = (m << 1) | (l >> 31); // neighbour x - 1
                nb[ob + 1][1] = m;
                nb[ob + 1][2] = (m >> 1) | (r << 31); // neighbour x + 1
            }
        }
    }
    unsigned any = 0;
#pragma unroll
    for (int ob = 0; ob < 3; ++ob)
#pragma unroll
        for (int oa = 0; oa < 3; ++oa)
            if (oa != 1 || ob != 1) any |= nb[ob][oa];
    // non-FLUID cells whose face is invalid and has a valid neighbour (a FLUID cell's own faces are valid: ~own covers ~fluid)
    const unsigned todo = cells_mask(p) & ~nb[1][1] & any;
    const int sa = C == 0 ? g.sy : 1, sb = C == 2 ? g.sy : g.sz;
    const int lane = threadIdx.x & 31;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int src) {
        unsigned nbw[3][3]; // the owner's neighbour words (shuffles: every lane takes part)
#pragma unroll
        for (int ob = 0; ob < 3; ++ob)
#pragma unroll
            for (int oa = 0; oa < 3; ++oa) nbw[ob][oa] = (oa != 1 || ob != 1) ? __shfl_sync(0xffffffffu, nb[ob][oa], src) : 0u;
        if (!on) return;
        const int i = lin(g, x, y, z);
        float numv = 0.0f, avg = 0.0f;
#pragma unroll
        for (int ob = -1; ob <= 1; ++ob)
#pragma unroll
            for (int oa = -1; oa <= 1; ++oa) {
                if (oa == 0 && ob == 0) continue;
                if ((nbw[ob + 1][oa + 1] >> lane) & 1u) {
                    numv += 1.0f;
                    avg += u[i + oa * sa + ob * sb];
                }
            }
        u[i] = avg / numv; // numv > 0: the cell is in `any`
    });
}
__global__ void __launch_bounds__(PT) extrapolate_kernel(GridDim g, FluidBits b, float *__restrict__ ux, float *__restrict__ uy, float *__restrict__ uz) {
    const WordPos p = word_of_thread(g, b);
    // nothing to do unless a FLUID cell lies within one cell of one of this word's cells
    const bool near = p.inside && near_fluid_word(g, b, p) != 0u;
    if (!__any_sync(0xffffffffu, near)) return;
    extrapolate_component<0>(g, b, p, near, ux);
    extrapolate_component<1>(g, b, p, near, uy);
    extrapolate_component<2>(g, b, p, near, uz);
}

// ------------------------------------------------------------------------------------------------ G2P + advection
__device__ __forceinline__ float grid_trilinear_clamp(const GridDim &g, const float *__restrict__ vol, float ux, float uy, float uz) {
    const float cx = ux - 0.5f, cy = uy - 0.5f, cz = uz - 0.5f;
    const float fx = floorf(cx), fy = floorf(cy), fz = floorf(cz);
    const float tx = cx - fx, ty = cy - fy, tz = cz - fz;
    const int x0 = clampi((int)fx, 0, g.nx - 1), x1 = clampi((int)fx + 1, 0, g.nx - 1);
    const int y0 = clampi((int)fy, 0, g.ny - 1), y1 = clampi((int)fy + 1, 0, g.ny - 1);
    const int z0 = clampi((int)fz, 0, g.nz - 1), z1 = clampi((int)fz + 1, 0, g.nz - 1);
    const float c00 = mixf(vol[lin(g, x0, y0, z0)], vol[lin(g, x1, y0, z0)], tx);
    const float c10 = mixf(vol[lin(g, x0, y1, z0)], vol[lin(g, x1, y1, z0)], tx);
    const float c01 = mixf(vol[lin(g, x0, y0, z1)], vol[lin(g, x1, y0, z1)], tx);
    const float c11 = mixf(vol[lin(g, x0, y1, z1)], vol[lin(g, x1, y1, z1)], tx);
    return mixf(mixf(c00, c10, ty), mixf(c01, c11, ty), tz);
}

// the per-particle body, advect_kernel_one, is in advect.cuh
template <bool MIGRATE>
__global__ void __launch_bounds__(PT) advect_kernel(GridDim g, const StepParams *__restrict__ params, float4 *__restrict__ pos,
                                                    float4 *__restrict__ rowx, float4 *__restrict__ rowy, float4 *__restrict__ rowz,
                                                    const float *__restrict__ ux, const float *__restrict__ uy,
                                                    const float *__restrict__ uz, const uint2 *__restrict__ vox,
                                                    int8_t *__restrict__ marker, MigrateOut mig) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < np_; i += gridDim.x * PT) advect_kernel_one<MIGRATE>(i, g, params, pos, rowx, rowy, rowz, ux, uy, uz, vox, marker, mig);
}

// ------------------------------------------------------------------------------------------------ density projection
// density_projection_correct_particles.comp:25-73 (fp32 software trilinear instead of the 8-bit hardware filter, SURVEY B5)
__device__ __forceinline__ void correct_particles_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params,
                                                               float4 *__restrict__ pos, const int8_t *__restrict__ marker,
                                                               const float *__restrict__ ux, const float *__restrict__ uy,
                                                               const float *__restrict__ uz) {
    if (i >= params->num_particles) return;
    const float4 p4 = pos[i];
    const float x0[3] = {p4.x, p4.y, p4.z};
    float ch[3];
    ch[0] = grid_trilinear_clamp(g, ux, fmaxf(0.0f, x0[0] - 0.5f), fmaxf(0.0f, x0[1]), fmaxf(0.0f, x0[2]));
    ch[1] = grid_trilinear_clamp(g, uy, fmaxf(0.0f, x0[0]), fmaxf(0.0f, x0[1] - 0.5f), fmaxf(0.0f, x0[2]));
    ch[2] = grid_trilinear_clamp(g, uz, fmaxf(0.0f, x0[0]), fmaxf(0.0f, x0[1]), fmaxf(0.0f, x0[2] - 0.5f));
    float x1[3] = {x0[0] + ch[0], x0[1] + ch[1], x0[2] + ch[2]};
    const float lo[3] = {1.001f, 1.001f, (float)g.z_wall_lo + 1.001f};
    const float hi[3] = {(float)g.nx - 1.001f, (float)g.ny - 1.001f, (float)(g.z_wall_hi + 1) - 1.001f};
    bool hit = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) hit = hit || (fminf(fmaxf(x1[k], lo[k]), hi[k]) != x1[k]);
    if (!hit) {
        const int x = clampi((int)floorf(x1[0]), 0, g.nx - 1), y = clampi((int)floorf(x1[1]), 0, g.ny - 1), z = clampi((int)floorf(x1[2]), 0, g.nz - 1);
        hit = marker[lin(g, x, y, z)] == CELL_SOLID;
    }
    if (hit) {
        const float len = sqrtf(ch[0] * ch[0] + ch[1] * ch[1] + ch[2] * ch[2]) + 1e-10f;
        const float dir[3] = {ch[0] / len, ch[1] / len, ch[2] / len};
        float maxstep = len;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float pc = fractf(x0[k]);
            maxstep = fminf(maxstep, (dir[k] > 0.0f ? pc : 1.0f - pc) / fabsf(dir[k]) - 0.001f);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) x1[k] = fminf(fmaxf(x0[k] + dir[k] * maxstep, lo[k]), hi[k]);
    }
    x1[2] = fminf(fmaxf(x1[2], g.z_keep_lo), g.z_keep_hi); // slab ranks only (no-op on one GPU)
    pos[i] = make_float4(x1[0], x1[1], x1[2], p4.w);
}
__global__ void __launch_bounds__(PT) correct_particles_kernel(GridDim g, const StepParams *__restrict__ params,
                                                               float4 *__restrict__ pos, const int8_t *__restrict__ marker,
                                                               const float *__restrict__ ux, const float *__restrict__ uy,
                                                               const float *__restrict__ uz) {
    // a bounded grid strides over the particles: launch cost does not grow with the CAPACITY a z-slab rank sizes its launches by
    const uint32_t np_ = params->num_particles;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; (i & ~31u) < np_; i += gridDim.x * PT) correct_particles_kernel_one(i, g, params, pos, marker, ux, uy, uz);
}

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }
// particle kernels: at most 128 blocks per SM (small enough for a negligible tail, few enough to launch quickly), a grid-stride loop over the rest
inline int particle_blocks(uint32_t np_upper) { return min(blocks_for(np_upper, PT), device_sm_count() * 128); }

} // namespace

// ------------------------------------------------------------------------------------------------ launchers
static int word_blocks(const GridDim &g, const FluidBits &bits) { return blocks_for((int64_t)bits.wpr * g.ny * g.nz, PT); }

void launch_divergence_compute(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, float *const u[3], const uint2 *vox, float *rhs) {
    BLUB_LAUNCH(divergence_compute_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, u[0], u[1], u[2], vox, rhs);
}

void launch_divergence_remove(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const float *p, const uint2 *vox,
                              const uint32_t *particle_words, float *const u[3], const float *const *beta) {
    BLUB_LAUNCH(divergence_remove_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, p, vox, particle_words, u[0], u[1], u[2],
                beta ? beta[0] : nullptr, beta ? beta[1] : nullptr, beta ? beta[2] : nullptr);
}

void launch_extrapolate(cudaStream_t st, const GridDim &g, const FluidBits &bits, float *const u[3]) {
    BLUB_LAUNCH(extrapolate_kernel, word_blocks(g, bits), PT, 0, st, g, bits, u[0], u[1], u[2]);
}

void launch_clear_marker(cudaStream_t st, const GridDim &g, int8_t *marker) {
    BLUB_CUDA_CHECK(cudaMemsetAsync(marker, 0xFF, (size_t)g.n, st));
}

void launch_advect(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                   float *const u[3], const uint2 *vox, int8_t *marker) {
    if (np_upper == 0) return;
    BLUB_LAUNCH(advect_kernel<false>, particle_blocks(np_upper), PT, 0, st, g, params, pos, row[0], row[1], row[2], u[0], u[1], u[2], vox, marker, MigrateOut{});
}

void launch_advect_migrate(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                           float *const u[3], const uint2 *vox, int8_t *marker, const MigrateOut &mig) {
    if (np_upper == 0) return;
    BLUB_LAUNCH(advect_kernel<true>, particle_blocks(np_upper), PT, 0, st, g, params, pos, row[0], row[1], row[2], u[0], u[1], u[2], vox, marker, mig);
}

void launch_position_change(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker, const float *p,
                            const uint32_t *particle_words, float *const u[3]) {
    BLUB_LAUNCH(position_change_kernel, word_blocks(g, bits), PT, 0, st, g, bits, params, marker, p, particle_words, u[0], u[1], u[2]);
}

void launch_correct_particles(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos,
                              const int8_t *marker, float *const u[3]) {
    if (np_upper == 0) return;
    BLUB_LAUNCH(correct_particles_kernel, particle_blocks(np_upper), PT, 0, st, g, params, pos, marker, u[0], u[1], u[2]);
}

} // namespace blub
