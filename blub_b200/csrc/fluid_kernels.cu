// fluid_kernels.cu -- grid passes and grid -> particle kernels of the fluid step (sm_90a); the particle -> grid transfers
// live in transfer_kernels.cu, the pressure solve in pcg.cu.
//
// Reference counterparts (relative to the reference's shader/simulation): divergence_compute.comp, divergence_remove.comp,
// extrapolate_velocity.comp, advect_particles.comp, density_projection_{position_change,correct_particles}.comp.
#include <cstdlib>
#include <cstring>

#include "fluid_kernels.hpp"
#include "grid_words.cuh"

namespace blub {
namespace {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
__device__ __forceinline__ float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; }
__device__ __forceinline__ float fractf(float x) { return x - floorf(x); }
__device__ __forceinline__ float signf(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }

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
// cells of a SOLID cell that holds a particle
__global__ void __launch_bounds__(PT) divergence_remove_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ marker,
                                                               const float *__restrict__ p, const uint2 *__restrict__ vox,
                                                               const uint32_t *__restrict__ pw, float *__restrict__ ux, float *__restrict__ uy,
                                                               float *__restrict__ uz) {
    const WordPos wp = word_of_thread(g, b);
    const unsigned todo = wp.inside ? (near_fluid_word(g, b, wp) | (pw != nullptr ? near_stray_word<2>(g, b, pw, wp) : 0u)) : 0u;
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
                    v = u[c][i] - (pc - pn);
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
__device__ __forceinline__ Voxel voxel_point_clamp(const GridDim &g, const uint2 *__restrict__ vox, float px, float py, float pz) {
    // texture(sampler3D(SceneVoxelization, SamplerPointClamp), pos / gridSize): nearest texel, clamp to edge
    const int x = clampi((int)floorf(px), 0, g.nx - 1), y = clampi((int)floorf(py), 0, g.ny - 1), z = clampi((int)floorf(pz), 0, g.nz - 1);
    return load_voxel(vox, lin(g, x, y, z));
}
__device__ __forceinline__ float voxel_w_trilinear(const GridDim &g, const uint2 *__restrict__ vox, float ux, float uy, float uz) {
    const float cx = ux - 0.5f, cy = uy - 0.5f, cz = uz - 0.5f;
    const float fx = floorf(cx), fy = floorf(cy), fz = floorf(cz);
    const float tx = cx - fx, ty = cy - fy, tz = cz - fz;
    const int x0 = clampi((int)fx, 0, g.nx - 1), x1 = clampi((int)fx + 1, 0, g.nx - 1);
    const int y0 = clampi((int)fy, 0, g.ny - 1), y1 = clampi((int)fy + 1, 0, g.ny - 1);
    const int z0 = clampi((int)fz, 0, g.nz - 1), z1 = clampi((int)fz + 1, 0, g.nz - 1);
    const float c00 = mixf(load_voxel(vox, lin(g, x0, y0, z0)).w, load_voxel(vox, lin(g, x1, y0, z0)).w, tx);
    const float c10 = mixf(load_voxel(vox, lin(g, x0, y1, z0)).w, load_voxel(vox, lin(g, x1, y1, z0)).w, tx);
    const float c01 = mixf(load_voxel(vox, lin(g, x0, y0, z1)).w, load_voxel(vox, lin(g, x1, y0, z1)).w, tx);
    const float c11 = mixf(load_voxel(vox, lin(g, x0, y1, z1)).w, load_voxel(vox, lin(g, x1, y1, z1)).w, tx);
    return mixf(mixf(c00, c10, ty), mixf(c01, c11, ty), tz);
}
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

struct Corners {
    float v[8][3]; // corner order 000,100,010,110,001,101,011,111; [..][component]
};
__device__ __forceinline__ void trilerp3(const Corners &c, const float ix[3], const float iy[3], const float iz[3], float out[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { // InterpolateTrilinear, advect_particles.comp:19-23
        const float a = mixf(mixf(c.v[0][k], c.v[1][k], ix[k]), mixf(c.v[2][k], c.v[3][k], ix[k]), iy[k]);
        const float b = mixf(mixf(c.v[4][k], c.v[5][k], ix[k]), mixf(c.v[6][k], c.v[7][k], ix[k]), iy[k]);
        out[k] = mixf(a, b, iz[k]);
    }
}

// advect_particles.comp:35-194.  Writes position + the three APIC rows, marks the new cell FLUID (:175-178); the
// linked-list rebuild of :179-181 has no counterpart (the density pass scatters).
// MIGRATE (z-slab ranks): instead of writing back in place, the kernel itself sorts its results -- stayers are compacted
// into the spare arrays, particles that left the slab go straight to the neighbour (see MigrateOut) -- so that migration
// costs one warp-aggregated atomic per warp instead of an extra pass over all particles.
template <bool MIGRATE>
__device__ __forceinline__ void advect_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params, float4 *__restrict__ pos,
                                                    float4 *__restrict__ rowx, float4 *__restrict__ rowy, float4 *__restrict__ rowz,
                                                    const float *__restrict__ ux, const float *__restrict__ uy,
                                                    const float *__restrict__ uz, const uint2 *__restrict__ vox,
                                                    int8_t *__restrict__ marker, MigrateOut mig) {
    if (i >= params->num_particles) return;
    const float dt = params->dt;
    const float4 p4 = pos[i];
    float x0[3] = {p4.x, p4.y, p4.z};
    const int S[3] = {g.nx, g.ny, g.nz};
    if (vox != nullptr) { // :45-64 particle "eaten" by a moving wall
        const Voxel s = voxel_point_clamp(g, vox, x0[0], x0[1], x0[2]);
        if (s.w > 0.0f) {
            const float ax = fabsf(s.x), ay = fabsf(s.y), az = fabsf(s.z);
            if (ax > ay) {
                if (ax > az) x0[0] += signf(s.x); else x0[2] += signf(s.z);
            } else {
                if (ay > az) x0[1] += signf(s.y); else x0[2] += signf(s.z);
            }
        }
    }
    Corners cn;
    float ix[3], iy[3], iz[3];
    const float *const U[3] = {ux, uy, uz};
#pragma unroll
    for (int c = 0; c < 3; ++c) { // :73-92
        float op[3];
        int lo[3], hi[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            op[k] = fmaxf(0.0f, x0[k] - (k == c ? 1.0f : 0.5f));
            lo[k] = (int)op[k];
            hi[k] = min(lo[k] + 1, S[k] - 1);
            lo[k] = min(lo[k], S[k] - 1); // only reachable for particles outside the domain
        }
        const float *u = U[c];
        cn.v[0][c] = u[lin(g, lo[0], lo[1], lo[2])]; cn.v[1][c] = u[lin(g, hi[0], lo[1], lo[2])];
        cn.v[2][c] = u[lin(g, lo[0], hi[1], lo[2])]; cn.v[3][c] = u[lin(g, hi[0], hi[1], lo[2])];
        cn.v[4][c] = u[lin(g, lo[0], lo[1], hi[2])]; cn.v[5][c] = u[lin(g, hi[0], lo[1], hi[2])];
        cn.v[6][c] = u[lin(g, lo[0], hi[1], hi[2])]; cn.v[7][c] = u[lin(g, hi[0], hi[1], hi[2])];
        ix[c] = fractf(op[0]); iy[c] = fractf(op[1]); iz[c] = fractf(op[2]);
    }
    float nv[3], cx[3], cy[3], cz[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { // :96-112
        const float vx00 = mixf(cn.v[0][k], cn.v[1][k], ix[k]), vx01 = mixf(cn.v[4][k], cn.v[5][k], ix[k]);
        const float vx10 = mixf(cn.v[2][k], cn.v[3][k], ix[k]), vx11 = mixf(cn.v[6][k], cn.v[7][k], ix[k]);
        const float vxy0 = mixf(vx00, vx10, iy[k]), vxy1 = mixf(vx01, vx11, iy[k]);
        nv[k] = mixf(vxy0, vxy1, iz[k]);
        cx[k] = mixf(mixf(cn.v[1][k], cn.v[3][k], iy[k]), mixf(cn.v[5][k], cn.v[7][k], iy[k]), iz[k]) -
                mixf(mixf(cn.v[0][k], cn.v[2][k], iy[k]), mixf(cn.v[4][k], cn.v[6][k], iy[k]), iz[k]);
        cy[k] = mixf(vx10, vx11, iz[k]) - mixf(vx00, vx01, iz[k]);
        cz[k] = vxy1 - vxy0;
    }
    // RK4 confined to the sampled cell, :116-126.  As written (quirk B17): the shader adds the step VECTOR element-wise to vec3s that are
    // indexed by the velocity component, so component k is re-sampled with all three of its interpolants advanced by step[k].
    float k2[3], k3[3], k4[3], ax[3], ay[3], az[3], st[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) st[k] = dt * 0.5f * nv[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ax[k] = saturatef(ix[k] + st[k]); ay[k] = saturatef(iy[k] + st[k]); az[k] = saturatef(iz[k] + st[k]); }
    trilerp3(cn, ax, ay, az, k2);
#pragma unroll
    for (int k = 0; k < 3; ++k) st[k] = dt * 0.5f * k2[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ax[k] = saturatef(ix[k] + st[k]); ay[k] = saturatef(iy[k] + st[k]); az[k] = saturatef(iz[k] + st[k]); }
    trilerp3(cn, ax, ay, az, k3);
#pragma unroll
    for (int k = 0; k < 3; ++k) st[k] = dt * k3[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ax[k] = saturatef(ix[k] + st[k]); ay[k] = saturatef(iy[k] + st[k]); az[k] = saturatef(iz[k] + st[k]); }
    trilerp3(cn, ax, ay, az, k4);
    float mv[3], x1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        mv[k] = dt * (1.0f / 6.0f) * (nv[k] + 2.0f * (k2[k] + k3[k]) + k4[k]);
        x1[k] = x0[k] + mv[k];
    }
    const float lo[3] = {1.001f, 1.001f, (float)g.z_wall_lo + 1.001f};
    const float hi[3] = {(float)g.nx - 1.001f, (float)g.ny - 1.001f, (float)(g.z_wall_hi + 1) - 1.001f};
    bool hit = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) hit = hit || (fminf(fmaxf(x1[k], lo[k]), hi[k]) != x1[k]);
    if (!hit && vox != nullptr) hit = voxel_point_clamp(g, vox, x1[0], x1[1], x1[2]).w > 0.0f;
    if (hit) { // :134-173
        const float len = sqrtf(mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2]) + 1e-10f;
        const float dir[3] = {mv[0] / len, mv[1] / len, mv[2] / len};
        float maxstep = len;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float pc = fractf(x0[k]);
            maxstep = fminf(maxstep, (dir[k] > 0.0f ? pc : 1.0f - pc) / fabsf(dir[k]) - 0.001f);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) mv[k] = dir[k] * maxstep;
        if ((int)x0[0] == (int)x1[0] && (int)x0[1] == (int)x1[1] && (int)x0[2] == (int)x1[2] && vox != nullptr) {
            float push[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float a[3] = {x1[0], x1[1], x1[2]}, b[3] = {x1[0], x1[1], x1[2]};
                a[k] -= 1.0f;
                b[k] += 1.0f;
                push[k] = voxel_w_trilinear(g, vox, a[0], a[1], a[2]) - voxel_w_trilinear(g, vox, b[0], b[1], b[2]);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) mv[k] += push[k] * (dt * 50.0f);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            x1[k] = fminf(fmaxf(x0[k] + mv[k], lo[k]), hi[k]);
            nv[k] = (dir[k] * maxstep) / dt;
        }
    }
    marker[lin(g, clampi((int)x1[0], 0, g.nx - 1), clampi((int)x1[1], 0, g.ny - 1), clampi((int)x1[2], 0, g.nz - 1))] = (int8_t)CELL_FLUID;
    const float4 out_pos = make_float4(x1[0], x1[1], x1[2], p4.w);
    const float4 out_rx = make_float4(cx[0], cx[1], cx[2], nv[0]); // :184-188 (B4: Jacobian columns stored as the rows)
    const float4 out_ry = make_float4(cy[0], cy[1], cy[2], nv[1]);
    const float4 out_rz = make_float4(cz[0], cz[1], cz[2], nv[2]);
    if (!MIGRATE) {
        pos[i] = out_pos;
        rowx[i] = out_rx;
        rowy[i] = out_ry;
        rowz[i] = out_rz;
        return;
    }
    const int dest = (x1[2] < mig.z_lo && mig.peer_down) ? 1 : ((x1[2] >= mig.z_hi && mig.peer_up) ? 2 : 0);
    const unsigned active = __activemask();
    unsigned slot = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) { // one atomic per destination per warp
        const unsigned m = __ballot_sync(active, dest == d);
        if (m == 0u) continue;
        const int leader = __ffs(m) - 1;
        unsigned base = 0;
        if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(mig.counters + d, (unsigned)__popc(m));
        base = __shfl_sync(active, base, leader);
        if (dest == d) slot = base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
    }
    if (dest == 0) {
        mig.pos[slot] = out_pos;
        mig.rx[slot] = out_rx;
        mig.ry[slot] = out_ry;
        mig.rz[slot] = out_rz;
    } else if (slot < mig.capacity) {
        MigrantRecord rec = {out_pos, out_rx, out_ry, out_rz};
        rec.pos.z += dest == 1 ? mig.zshift : -mig.zshift; // re-base into the neighbour's local frame
        (dest == 1 ? mig.peer_down : mig.peer_up)[slot] = rec; // P2P store over NVLink
    } else {
        mig.counters[3] = 1u; // cannot happen with a CFL-limited flow; never overrun the neighbour's buffer
    }
}
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
                              const uint32_t *particle_words, float *const u[3]) {
    BLUB_LAUNCH(divergence_remove_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, p, vox, particle_words, u[0], u[1], u[2]);
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
