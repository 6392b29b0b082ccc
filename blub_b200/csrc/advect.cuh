// advect.cuh -- the per-particle body of stage 7, G2P + advection (advect_particles.comp:35-194): fluid_kernels.cu launches it alone,
// transfer_kernels.cu with the density scatter fused in behind it.
#pragma once
#include "grid_words.cuh"

namespace blub {
namespace {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
__device__ __forceinline__ float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; }
__device__ __forceinline__ float fractf(float x) { return x - floorf(x); }
__device__ __forceinline__ float signf(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }

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

// The MAC trilinear sample of the grid velocity at x0 (advect_particles.comp:73-92): per component c the eight faces around x0 into
// cn.v[..][c] and the interpolants into ix[c], iy[c], iz[c]; trilerp3(cn, ix, iy, iz) is then the velocity there.  Advection and the
// whitewater pass (whitewater_kernels.cu) both sample with it.
__device__ __forceinline__ void mac_corners(const GridDim &g, const float x0[3], const float *const U[3], Corners &cn, float ix[3], float iy[3],
                                            float iz[3]) {
    const int S[3] = {g.nx, g.ny, g.nz};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
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
}

// advect_particles.comp:35-194.  Writes position + the three APIC rows, marks the new cell FLUID (:175-178); the
// linked-list rebuild of :179-181 has no counterpart (the density pass scatters).
// MIGRATE (z-slab ranks): instead of writing back in place, the kernel itself sorts its results -- stayers are compacted
// into the spare arrays, particles that left the slab go straight to the neighbour (see MigrateOut) -- so that migration
// costs one warp-aggregated atomic per warp instead of an extra pass over all particles.
// Returns the new position (tag included) -- for a particle beyond the last one the stand-in (1.5, 1.5, 1.5) the scatters give such lanes.
template <bool MIGRATE>
__device__ __forceinline__ float4 advect_kernel_one(uint32_t i, GridDim g, const StepParams *__restrict__ params, float4 *__restrict__ pos,
                                                    float4 *__restrict__ rowx, float4 *__restrict__ rowy, float4 *__restrict__ rowz,
                                                    const float *__restrict__ ux, const float *__restrict__ uy,
                                                    const float *__restrict__ uz, const uint2 *__restrict__ vox,
                                                    int8_t *__restrict__ marker, MigrateOut mig) {
    if (i >= params->num_particles) return make_float4(1.5f, 1.5f, 1.5f, 0.0f);
    const float dt = params->dt;
    const float4 p4 = pos[i];
    float x0[3] = {p4.x, p4.y, p4.z};
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
    mac_corners(g, x0, U, cn, ix, iy, iz);
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
        return out_pos;
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
    return out_pos;
}
} // namespace
} // namespace blub
