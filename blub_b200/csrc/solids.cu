// solids.cu -- analytic rigid solids written straight into the RGBA16F solid-voxel volume (SURVEY.md section 8 f1).
//
// The reference voxelizes triangle meshes with a conservative-rasterization render pass every step
// (src/scene/voxelization.rs:118-157, shader/voxelize/conservative_hull.{vert,frag}); its meshes are git-LFS stubs in this
// checkout, and a raster pipeline has no CUDA counterpart on this path.  What the fluid step consumes is only the volume:
// xyz = solid velocity in cells/s, w = 1 inside solids.  This file produces that volume for oriented boxes (and spheres) driven
// by the reference's own rigid animation maths:
//   position   StaticMeshData::world_position_at_time  (src/scene/models.rs:154-171: ping-pong translation, Linear / SmoothStep)
//   velocity   finite difference over one simulation step (models.rs:186-191)
//   rotation   static Euler angles * axis-angle(deg_per_sec * t) (models.rs:173-184), angular velocity axis scaled in rad/s
//   voxel velocity  ComputeVoxelSpeed: cross(a, p - dot(p, a) a) + v with p = voxelPos - centre (conservative_hull.frag:17-23;
//              as written the axis `a` carries the angular speed, so the projection term is a*|a|^2-scaled -- replicated)
// Deviation (documented): the whole interior is marked, the reference marks the hull only.
#include <cmath>

#include "../../include/blub_fluid.h"
#include "blub_core.hpp"

namespace blub {
namespace {

struct Quat {
    float s, x, y, z;
};
inline Quat qmul(const Quat &a, const Quat &b) {
    return {a.s * b.s - a.x * b.x - a.y * b.y - a.z * b.z, a.s * b.x + a.x * b.s + a.y * b.z - a.z * b.y,
            a.s * b.y - a.x * b.z + a.y * b.s + a.z * b.x, a.s * b.z + a.x * b.y - a.y * b.x + a.z * b.s};
}
// cgmath 0.18 `Quaternion::from(Euler { x, y, z })` (third-party, not vendored; restated from its published source)
inline Quat quat_from_euler_deg(const float deg[3]) {
    const float h = 0.5f * 3.14159265358979323846f / 180.0f;
    const float sx = std::sin(deg[0] * h), cx = std::cos(deg[0] * h), sy = std::sin(deg[1] * h), cy = std::cos(deg[1] * h), sz = std::sin(deg[2] * h),
                cz = std::cos(deg[2] * h);
    return {-sx * sy * sz + cx * cy * cz, sx * cy * cz + sy * sz * cx, -sx * sz * cy + sy * cx * cz, sx * sy * cz + sz * cx * cy};
}
inline Quat quat_axis_angle(const float axis[3], float rad) {
    const float n = std::sqrt(axis[0] * axis[0] + axis[1] * axis[1] + axis[2] * axis[2]);
    const float s = std::sin(0.5f * rad) / (n > 0.0f ? n : 1.0f);
    return {std::cos(0.5f * rad), axis[0] * s, axis[1] * s, axis[2] * s};
}

// models.rs:154-171
void world_position_at_time(const BlubRigidObject &o, float t, float out[3]) {
    if (!o.has_translation) {
        for (int k = 0; k < 3; ++k) out[k] = o.world_position[k];
        return;
    }
    float progress = std::fmod(t, o.translation_duration * 2.0f);
    if (progress > o.translation_duration) progress = o.translation_duration * 2.0f - progress;
    progress /= o.translation_duration;
    progress = progress < 0.0f ? 0.0f : (progress > 1.0f ? 1.0f : progress);
    if (o.translation_curve == 1) progress = progress * progress * (3.0f - 2.0f * progress); // SmoothStep
    for (int k = 0; k < 3; ++k) out[k] = o.world_position[k] * (1.0f - progress) + o.translation_target[k] * progress;
}

struct BoxParams {
    float centre[3];   // voxel space
    float half[3];     // voxel space half extents (sphere: half[0] = radius)
    float rot[9];      // world->local rotation (row major): local = R^T (p - centre)
    float velocity[3]; // cells / s
    float axis[3];     // rotation axis scaled by rad / s
    int sphere;
};

__global__ void __launch_bounds__(256) voxelize_box_kernel(uint2 *__restrict__ vox, int nx, int ny, int nz, BoxParams b, int clear_first) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)nx * ny * nz) return;
    const int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((int64_t)nx * ny));
    // inside test at the voxel centre
    const float d[3] = {(float)x + 0.5f - b.centre[0], (float)y + 0.5f - b.centre[1], (float)z + 0.5f - b.centre[2]};
    bool inside;
    if (b.sphere) {
        inside = d[0] * d[0] + d[1] * d[1] + d[2] * d[2] <= b.half[0] * b.half[0];
    } else {
        const float lx = b.rot[0] * d[0] + b.rot[3] * d[1] + b.rot[6] * d[2];
        const float ly = b.rot[1] * d[0] + b.rot[4] * d[1] + b.rot[7] * d[2];
        const float lz = b.rot[2] * d[0] + b.rot[5] * d[1] + b.rot[8] * d[2];
        inside = fabsf(lx) <= b.half[0] && fabsf(ly) <= b.half[1] && fabsf(lz) <= b.half[2];
    }
    if (!inside) {
        if (clear_first) vox[i] = make_uint2(0u, 0u);
        return;
    }
    // ComputeVoxelSpeed at the integer voxel position (conservative_hull.frag:17-23,34-35)
    const float p[3] = {(float)x - b.centre[0], (float)y - b.centre[1], (float)z - b.centre[2]};
    const float pa = p[0] * b.axis[0] + p[1] * b.axis[1] + p[2] * b.axis[2];
    const float q[3] = {p[0] - pa * b.axis[0], p[1] - pa * b.axis[1], p[2] - pa * b.axis[2]};
    const float vx = b.axis[1] * q[2] - b.axis[2] * q[1] + b.velocity[0];
    const float vy = b.axis[2] * q[0] - b.axis[0] * q[2] + b.velocity[1];
    const float vz = b.axis[0] * q[1] - b.axis[1] * q[0] + b.velocity[2];
    __half2 lo = __floats2half2_rn(vx, vy), hi = __floats2half2_rn(vz, 1.0f);
    vox[i] = make_uint2(*reinterpret_cast<unsigned *>(&lo), *reinterpret_cast<unsigned *>(&hi));
}

} // namespace

void quat_from_euler_deg_wxyz(const float deg[3], float q[4]) {
    const Quat r = quat_from_euler_deg(deg);
    q[0] = r.s;
    q[1] = r.x;
    q[2] = r.y;
    q[3] = r.z;
}

// StaticMeshData::to_gpu (src/scene/models.rs:186-224) evaluated on the host: where the object is, how it is rotated and how it moves,
// in voxel space.  Shared by the analytic solids below and the mesh voxelizer (mesh_voxelizer.cu).
void rigid_state_at(const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3], double total_time, double delta,
                    BlubRigidState &out) {
    const float t = (float)total_time, dt = (float)delta;
    float pos[3], prev[3], vel[3] = {0, 0, 0};
    world_position_at_time(o, t, pos);
    if (total_time > delta) { // models.rs:186-191
        world_position_at_time(o, t - dt, prev);
        for (int k = 0; k < 3; ++k) vel[k] = (pos[k] - prev[k]) / dt;
    }
    Quat q = quat_from_euler_deg(o.rotation_angles_deg);
    float axis_scaled[3] = {0, 0, 0};
    if (o.has_rotation) {
        const float rad_per_s = o.rotation_deg_per_sec * 3.14159265358979323846f / 180.0f;
        q = qmul(q, quat_axis_angle(o.rotation_axis, rad_per_s * t));
        const float n = std::sqrt(o.rotation_axis[0] * o.rotation_axis[0] + o.rotation_axis[1] * o.rotation_axis[1] + o.rotation_axis[2] * o.rotation_axis[2]);
        for (int k = 0; k < 3; ++k) axis_scaled[k] = o.rotation_axis[k] / (n > 0.0f ? n : 1.0f) * rad_per_s;
    }
    // local -> world rotation matrix from the quaternion (columns = rotated basis vectors)
    const float R[9] = {1 - 2 * (q.y * q.y + q.z * q.z), 2 * (q.x * q.y - q.z * q.s),     2 * (q.x * q.z + q.y * q.s),
                        2 * (q.x * q.y + q.z * q.s),     1 - 2 * (q.x * q.x + q.z * q.z), 2 * (q.y * q.z - q.x * q.s),
                        2 * (q.x * q.z - q.y * q.s),     2 * (q.y * q.z + q.x * q.s),     1 - 2 * (q.x * q.x + q.y * q.y)};
    for (int k = 0; k < 9; ++k) out.rotation[k] = R[k];
    for (int k = 0; k < 3; ++k) {
        out.centre_voxel[k] = (pos[k] - fluid_world_position[k]) / grid_to_world_scale; // transform_voxel, models.rs:196-198
        out.velocity_voxel[k] = vel[k] / grid_to_world_scale;                           // fluid_space_velocity, :206
        out.axis_scaled[k] = axis_scaled[k];                                            // fluid_space_rotation_axis_scaled, :207-216
    }
}

// analytic box / sphere: evaluates the animation and enqueues one kernel
void voxelize_rigid_solid(void *rgba16f, const uint32_t dim[3], const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3],
                          double total_time, double delta, int clear_first, cudaStream_t stream, BlubRigidState *state_out) {
    BlubRigidState st;
    rigid_state_at(o, grid_to_world_scale, fluid_world_position, total_time, delta, st);
    if (state_out) *state_out = st;
    BoxParams b;
    for (int k = 0; k < 9; ++k) b.rot[k] = st.rotation[k];
    for (int k = 0; k < 3; ++k) {
        b.centre[k] = st.centre_voxel[k];
        b.half[k] = o.half_extent[k] * o.scale / grid_to_world_scale;
        b.velocity[k] = st.velocity_voxel[k];
        b.axis[k] = st.axis_scaled[k];
    }
    b.sphere = o.shape == 1;
    const int64_t n = (int64_t)dim[0] * dim[1] * dim[2];
    BLUB_LAUNCH(voxelize_box_kernel, (int)((n + 255) / 256), 256, 0, stream, static_cast<uint2 *>(rgba16f), (int)dim[0], (int)dim[1], (int)dim[2], b, clear_first);
}

} // namespace blub
