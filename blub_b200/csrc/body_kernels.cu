// body_kernels.cu -- floating bodies (DESIGN.md §8 "Floating bodies").  Not in the reference.
//
// Stage 0 writes every body into the fluid's composite solid volume (a copy of the borrowed one); the end of stage 2 sums the projection
// pressure on each body's wetted faces with the probes' face rule (solid_faces.cuh) and one warp integrates the bodies.  Every float operation
// of the cell rule, the voxel velocity and the integrator is an explicit round-to-nearest intrinsic, so that tests/body_ref.py restates them
// bit for bit in NumPy; the sums are int64 fixed point and do not depend on the launch order.
#include <algorithm>
#include <cmath>

#include "fluid_kernels.hpp"
#include "solid_faces.cuh"

namespace blub {

namespace {

constexpr int PT = 256;

inline int blocks_for(int64_t n, int per_block) { return (int)((n + per_block - 1) / per_block); }

// R (row major, body -> grid) of the unit quaternion q = (w, x, y, z)
__device__ __forceinline__ void rotation_of(const float q[4], float R[9]) {
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z), xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
    const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
    R[0] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(yy, zz)));
    R[1] = __fmul_rn(2.0f, __fsub_rn(xy, wz));
    R[2] = __fmul_rn(2.0f, __fadd_rn(xz, wy));
    R[3] = __fmul_rn(2.0f, __fadd_rn(xy, wz));
    R[4] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, zz)));
    R[5] = __fmul_rn(2.0f, __fsub_rn(yz, wx));
    R[6] = __fmul_rn(2.0f, __fsub_rn(xz, wy));
    R[7] = __fmul_rn(2.0f, __fadd_rn(yz, wx));
    R[8] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, yy)));
}

// ((a0 b0 + a1 b1) + a2 b2)
__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// Half extents of the grid-axis bounding box: sum_j |R_kj| h_j for a box, r for a sphere.
__device__ __forceinline__ void bounding_extents(const BlubBody &b, const float R[9], float e[3]) {
    for (int k = 0; k < 3; ++k)
        e[k] = b.shape == 1 ? b.half_extent[0]
                            : dot3(fabsf(R[3 * k]), fabsf(R[3 * k + 1]), fabsf(R[3 * k + 2]), b.half_extent[0], b.half_extent[1], b.half_extent[2]);
}

// The cell rule: the cell centre (index + 0.5) lies inside the body.  d = centre - c on return.
__device__ __forceinline__ bool covers(const BlubBody &b, const float R[9], int x, int y, int z, float d[3]) {
    d[0] = __fsub_rn((float)x + 0.5f, b.centre[0]);
    d[1] = __fsub_rn((float)y + 0.5f, b.centre[1]);
    d[2] = __fsub_rn((float)z + 0.5f, b.centre[2]);
    if (b.shape == 1) return dot3(d[0], d[1], d[2], d[0], d[1], d[2]) <= __fmul_rn(b.half_extent[0], b.half_extent[0]);
    for (int j = 0; j < 3; ++j) // body coordinate j = (R^T d)_j
        if (!(fabsf(dot3(R[j], R[3 + j], R[6 + j], d[0], d[1], d[2])) <= b.half_extent[j])) return false;
    return true;
}

// The first cell of the launch cube of body b: floor(c - e), at least 0.
__device__ __forceinline__ void cube_origin(const BlubBody &b, const float R[9], int lo[3]) {
    float e[3];
    bounding_extents(b, R, e);
    for (int k = 0; k < 3; ++k) lo[k] = max(0, (int)floorf(__fsub_rn(b.centre[k], e[k])));
}

// blockIdx.y = body; the blocks of x stride over its cube.  A covered cell that no later body covers gets w = 1 and the rigid velocity
// v + w x (centre - c): later bodies win, whatever order the blocks run in.
__global__ void __launch_bounds__(PT) body_composite_kernel(GridDim g, int num_bodies, uint32_t cube, const BlubBody *__restrict__ bodies,
                                                            uint2 *__restrict__ vox) {
    const int bi = blockIdx.y;
    const BlubBody b = bodies[bi];
    float R[9];
    rotation_of(b.rotation, R);
    int lo[3];
    cube_origin(b, R, lo);
    const uint32_t cells = cube * cube * cube;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < cells; i += gridDim.x * PT) {
        const int x = lo[0] + (int)(i % cube), y = lo[1] + (int)(i / cube % cube), z = lo[2] + (int)(i / (cube * cube));
        if (x >= g.nx || y >= g.ny || z >= g.nz) continue;
        float d[3];
        if (!covers(b, R, x, y, z, d)) continue;
        bool later = false;
        for (int k = bi + 1; k < num_bodies && !later; ++k) {
            const BlubBody o = bodies[k];
            float Ro[9], dd[3];
            rotation_of(o.rotation, Ro);
            later = covers(o, Ro, x, y, z, dd);
        }
        if (later) continue;
        const float *v = b.velocity, *w = b.angular_velocity;
        const float vx = __fadd_rn(v[0], __fsub_rn(__fmul_rn(w[1], d[2]), __fmul_rn(w[2], d[1])));
        const float vy = __fadd_rn(v[1], __fsub_rn(__fmul_rn(w[2], d[0]), __fmul_rn(w[0], d[2])));
        const float vz = __fadd_rn(v[2], __fsub_rn(__fmul_rn(w[0], d[1]), __fmul_rn(w[1], d[0])));
        __half2 h0 = __floats2half2_rn(vx, vy), h1 = __floats2half2_rn(vz, 1.0f);
        vox[(int64_t)x + (int64_t)y * g.sy + (int64_t)z * g.sz] = make_uint2(*reinterpret_cast<unsigned *>(&h0), *reinterpret_cast<unsigned *>(&h1));
    }
}

// blockIdx.y = body; the blocks of x stride over its cube.  Every SOLID cell the body covers adds its wetted faces with the pivot at the
// centre; the block issues one atomic per non-zero field into sums[8 * body + field].
__global__ void __launch_bounds__(PT) body_load_kernel(GridDim g, const StepParams *__restrict__ params, uint32_t cube, const BlubBody *__restrict__ bodies,
                                                       const int8_t *__restrict__ marker, const float *__restrict__ p_vel,
                                                       unsigned long long *__restrict__ sums) {
    __shared__ unsigned long long part[PT / 32][LOAD_FIELDS];
    const BlubBody b = bodies[blockIdx.y];
    float R[9];
    rotation_of(b.rotation, R);
    int lo[3];
    cube_origin(b, R, lo);
    const float inv_dt = params->inv_dt;
    long long acc[6] = {0, 0, 0, 0, 0, 0};
    unsigned long long faces = 0;
    const uint32_t cells = cube * cube * cube;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < cells; i += gridDim.x * PT) {
        const int c[3] = {lo[0] + (int)(i % cube), lo[1] + (int)(i / cube % cube), lo[2] + (int)(i / (cube * cube))};
        if (c[0] >= g.nx || c[1] >= g.ny || c[2] >= g.nz) continue;
        const int64_t s = (int64_t)c[0] + (int64_t)c[1] * g.sy + (int64_t)c[2] * g.sz;
        float d[3];
        if (marker[s] != CELL_SOLID || !covers(b, R, c[0], c[1], c[2], d)) continue;
        faces += add_wetted_faces(g, marker, p_vel, inv_dt, c, s, b.centre, acc);
    }
    const unsigned long long sum = block_load_sum<PT>(acc, faces, part);
    if (sum != 0) atomicAdd(&sums[8 * blockIdx.y + threadIdx.x], sum);
}

// One warp, lane = body: semi-implicit Euler in float32 with the tank clamp, then the record.  Reads and re-zeroes the body's sums.
__global__ void body_integrate_kernel(GridDim g, const StepParams *__restrict__ params, int num_bodies, BlubBody *__restrict__ bodies,
                                      unsigned long long *__restrict__ sums, BlubBodyRecord *__restrict__ ring) {
    const int bi = threadIdx.x;
    if (bi >= num_bodies) return;
    BlubBody b = bodies[bi];
    unsigned long long *s = sums + 8 * bi;
    float F[3], tau[3];
    for (int k = 0; k < 3; ++k) {
        // exact power-of-two scalings of the int64 sums
        F[k] = __fmul_rn(__ll2float_rn((long long)s[k]), 1.0f / (float)(1 << BLUB_LOAD_FORCE_FRAC_BITS));
        tau[k] = __fmul_rn(__ll2float_rn((long long)s[3 + k]), 1.0f / (float)(1 << BLUB_LOAD_TORQUE_FRAC_BITS));
    }
    BlubBodyRecord rec;
    rec.step = params->step_count;
    rec.wetted_faces = (uint32_t)s[6];
    for (int k = 0; k < 3; ++k) {
        rec.force_fx[k] = (long long)s[k];
        rec.torque_fx[k] = (long long)s[3 + k];
    }
    for (int k = 0; k < 7; ++k) s[k] = 0ull;
    // mass and body-frame inertia per unit fluid density
    const float *h = b.half_extent;
    float m, I[3];
    if (b.shape == 1) {
        const float r = h[0];
        m = __fmul_rn(b.relative_density, __fmul_rn(__fmul_rn(__fmul_rn(4.18879032f, r), r), r)); // float32(4 pi / 3)
        I[0] = I[1] = I[2] = __fmul_rn(__fmul_rn(0.4f, m), __fmul_rn(r, r));
    } else {
        m = __fmul_rn(b.relative_density, __fmul_rn(__fmul_rn(__fmul_rn(8.0f, h[0]), h[1]), h[2]));
        const float hh[3] = {__fmul_rn(h[0], h[0]), __fmul_rn(h[1], h[1]), __fmul_rn(h[2], h[2])};
        I[0] = __fdiv_rn(__fmul_rn(m, __fadd_rn(hh[1], hh[2])), 3.0f);
        I[1] = __fdiv_rn(__fmul_rn(m, __fadd_rn(hh[0], hh[2])), 3.0f);
        I[2] = __fdiv_rn(__fmul_rn(m, __fadd_rn(hh[0], hh[1])), 3.0f);
    }
    const float dt = params->dt;
    float R[9];
    rotation_of(b.rotation, R);
    float ab[3];
    for (int j = 0; j < 3; ++j) ab[j] = __fdiv_rn(dot3(R[j], R[3 + j], R[6 + j], tau[0], tau[1], tau[2]), I[j]); // I_b^-1 (R^T tau)
    for (int k = 0; k < 3; ++k) {
        b.velocity[k] = __fadd_rn(b.velocity[k], __fmul_rn(dt, __fadd_rn(params->gravity[k], __fdiv_rn(F[k], m))));
        b.angular_velocity[k] = __fadd_rn(b.angular_velocity[k], __fmul_rn(dt, dot3(R[3 * k], R[3 * k + 1], R[3 * k + 2], ab[0], ab[1], ab[2])));
        b.centre[k] = __fadd_rn(b.centre[k], __fmul_rn(dt, b.velocity[k]));
    }
    // q += dt/2 (0, w) q, then normalise
    const float *w = b.angular_velocity, *q = b.rotation;
    const float dq[4] = {-dot3(w[0], w[1], w[2], q[1], q[2], q[3]),
                         __fadd_rn(__fmul_rn(q[0], w[0]), __fsub_rn(__fmul_rn(w[1], q[3]), __fmul_rn(w[2], q[2]))),
                         __fadd_rn(__fmul_rn(q[0], w[1]), __fsub_rn(__fmul_rn(w[2], q[1]), __fmul_rn(w[0], q[3]))),
                         __fadd_rn(__fmul_rn(q[0], w[2]), __fsub_rn(__fmul_rn(w[0], q[2]), __fmul_rn(w[1], q[1])))};
    const float half_dt = __fmul_rn(0.5f, dt);
    float qn[4];
    for (int k = 0; k < 4; ++k) qn[k] = __fadd_rn(q[k], __fmul_rn(half_dt, dq[k]));
    const float norm = __fsqrt_rn(__fadd_rn(dot3(qn[0], qn[1], qn[2], qn[0], qn[1], qn[2]), __fmul_rn(qn[3], qn[3])));
    for (int k = 0; k < 4; ++k) b.rotation[k] = __fdiv_rn(qn[k], norm);
    // the tank clamp: the bounding box at the new pose stays in [1, dim - 1]; the outward velocity component is zeroed
    rotation_of(b.rotation, R);
    float e[3];
    bounding_extents(b, R, e);
    const int dim[3] = {g.nx, g.ny, g.nz};
    for (int k = 0; k < 3; ++k) {
        if (__fsub_rn(b.centre[k], e[k]) < 1.0f) {
            b.centre[k] = __fadd_rn(1.0f, e[k]);
            if (b.velocity[k] < 0.0f) b.velocity[k] = 0.0f;
        }
        const float top = (float)(dim[k] - 1);
        if (__fadd_rn(b.centre[k], e[k]) > top) {
            b.centre[k] = __fsub_rn(top, e[k]);
            if (b.velocity[k] > 0.0f) b.velocity[k] = 0.0f;
        }
    }
    bodies[bi] = b;
    for (int k = 0; k < 3; ++k) {
        rec.centre[k] = b.centre[k];
        rec.velocity[k] = b.velocity[k];
        rec.angular_velocity[k] = b.angular_velocity[k];
    }
    for (int k = 0; k < 4; ++k) rec.rotation[k] = b.rotation[k];
    rec.reserved = 0u;
    ring[(size_t)bi * BODY_HISTORY_LENGTH + rec.step % BODY_HISTORY_LENGTH] = rec;
}

} // namespace

uint32_t body_cube_side(const BlubBody &b) {
    const float *h = b.half_extent;
    const double r = b.shape == 1 ? (double)h[0] : std::sqrt((double)h[0] * h[0] + (double)h[1] * h[1] + (double)h[2] * h[2]);
    return (uint32_t)std::ceil(2.0 * r) + 2u; // floor(c - e) .. floor(c + e) with e <= r
}

void body_bounding_extents(const BlubBody &b, float e[3]) {
    const float *q = b.rotation;
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                        2 * (y * z - w * x), 2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
    for (int k = 0; k < 3; ++k)
        e[k] = b.shape == 1 ? b.half_extent[0]
                            : std::fabs(R[3 * k]) * b.half_extent[0] + std::fabs(R[3 * k + 1]) * b.half_extent[1] + std::fabs(R[3 * k + 2]) * b.half_extent[2];
}

void launch_body_composite(cudaStream_t st, const GridDim &g, const uint2 *vox, uint2 *composite, int num_bodies, uint32_t cube, const BlubBody *bodies) {
    if (num_bodies <= 0) return;
    const size_t bytes = (size_t)g.n * sizeof(uint2);
    if (vox) BLUB_CUDA_CHECK(cudaMemcpyAsync(composite, vox, bytes, cudaMemcpyDeviceToDevice, st));
    else BLUB_CUDA_CHECK(cudaMemsetAsync(composite, 0, bytes, st));
    const dim3 grid((unsigned)std::min(blocks_for((int64_t)cube * cube * cube, PT), device_sm_count() * 8), (unsigned)num_bodies);
    BLUB_LAUNCH(body_composite_kernel, grid, PT, 0, st, g, num_bodies, cube, bodies, composite);
}

void launch_body_step(cudaStream_t st, const GridDim &g, const StepParams *params, int num_bodies, uint32_t cube, BlubBody *bodies, const int8_t *marker,
                      const float *p_vel, unsigned long long *sums, BlubBodyRecord *ring) {
    if (num_bodies <= 0) return;
    const dim3 grid((unsigned)std::min(blocks_for((int64_t)cube * cube * cube, PT), device_sm_count() * 8), (unsigned)num_bodies);
    BLUB_LAUNCH(body_load_kernel, grid, PT, 0, st, g, params, cube, bodies, marker, p_vel, sums);
    BLUB_LAUNCH(body_integrate_kernel, 1, 32, 0, st, g, params, num_bodies, bodies, sums, ring);
}

} // namespace blub
