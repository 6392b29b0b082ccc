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

// A mesh body's grid-axis bounding box is centred on c + R mid, not on c: off = R mid (dot3 order).
__device__ __forceinline__ void mesh_box_offset(const float R[9], const float mid[3], float off[3]) {
    for (int k = 0; k < 3; ++k) off[k] = dot3(R[3 * k], R[3 * k + 1], R[3 * k + 2], mid[0], mid[1], mid[2]);
}

// The first cell of a mesh body's launch cube: floor((c + R mid) - e), at least 0.  Computed once per step by the transform kernel.
__device__ __forceinline__ void mesh_cube_origin(const BlubBody &b, const float R[9], const float mid[3], int lo[3]) {
    float e[3], off[3];
    bounding_extents(b, R, e);
    mesh_box_offset(R, mid, off);
    for (int k = 0; k < 3; ++k) lo[k] = max(0, (int)floorf(__fsub_rn(__fadd_rn(b.centre[k], off[k]), e[k])));
}

// The first cell of the launch cube of body b: floor(c - e), at least 0; a mesh body's as the transform kernel stored it this step.
__device__ __forceinline__ void cube_origin(const BlubBody &b, const float R[9], const MeshBodies &mb, int bi, int lo[3]) {
    if (b.shape == 2) {
        for (int k = 0; k < 3; ++k) lo[k] = mb.origin[3 * bi + k];
        return;
    }
    float e[3];
    bounding_extents(b, R, e);
    for (int k = 0; k < 3; ++k) lo[k] = max(0, (int)floorf(__fsub_rn(b.centre[k], e[k])));
}

// The cell rule: the cell centre (index + 0.5) lies inside the body.  d = centre - c on return.  A mesh body (shape 2) reads the parity
// bit stage 0 filled for body bi over its launch cube.
__device__ __forceinline__ bool covers(const BlubBody &b, const float R[9], int x, int y, int z, float d[3], const MeshBodies &mb, int bi, uint32_t cube) {
    d[0] = __fsub_rn((float)x + 0.5f, b.centre[0]);
    d[1] = __fsub_rn((float)y + 0.5f, b.centre[1]);
    d[2] = __fsub_rn((float)z + 0.5f, b.centre[2]);
    if (b.shape == 1) return dot3(d[0], d[1], d[2], d[0], d[1], d[2]) <= __fmul_rn(b.half_extent[0], b.half_extent[0]);
    if (b.shape == 2) {
        int lo[3];
        cube_origin(b, R, mb, bi, lo);
        const int lx = x - lo[0], ly = y - lo[1], lz = z - lo[2];
        if (lx < 0 || ly < 0 || lz < 0 || lx >= (int)cube || ly >= (int)cube || lz >= (int)cube) return false;
        const uint32_t w = mb.bits[(((size_t)bi * cube + lz) * cube + ly) * mb.words + (lx >> 5)];
        return (w >> (lx & 31)) & 1u;
    }
    for (int j = 0; j < 3; ++j) // body coordinate j = (R^T d)_j
        if (!(fabsf(dot3(R[j], R[3 + j], R[6 + j], d[0], d[1], d[2])) <= b.half_extent[j])) return false;
    return true;
}

// ---- the mesh bodies' solid fill (stage 0, before the composite kernel) ----

// blockIdx.y = body; the blocks of x stride over its vertices: grid position c + R v, each coordinate c_k + dot3(R_k, v).  Thread 0 of
// block 0 stores the body's launch cube origin for the later kernels of the step.
__global__ void __launch_bounds__(PT) mesh_body_transform_kernel(const BlubBody *__restrict__ bodies, const MeshBodyDev *__restrict__ info,
                                                                 const float *__restrict__ vb, float *__restrict__ vg, int *__restrict__ origin) {
    const MeshBodyDev m = info[blockIdx.y];
    if (m.num_triangles == 0) return;
    const BlubBody b = bodies[blockIdx.y];
    float R[9];
    rotation_of(b.rotation, R);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int lo[3];
        mesh_cube_origin(b, R, m.mid, lo);
        for (int k = 0; k < 3; ++k) origin[3 * blockIdx.y + k] = lo[k];
    }
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < m.num_vertices; i += gridDim.x * PT) {
        const float *v = vb + 3 * (size_t)(m.first_vertex + i);
        float *o = vg + 3 * (size_t)(m.first_vertex + i);
        for (int k = 0; k < 3; ++k) o[k] = __fadd_rn(b.centre[k], dot3(R[3 * k], R[3 * k + 1], R[3 * k + 2], v[0], v[1], v[2]));
    }
}

// The 2D edge function of the projection onto (y, z): (v - u) x (p - u), in float64 from the float32 coordinates, with the endpoints in a
// canonical order (lexicographic in (y, z)) and the value negated when they were swapped: the two triangles that share an edge get exactly
// opposite values.
__device__ __forceinline__ double edge_function(float uy, float uz, float vy, float vz, double py, double pz) {
    const bool swap = uy > vy || (uy == vy && uz > vz);
    const double ay = swap ? vy : uy, az = swap ? vz : uz, by = swap ? uy : vy, bz = swap ? uz : vz;
    const double e = __dsub_rn(__dmul_rn(__dsub_rn(by, ay), __dsub_rn(pz, az)), __dmul_rn(__dsub_rn(bz, az), __dsub_rn(py, ay)));
    return swap ? -e : e;
}

// Top-left in the counter-clockwise-normalised projection: the edge's direction d = (dy, dz) has dz > 0, or dz == 0 and dy < 0.  Exactly one
// of d and -d is top-left, so a row on a shared edge is counted by one of the two triangles.
__device__ __forceinline__ bool top_left(float dy, float dz) { return dz > 0.0f || (dz == 0.0f && dy < 0.0f); }

// blockIdx.y = body; the warps of x stride over its triangles, the lanes of a warp over the triangle's rows.  For every cell-centre row
// (y + 0.5, z + 0.5) of the launch cube inside the triangle's yz projection, the crossing x* flips the bit of the first cell whose centre lies
// beyond it (x + 0.5 > x*).
__global__ void __launch_bounds__(PT) mesh_body_cross_kernel(GridDim g, uint32_t cube, uint32_t words, const BlubBody *__restrict__ bodies,
                                                             const MeshBodyDev *__restrict__ info, const int *__restrict__ origin,
                                                             const uint32_t *__restrict__ indices, const float *__restrict__ vg,
                                                             uint32_t *__restrict__ bits) {
    const int bi = blockIdx.y;
    const MeshBodyDev m = info[bi];
    if (m.num_triangles == 0) return;
    const int lo[3] = {origin[3 * bi], origin[3 * bi + 1], origin[3 * bi + 2]};
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t *body_bits = bits + (size_t)bi * cube * cube * words;
    for (uint32_t t = (blockIdx.x * PT + threadIdx.x) >> 5; t < m.num_triangles; t += gridDim.x * (PT / 32)) {
        const uint32_t *tri = indices + 3 * (size_t)(m.first_triangle + t);
        float v[3][3];
        for (int c = 0; c < 3; ++c)
            for (int k = 0; k < 3; ++k) v[c][k] = vg[3 * (size_t)tri[c] + k];
        // orientation of the projection; a triangle whose projection has zero area crosses no row
        const double area = edge_function(v[0][1], v[0][2], v[1][1], v[1][2], v[2][1], v[2][2]);
        if (area == 0.0) continue;
        const double s = area > 0.0 ? 1.0 : -1.0;
        bool tl[3]; // edge c runs from corner c + 1 to corner c + 2 (counter-clockwise after normalisation)
        for (int c = 0; c < 3; ++c) {
            const int a = (c + 1) % 3, e = (c + 2) % 3;
            const float dy = __fsub_rn(v[e][1], v[a][1]), dz = __fsub_rn(v[e][2], v[a][2]);
            tl[c] = area > 0.0 ? top_left(dy, dz) : top_left(-dy, -dz);
        }
        const float ymin = fminf(fminf(v[0][1], v[1][1]), v[2][1]), ymax = fmaxf(fmaxf(v[0][1], v[1][1]), v[2][1]);
        const float zmin = fminf(fminf(v[0][2], v[1][2]), v[2][2]), zmax = fmaxf(fmaxf(v[0][2], v[1][2]), v[2][2]);
        const int y0 = max(lo[1], (int)floorf(ymin - 0.5f)), y1 = min(lo[1] + (int)cube - 1, (int)ceilf(ymax - 0.5f));
        const int z0 = max(lo[2], (int)floorf(zmin - 0.5f)), z1 = min(lo[2] + (int)cube - 1, (int)ceilf(zmax - 0.5f));
        if (y1 < y0 || z1 < z0) continue;
        const uint32_t ny = (uint32_t)(y1 - y0 + 1), rows = ny * (uint32_t)(z1 - z0 + 1);
        for (uint32_t r = lane; r < rows; r += 32) {
            const int y = y0 + (int)(r % ny), z = z0 + (int)(r / ny);
            const double py = (double)y + 0.5, pz = (double)z + 0.5;
            double w[3];
            bool inside = true;
            for (int c = 0; c < 3 && inside; ++c) {
                const int a = (c + 1) % 3, e = (c + 2) % 3;
                w[c] = edge_function(v[a][1], v[a][2], v[e][1], v[e][2], py, pz);
                const double wn = s * w[c];
                inside = wn > 0.0 || (wn == 0.0 && tl[c]);
            }
            if (!inside) continue;
            // x* = (w0 x0 + w1 x1 + w2 x2) / (w0 + w1 + w2), in float64 in this order
            const double num = __dadd_rn(__dadd_rn(__dmul_rn(w[0], (double)v[0][0]), __dmul_rn(w[1], (double)v[1][0])), __dmul_rn(w[2], (double)v[2][0]));
            const double xs = __ddiv_rn(num, __dadd_rn(__dadd_rn(w[0], w[1]), w[2]));
            const long long first = (long long)floor(__dsub_rn(xs, 0.5)) + 1 - lo[0]; // the first cell with x + 0.5 > x*
            if (first >= (long long)cube) continue;
            const uint32_t lx = first < 0 ? 0u : (uint32_t)first;
            atomicXor(&body_bits[((size_t)(z - lo[2]) * cube + (y - lo[1])) * words + (lx >> 5)], 1u << (lx & 31));
        }
    }
}

// One thread per (body, z, y) row of the launch cubes: the inclusive prefix XOR along x turns the crossing bits into the crossing parity.
__global__ void __launch_bounds__(PT) mesh_body_parity_kernel(uint32_t rows, uint32_t cube, uint32_t words, const MeshBodyDev *__restrict__ info,
                                                              uint32_t *__restrict__ bits) {
    const uint32_t r = blockIdx.x * PT + threadIdx.x;
    if (r >= rows || info[r / (cube * cube)].num_triangles == 0) return;
    uint32_t *row = bits + (size_t)r * words, carry = 0u;
    for (uint32_t k = 0; k < words; ++k) {
        uint32_t x = row[k];
        x ^= x << 1;
        x ^= x << 2;
        x ^= x << 4;
        x ^= x << 8;
        x ^= x << 16;
        x ^= 0u - carry; // the parity of the words before
        row[k] = x;
        carry = x >> 31;
    }
}

// blockIdx.y = body; the blocks of x stride over its cube.  A covered cell that no later body covers gets w = 1 and the rigid velocity
// v + w x (centre - c): later bodies win, whatever order the blocks run in.
__global__ void __launch_bounds__(PT) body_composite_kernel(GridDim g, int num_bodies, uint32_t cube, const BlubBody *__restrict__ bodies,
                                                            uint2 *__restrict__ vox, MeshBodies mb) {
    const int bi = blockIdx.y;
    const BlubBody b = bodies[bi];
    float R[9];
    rotation_of(b.rotation, R);
    int lo[3];
    cube_origin(b, R, mb, bi, lo);
    const uint32_t cells = cube * cube * cube;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < cells; i += gridDim.x * PT) {
        const int x = lo[0] + (int)(i % cube), y = lo[1] + (int)(i / cube % cube), z = lo[2] + (int)(i / (cube * cube));
        if (x >= g.nx || y >= g.ny || z >= g.nz) continue;
        float d[3];
        if (!covers(b, R, x, y, z, d, mb, bi, cube)) continue;
        bool later = false;
        for (int k = bi + 1; k < num_bodies && !later; ++k) {
            const BlubBody o = bodies[k];
            float Ro[9], dd[3];
            rotation_of(o.rotation, Ro);
            later = covers(o, Ro, x, y, z, dd, mb, k, cube);
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
                                                       unsigned long long *__restrict__ sums, MeshBodies mb) {
    __shared__ unsigned long long part[PT / 32][LOAD_FIELDS];
    const int bi = blockIdx.y;
    const BlubBody b = bodies[bi];
    float R[9];
    rotation_of(b.rotation, R);
    int lo[3];
    cube_origin(b, R, mb, bi, lo);
    const float inv_dt = params->inv_dt;
    long long acc[6] = {0, 0, 0, 0, 0, 0};
    unsigned long long faces = 0;
    const uint32_t cells = cube * cube * cube;
    for (uint32_t i = blockIdx.x * PT + threadIdx.x; i < cells; i += gridDim.x * PT) {
        const int c[3] = {lo[0] + (int)(i % cube), lo[1] + (int)(i / cube % cube), lo[2] + (int)(i / (cube * cube))};
        if (c[0] >= g.nx || c[1] >= g.ny || c[2] >= g.nz) continue;
        const int64_t s = (int64_t)c[0] + (int64_t)c[1] * g.sy + (int64_t)c[2] * g.sz;
        float d[3];
        if (marker[s] != CELL_SOLID || !covers(b, R, c[0], c[1], c[2], d, mb, bi, cube)) continue;
        faces += add_wetted_faces(g, marker, p_vel, inv_dt, c, s, b.centre, acc);
    }
    const unsigned long long sum = block_load_sum<PT>(acc, faces, part);
    if (sum != 0) atomicAdd(&sums[8 * blockIdx.y + threadIdx.x], sum);
}

// One warp, lane = body: semi-implicit Euler in float32 with the tank clamp, then the record.  Reads and re-zeroes the body's sums.
__global__ void body_integrate_kernel(GridDim g, const StepParams *__restrict__ params, int num_bodies, BlubBody *__restrict__ bodies,
                                      unsigned long long *__restrict__ sums, BlubBodyRecord *__restrict__ ring, MeshBodies mb) {
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
    if (b.shape == 2) { // the mesh's, computed on the host at set time
        const MeshBodyDev &md = mb.info[bi];
        m = md.mass;
        for (int k = 0; k < 3; ++k) I[k] = md.inertia[k];
    } else if (b.shape == 1) {
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
    if (b.shape == 2) { // the box is centred on c + R mid: the lowest corner rests at 1, not a symmetric bound
        float off[3];
        mesh_box_offset(R, mb.info[bi].mid, off);
        for (int k = 0; k < 3; ++k) {
            if (__fsub_rn(__fadd_rn(b.centre[k], off[k]), e[k]) < 1.0f) {
                b.centre[k] = __fsub_rn(__fadd_rn(1.0f, e[k]), off[k]);
                if (b.velocity[k] < 0.0f) b.velocity[k] = 0.0f;
            }
            const float top = (float)(dim[k] - 1);
            if (__fadd_rn(__fadd_rn(b.centre[k], off[k]), e[k]) > top) {
                b.centre[k] = __fsub_rn(__fsub_rn(top, e[k]), off[k]);
                if (b.velocity[k] > 0.0f) b.velocity[k] = 0.0f;
            }
        }
    }
    for (int k = 0; k < 3 && b.shape != 2; ++k) {
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

void launch_mesh_body_fill(cudaStream_t st, const GridDim &g, int num_bodies, uint32_t cube, const BlubBody *bodies, const MeshBodySet &mesh) {
    if (num_bodies <= 0 || !mesh.info) return;
    const uint32_t rows = (uint32_t)num_bodies * cube * cube;
    BLUB_CUDA_CHECK(cudaMemsetAsync(mesh.bits, 0, (size_t)rows * mesh.words * sizeof(uint32_t), st));
    const int cap = device_sm_count() * 8;
    BLUB_LAUNCH(mesh_body_transform_kernel, dim3((unsigned)std::min(blocks_for(mesh.max_vertices, PT), cap), (unsigned)num_bodies), PT, 0, st, bodies,
                mesh.info, mesh.body_vertices, mesh.grid_vertices, mesh.origin);
    BLUB_LAUNCH(mesh_body_cross_kernel, dim3((unsigned)std::min(blocks_for((int64_t)mesh.max_triangles * 32, PT), cap), (unsigned)num_bodies), PT, 0, st,
                g, cube, mesh.words, bodies, mesh.info, mesh.origin, mesh.indices, mesh.grid_vertices, mesh.bits);
    BLUB_LAUNCH(mesh_body_parity_kernel, blocks_for(rows, PT), PT, 0, st, rows, cube, mesh.words, mesh.info, mesh.bits);
}

void launch_body_composite(cudaStream_t st, const GridDim &g, const uint2 *vox, uint2 *composite, int num_bodies, uint32_t cube, const BlubBody *bodies,
                           const MeshBodies &mesh) {
    if (num_bodies <= 0) return;
    const size_t bytes = (size_t)g.n * sizeof(uint2);
    if (vox) BLUB_CUDA_CHECK(cudaMemcpyAsync(composite, vox, bytes, cudaMemcpyDeviceToDevice, st));
    else BLUB_CUDA_CHECK(cudaMemsetAsync(composite, 0, bytes, st));
    const dim3 grid((unsigned)std::min(blocks_for((int64_t)cube * cube * cube, PT), device_sm_count() * 8), (unsigned)num_bodies);
    BLUB_LAUNCH(body_composite_kernel, grid, PT, 0, st, g, num_bodies, cube, bodies, composite, mesh);
}

void launch_body_step(cudaStream_t st, const GridDim &g, const StepParams *params, int num_bodies, uint32_t cube, BlubBody *bodies, const int8_t *marker,
                      const float *p_vel, unsigned long long *sums, BlubBodyRecord *ring, const MeshBodies &mesh) {
    if (num_bodies <= 0) return;
    const dim3 grid((unsigned)std::min(blocks_for((int64_t)cube * cube * cube, PT), device_sm_count() * 8), (unsigned)num_bodies);
    BLUB_LAUNCH(body_load_kernel, grid, PT, 0, st, g, params, cube, bodies, marker, p_vel, sums, mesh);
    BLUB_LAUNCH(body_integrate_kernel, 1, 32, 0, st, g, params, num_bodies, bodies, sums, ring, mesh);
}

} // namespace blub
