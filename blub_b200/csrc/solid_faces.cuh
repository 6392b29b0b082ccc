// solid_faces.cuh -- the face rule of the solid load probes (DESIGN.md §8 "Solid load probes"), shared by the probes (load_kernels.cu) and the
// floating bodies (body_kernels.cu), so that both sum the same fixed-point values.
#pragma once
#include "common.cuh"

namespace blub {

constexpr int LOAD_FIELDS = 7; // force x, y, z, torque x, y, z, wetted faces

__device__ __forceinline__ long long force_fixed(float q) { return __float2ll_rn(__fmul_rn(q, (float)(1 << BLUB_LOAD_FORCE_FRAC_BITS))); }
__device__ __forceinline__ long long torque_fixed(float r, float q) {
    return __float2ll_rn(__fmul_rn(__fmul_rn(r, q), (float)(1 << BLUB_LOAD_TORQUE_FRAC_BITS)));
}

// The wetted faces of the SOLID cell c (linear index s): every FLUID neighbour inside the grid adds its fixed-point force to acc[0..2] and its
// torque about `pivot` to acc[3..5].  Returns the number of faces.
__device__ __forceinline__ unsigned add_wetted_faces(const GridDim &g, const int8_t *__restrict__ marker, const float *__restrict__ p_vel, float inv_dt,
                                                     const int c[3], int64_t s, const float pivot[3], long long acc[6]) {
    const int dim[3] = {g.nx, g.ny, g.nz};
    const int64_t stride[3] = {1, g.sy, g.sz};
    unsigned faces = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int d = -1; d <= 1; d += 2) {
            const int n = c[a] + d;
            if (n < 0 || n >= dim[a]) continue;
            const int64_t f = s + d * stride[a];
            if (marker[f] != CELL_FLUID) continue;
            // the solver's volume holds -p dt / density (divergence_remove: u_face -= p_cell - p_next): q = p / density
            const float q = -__fmul_rn(p_vel[f], inv_dt);
            // face centre: the mean of the two cell centres; r = centre - pivot
            float r[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float centre = k == a ? (float)(d > 0 ? n : c[a]) : (float)c[k] + 0.5f;
                r[k] = __fsub_rn(centre, pivot[k]);
            }
            // force -d * q along a; torque components b1 = a + 1, b2 = a + 2 (mod 3): tau_b1 = r_b2 * F_a, tau_b2 = -r_b1 * F_a
            const int b1 = a == 2 ? 0 : a + 1, b2 = a == 0 ? 2 : a - 1;
            const long long fq = force_fixed(q), t1 = torque_fixed(r[b2], q), t2 = torque_fixed(r[b1], q);
            if (d > 0) {
                acc[a] -= fq;
                acc[3 + b1] -= t1;
                acc[3 + b2] += t2;
            } else {
                acc[a] += fq;
                acc[3 + b1] += t1;
                acc[3 + b2] -= t2;
            }
            faces += 1u;
        }
    }
    return faces;
}

// The block's sums of the seven fields: the warp reduces with shuffles, the block adds its warps in shared memory.  Every thread of the
// block must call it; thread k < LOAD_FIELDS returns the sum of field k (two's complement: signed sums come out right), the others 0.
template <int BLOCK>
__device__ __forceinline__ unsigned long long block_load_sum(const long long acc[6], unsigned long long faces, unsigned long long (*part)[LOAD_FIELDS]) {
    unsigned long long v[LOAD_FIELDS] = {(unsigned long long)acc[0], (unsigned long long)acc[1], (unsigned long long)acc[2], (unsigned long long)acc[3],
                                         (unsigned long long)acc[4], (unsigned long long)acc[5], faces};
#pragma unroll
    for (int k = 0; k < LOAD_FIELDS; ++k)
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
        for (int k = 0; k < LOAD_FIELDS; ++k) part[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x >= LOAD_FIELDS) return 0;
    unsigned long long sum = 0;
    for (int w = 0; w < BLOCK / 32; ++w) sum += part[w][threadIdx.x];
    return sum;
}

} // namespace blub
