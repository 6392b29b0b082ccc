// surface_tension_kernels.cu -- surface tension as a pressure jump across the free surface (DESIGN.md §8 "Surface tension").  Not in the
// reference, whose free surface carries P_air = 0 and nothing else.
//
// With a kinematic surface tension s > 0 (cells^3/s^2) stage 1 of every step, after the divergence, measures the free surface's curvature and
// moves the velocity solve's Dirichlet value on AIR from 0 to the ghost value g = -dt s (k_i + k_j) / 2 of each FLUID-AIR face; stage 4, after
// the projection, adds to those faces the g the solve assumed.  pcg.cu is not touched: AIR cells stay outside the solve (p == 0 there).
//
//   1. the density splat of transfer_kernels.cu (64-bit fixed point, 2^-40) into the density accumulator, which stage 9 rebuilds anyway;
//   2. wall rule (surface_wall_kernel, the cells within 3 of FLUID): psi = (splat >> 8) + 9 * 2^28 per SOLID face neighbour on a non-SOLID
//      cell (2^-32 units: 9 * 2^28 is the 0.5625 of density_rhs_kernel); a SOLID cell takes the largest psi of its non-SOLID face
//      neighbours, without one of its edge neighbours, without one of its vertex neighbours (0 without any), so that the field is mirrored
//      across a wall, along a tank's edges and around its corners, and a flat surface meets a wall at 90 degrees;
//   3. one 1-2-1 binomial filter per axis (surface_smooth_kernel, the cells within 2 of FLUID, coordinates clamped into the grid) in int64:
//      phi = sum w psi, written into the density accumulator.  psi < 2^56 + 2^34 whatever the splat holds, so phi < 2^62 + 2^40 cannot
//      overflow;
//   4. curvature (surface_curvature_kernel, the band: FLUID cells with an AIR face neighbour and AIR cells with a FLUID one) by central
//      differences of phi in float64: integer differences first, then k = -[lap |grad|^2 - grad^T H grad] / |grad|^3, 0 when the three
//      integer differences of the gradient are 0, clamped to [-2, 2] and rounded to float32 once.  The volume is zeroed first;
//   5. right-hand side (surface_rhs_kernel): rhs_i += sum of g over the AIR face neighbours, in the order +x, +y, +z, -x, -y, -z;
//   6. stage 4 (surface_faces_kernel): u += g where the + side of a face is AIR and its - side FLUID, u -= g the other way round.
//
// Interfacial tension (DESIGN.md §8 "Interfacial tension"): with s_AB > 0 the interface between the phase-B particles (tags in a set) and
// the rest of the liquid (phase A) carries P_B - P_A = s_AB k.  Stage 1 splats every particle (the same splat as above, done once) and the
// phase-B particles alone (launch_phase_scatter), forms psi = (2 splat_B - splat_all) >> 8 with a signed wall compensation
// (interface_wall_kernel), smooths it with surface_smooth_kernel into phi (> 0 in B), measures the curvature with the same formula on the
// FLUID cells that have a FLUID face neighbour of the other phase (interface_curvature_kernel), and moves the right-hand side by +-beta_f g_f
// over those faces (interface_rhs_kernel); stage 4 applies the same beta_f g_f to the faces (interface_faces_kernel).  The matrix is unchanged.
//
// The file is compiled without FMA contraction: tests/surface_tension_ref.py and tests/interfacial_tension_ref.py restate every operation in
// the same order.
#include "fluid_kernels.hpp"
#include "grid_words.cuh"

namespace blub {
namespace {

constexpr long long WALL_COMPENSATION = 9ll << 28; // 0.5625 in units of 2^-32

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
__device__ __forceinline__ bool in_grid(const GridDim &g, int x, int y, int z) { return x >= 0 && x < g.nx && y >= 0 && y < g.ny && z >= 0 && z < g.nz; }
// the marker, SOLID outside the grid
__device__ __forceinline__ int marker_at(const GridDim &g, const int8_t *__restrict__ m, int x, int y, int z) {
    return in_grid(g, x, y, z) ? (int)m[lin(g, x, y, z)] : CELL_SOLID;
}

// FLUID cells of the word dilated by R cells in every dimension (R <= 31)
template <int R> __device__ __forceinline__ unsigned near_fluid_r(const GridDim &g, const FluidBits &b, const WordPos &p) {
    unsigned near = 0;
#pragma unroll
    for (int dz = -R; dz <= R; ++dz)
#pragma unroll
        for (int dy = -R; dy <= R; ++dy) {
            const unsigned f = fbits(g, b, p.xw, p.y + dy, p.z + dz);
            const unsigned l = fbits(g, b, p.xw - 1, p.y + dy, p.z + dz), r = fbits(g, b, p.xw + 1, p.y + dy, p.z + dz);
            near |= f;
#pragma unroll
            for (int k = 1; k <= R; ++k) near |= (f << k) | (f >> k) | (l >> (32 - k)) | (r << (32 - k));
        }
    return near & cells_mask(p);
}

// psi of a non-SOLID cell: the splat in 2^-32 units plus the wall compensation
__device__ __forceinline__ long long compensated(const GridDim &g, const int8_t *__restrict__ m, const long long *__restrict__ splat, int x, int y, int z) {
    long long v = (long long)((unsigned long long)splat[lin(g, x, y, z)] >> 8);
    const int d[6][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {-1, 0, 0}, {0, -1, 0}, {0, 0, -1}};
#pragma unroll
    for (int k = 0; k < 6; ++k)
        if (marker_at(g, m, x + d[k][0], y + d[k][1], z + d[k][2]) == CELL_SOLID) v += WALL_COMPENSATION;
    return v;
}

__global__ void __launch_bounds__(PT) surface_wall_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ m, const long long *__restrict__ splat,
                                                          long long *__restrict__ psi) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_r<3>(g, b, p) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        long long v = 0;
        if (m[lin(g, x, y, z)] != CELL_SOLID) {
            v = compensated(g, m, splat, x, y, z);
        } else { // the nearest shell with a non-SOLID cell: face, then edge, then vertex neighbours
            bool found = false;
            for (int shell = 1; shell <= 3 && !found; ++shell)
                for (int k = 0; k < 27; ++k) {
                    const int dx = k % 3 - 1, dy = k / 3 % 3 - 1, dz = k / 9 - 1;
                    if (dx * dx + dy * dy + dz * dz != shell || marker_at(g, m, x + dx, y + dy, z + dz) == CELL_SOLID) continue;
                    v = max(v, compensated(g, m, splat, x + dx, y + dy, z + dz));
                    found = true;
                }
        }
        psi[lin(g, x, y, z)] = v;
    });
}

__global__ void __launch_bounds__(PT) surface_smooth_kernel(GridDim g, FluidBits b, const long long *__restrict__ psi, long long *__restrict__ phi) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_r<2>(g, b, p) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        long long s = 0;
#pragma unroll
        for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
                for (int dx = -1; dx <= 1; ++dx) {
                    const long long w = (long long)((2 - dx * dx) * (2 - dy * dy) * (2 - dz * dz));
                    s += w * psi[lin(g, clampi(x + dx, 0, g.nx - 1), clampi(y + dy, 0, g.ny - 1), clampi(z + dz, 0, g.nz - 1))];
                }
        phi[lin(g, x, y, z)] = s;
    });
}

// the band: FLUID with an AIR face neighbour, AIR with a FLUID face neighbour
__device__ __forceinline__ bool in_band(const GridDim &g, const int8_t *__restrict__ m, int x, int y, int z) {
    const int mc = m[lin(g, x, y, z)];
    if (mc == CELL_SOLID) return false;
    const int other = mc == CELL_FLUID ? CELL_AIR : CELL_FLUID;
    return marker_at(g, m, x + 1, y, z) == other || marker_at(g, m, x - 1, y, z) == other || marker_at(g, m, x, y + 1, z) == other ||
           marker_at(g, m, x, y - 1, z) == other || marker_at(g, m, x, y, z + 1) == other || marker_at(g, m, x, y, z - 1) == other;
}

// the curvature of phi at cell i (not on the border: its 3^3 neighbourhood lies in the grid), shared by the free surface and the interface
__device__ __forceinline__ float curvature_at(const GridDim &g, const long long *__restrict__ phi, int i) {
    auto f = [&](int dx, int dy, int dz) { return phi[i + dx + dy * g.sy + dz * g.sz]; };
    const long long c = f(0, 0, 0);
    const long long ix = f(1, 0, 0) - f(-1, 0, 0), iy = f(0, 1, 0) - f(0, -1, 0), iz = f(0, 0, 1) - f(0, 0, -1);
    float out = 0.0f;
    if (ix != 0 || iy != 0 || iz != 0) {
        const double gx = 0.5 * (double)ix, gy = 0.5 * (double)iy, gz = 0.5 * (double)iz;
        const double fxx = (double)(f(1, 0, 0) - c) - (double)(c - f(-1, 0, 0));
        const double fyy = (double)(f(0, 1, 0) - c) - (double)(c - f(0, -1, 0));
        const double fzz = (double)(f(0, 0, 1) - c) - (double)(c - f(0, 0, -1));
        const double fxy = 0.25 * ((double)(f(1, 1, 0) - f(1, -1, 0)) - (double)(f(-1, 1, 0) - f(-1, -1, 0)));
        const double fxz = 0.25 * ((double)(f(1, 0, 1) - f(1, 0, -1)) - (double)(f(-1, 0, 1) - f(-1, 0, -1)));
        const double fyz = 0.25 * ((double)(f(0, 1, 1) - f(0, 1, -1)) - (double)(f(0, -1, 1) - f(0, -1, -1)));
        const double g2 = gx * gx + gy * gy + gz * gz;
        const double lap = fxx + fyy + fzz;
        const double hess = gx * gx * fxx + gy * gy * fyy + gz * gz * fzz + 2.0 * gx * gy * fxy + 2.0 * gx * gz * fxz + 2.0 * gy * gz * fyz;
        double k = -(lap * g2 - hess) / (g2 * sqrt(g2));
        k = fmin(fmax(k, -2.0), 2.0);
        out = (float)k;
    }
    return out;
}

__global__ void __launch_bounds__(PT) surface_curvature_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ m, const long long *__restrict__ phi,
                                                               float *__restrict__ kappa) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_word(g, b, p) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on || !in_band(g, m, x, y, z)) return;
        // a band cell is not on the border (border cells are SOLID)
        const int i = lin(g, x, y, z);
        kappa[i] = curvature_at(g, phi, i);
    });
}

// the ghost value of a FLUID-AIR face in the velocity solve's units (-P dt / density): c = -(dt s)
__device__ __forceinline__ float ghost(float c, float ki, float kj) { return c * (0.5f * (ki + kj)); }

__global__ void __launch_bounds__(PT) surface_rhs_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params, const float *__restrict__ sigma,
                                                         const int8_t *__restrict__ m, const float *__restrict__ kappa, float *__restrict__ rhs) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? fbits(g, b, p.xw, p.y, p.z) : 0u;
    const float c = -(params->dt * *sigma);
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z); // FLUID: not on the border
        const int nb[6] = {i + 1, i + g.sy, i + g.sz, i - 1, i - g.sy, i - g.sz};
        const float ki = kappa[i];
        float s = 0.0f;
        bool any = false;
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (m[nb[k]] == CELL_AIR) {
                s += ghost(c, ki, kappa[nb[k]]);
                any = true;
            }
        if (any) rhs[i] = rhs[i] + s;
    });
}

__global__ void __launch_bounds__(PT) surface_faces_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params, const float *__restrict__ sigma,
                                                           const int8_t *__restrict__ m, const float *__restrict__ kappa, float *__restrict__ ux,
                                                           float *__restrict__ uy, float *__restrict__ uz) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_word(g, b, p) : 0u;
    const float c = -(params->dt * *sigma);
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z);
        const int mc = m[i];
        if (mc == CELL_SOLID) return;
        float *const u[3] = {ux, uy, uz};
        const int nb[3] = {i + 1, i + g.sy, i + g.sz};
        const bool inb[3] = {x + 1 < g.nx, y + 1 < g.ny, z + 1 < g.nz};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int mn = inb[k] ? (int)m[nb[k]] : CELL_SOLID;
            if (mc == CELL_FLUID && mn == CELL_AIR) u[k][i] = u[k][i] + ghost(c, kappa[i], kappa[nb[k]]);
            else if (mc == CELL_AIR && mn == CELL_FLUID) u[k][i] = u[k][i] - ghost(c, kappa[nb[k]], kappa[i]);
        }
    });
}

// ---- interfacial tension ----------------------------------------------------------------------------------------------------------------

// psi of a non-SOLID cell: (2 splat_B - splat_all) >> 8 as hi_B - hi_A - borrow (splat_A = splat_all - splat_B modulo 2^64, so |psi| < 2^56
// whatever the splats hold), plus the wall compensation with the sign of that value
__device__ __forceinline__ long long phase_compensated(const GridDim &g, const int8_t *__restrict__ m, const long long *__restrict__ splat_all,
                                                       const long long *__restrict__ splat_b, int x, int y, int z) {
    const int i = lin(g, x, y, z);
    const unsigned long long sb = (unsigned long long)splat_b[i], sa = (unsigned long long)splat_all[i] - sb;
    long long v = (long long)(sb >> 8) - (long long)(sa >> 8) - (long long)((sb & 255ull) < (sa & 255ull));
    const long long w = v > 0 ? WALL_COMPENSATION : (v < 0 ? -WALL_COMPENSATION : 0ll);
    const int d[6][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {-1, 0, 0}, {0, -1, 0}, {0, 0, -1}};
#pragma unroll
    for (int k = 0; k < 6; ++k)
        if (marker_at(g, m, x + d[k][0], y + d[k][1], z + d[k][2]) == CELL_SOLID) v += w;
    return v;
}

// a replaces b: the larger magnitude, of two equal magnitudes the positive value
__device__ __forceinline__ bool larger_magnitude(long long a, long long b) {
    const unsigned long long ma = a < 0 ? 0ull - (unsigned long long)a : (unsigned long long)a, mb = b < 0 ? 0ull - (unsigned long long)b : (unsigned long long)b;
    return ma > mb || (ma == mb && a > b);
}

__global__ void __launch_bounds__(PT) interface_wall_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ m, const long long *__restrict__ splat_all,
                                                            const long long *__restrict__ splat_b, long long *__restrict__ psi) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_r<3>(g, b, p) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        long long v = 0;
        if (m[lin(g, x, y, z)] != CELL_SOLID) {
            v = phase_compensated(g, m, splat_all, splat_b, x, y, z);
        } else { // the nearest shell with a non-SOLID cell, as surface_wall_kernel
            bool found = false;
            for (int shell = 1; shell <= 3 && !found; ++shell)
                for (int k = 0; k < 27; ++k) {
                    const int dx = k % 3 - 1, dy = k / 3 % 3 - 1, dz = k / 9 - 1;
                    if (dx * dx + dy * dy + dz * dz != shell || marker_at(g, m, x + dx, y + dy, z + dz) == CELL_SOLID) continue;
                    const long long c = phase_compensated(g, m, splat_all, splat_b, x + dx, y + dy, z + dz);
                    if (larger_magnitude(c, v)) v = c;
                    found = true;
                }
        }
        psi[lin(g, x, y, z)] = v;
    });
}

// FLUID cell i (not on the border) and its FLUID face neighbour j of the other phase
__device__ __forceinline__ bool interface_face(const int8_t *__restrict__ m, const long long *__restrict__ phi, bool bi, int j) {
    return m[j] == CELL_FLUID && (phi[j] > 0) != bi;
}

__global__ void __launch_bounds__(PT) interface_curvature_kernel(GridDim g, FluidBits b, const int8_t *__restrict__ m, const long long *__restrict__ phi,
                                                                 float *__restrict__ kappa) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? fbits(g, b, p.xw, p.y, p.z) : 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z); // FLUID: not on the border
        const bool bi = phi[i] > 0;
        const int nb[6] = {i + 1, i + g.sy, i + g.sz, i - 1, i - g.sy, i - g.sz};
        bool band = false;
#pragma unroll
        for (int k = 0; k < 6; ++k) band |= interface_face(m, phi, bi, nb[k]);
        if (band) kappa[i] = curvature_at(g, phi, i);
    });
}

// beta_f g_f of the face between FLUID cells i and j: beta_f from the density table's face array, 1 without one
__device__ __forceinline__ float weighted_ghost(float c, float ki, float kj, const float *__restrict__ beta, int f) {
    const float gf = ghost(c, ki, kj);
    return beta ? beta[f] * gf : gf;
}

__global__ void __launch_bounds__(PT) interface_rhs_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params,
                                                           const InterfacialTensionBlock *__restrict__ blk, const int8_t *__restrict__ m,
                                                           const long long *__restrict__ phi, const float *__restrict__ kappa,
                                                           const float *__restrict__ bx, const float *__restrict__ by, const float *__restrict__ bz,
                                                           float *__restrict__ rhs) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? fbits(g, b, p.xw, p.y, p.z) : 0u;
    const float c = -(params->dt * blk->s);
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z); // FLUID: not on the border
        const int nb[6] = {i + 1, i + g.sy, i + g.sz, i - 1, i - g.sy, i - g.sz};
        const float *const beta[6] = {bx, by, bz, bx, by, bz};
        const bool bi = phi[i] > 0;
        const float ki = kappa[i];
        float s = 0.0f;
        bool any = false;
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (interface_face(m, phi, bi, nb[k])) {
                const float w = weighted_ghost(c, ki, kappa[nb[k]], beta[k], k < 3 ? i : nb[k]);
                s = bi ? s + w : s - w;
                any = true;
            }
        if (any) rhs[i] = rhs[i] + s;
    });
}

__global__ void __launch_bounds__(PT) interface_faces_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params,
                                                             const InterfacialTensionBlock *__restrict__ blk, const int8_t *__restrict__ m,
                                                             const long long *__restrict__ phi, const float *__restrict__ kappa,
                                                             const float *__restrict__ bx, const float *__restrict__ by, const float *__restrict__ bz,
                                                             float *__restrict__ ux, float *__restrict__ uy, float *__restrict__ uz) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? fbits(g, b, p.xw, p.y, p.z) : 0u;
    const float c = -(params->dt * blk->s);
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int) {
        if (!on) return;
        const int i = lin(g, x, y, z); // FLUID: not on the border
        float *const u[3] = {ux, uy, uz};
        const float *const beta[3] = {bx, by, bz};
        const int nb[3] = {i + 1, i + g.sy, i + g.sz};
        const bool bi = phi[i] > 0;
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (interface_face(m, phi, bi, nb[k])) {
                const float w = weighted_ghost(c, kappa[i], kappa[nb[k]], beta[k], i);
                u[k][i] = bi ? u[k][i] + w : u[k][i] - w;
            }
    });
}

inline int word_blocks(const GridDim &g, const FluidBits &bits) { return (int)(((int64_t)bits.wpr * g.ny * g.nz + PT - 1) / PT); }

} // namespace

void launch_surface_curvature(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, long long *density,
                              const SurfaceTensionWork &w) {
    BLUB_LAUNCH(surface_wall_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, density, w.psi);
    BLUB_LAUNCH(surface_smooth_kernel, word_blocks(g, bits), PT, 0, st, g, bits, w.psi, density);
    BLUB_CUDA_CHECK(cudaMemsetAsync(w.kappa, 0, (size_t)g.n * sizeof(float), st));
    BLUB_LAUNCH(surface_curvature_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, density, w.kappa);
}

void launch_surface_rhs(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                        const SurfaceTensionWork &w, float *rhs) {
    BLUB_LAUNCH(surface_rhs_kernel, word_blocks(g, bits), PT, 0, st, g, bits, params, w.sigma, marker, w.kappa, rhs);
}

void launch_surface_faces(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                          const SurfaceTensionWork &w, float *const u[3]) {
    BLUB_LAUNCH(surface_faces_kernel, word_blocks(g, bits), PT, 0, st, g, bits, params, w.sigma, marker, w.kappa, u[0], u[1], u[2]);
}

void launch_interface_psi(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const long long *splat_all,
                          const InterfacialTensionWork &w) {
    BLUB_LAUNCH(interface_wall_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, splat_all, w.phi, w.psi);
}

void launch_interface_curvature(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const InterfacialTensionWork &w) {
    BLUB_LAUNCH(surface_smooth_kernel, word_blocks(g, bits), PT, 0, st, g, bits, w.psi, w.phi);
    BLUB_CUDA_CHECK(cudaMemsetAsync(w.kappa, 0, (size_t)g.n * sizeof(float), st));
    BLUB_LAUNCH(interface_curvature_kernel, word_blocks(g, bits), PT, 0, st, g, bits, marker, w.phi, w.kappa);
}

void launch_interface_rhs(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                          const InterfacialTensionWork &w, const float *const *beta, float *rhs) {
    BLUB_LAUNCH(interface_rhs_kernel, word_blocks(g, bits), PT, 0, st, g, bits, params, w.block, marker, w.phi, w.kappa, beta ? beta[0] : nullptr,
                beta ? beta[1] : nullptr, beta ? beta[2] : nullptr, rhs);
}

void launch_interface_faces(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                            const InterfacialTensionWork &w, const float *const *beta, float *const u[3]) {
    BLUB_LAUNCH(interface_faces_kernel, word_blocks(g, bits), PT, 0, st, g, bits, params, w.block, marker, w.phi, w.kappa, beta ? beta[0] : nullptr,
                beta ? beta[1] : nullptr, beta ? beta[2] : nullptr, u[0], u[1], u[2]);
}

} // namespace blub
