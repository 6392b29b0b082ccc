// viscosity_kernels.cu -- viscous liquids: the component-wise implicit diffusion (I - k Laplace) x_c = w_c, k = nu * dt, of the three grid
// velocity components at the end of stage 0 (sm_90a).  The rule is in DESIGN.md §8 "Viscous liquids".  Not in the reference.
//
// A set-up pass in the shape of the grid passes classifies the faces and lists the 32-cell words that hold a live face; one persistent
// cooperative kernel then runs Jacobi-preconditioned CG on all three components at once, warps walking the word list with lane = cell.
#include "fluid_kernels.hpp"
#include "grid_reduce.cuh"
#include "grid_words.cuh"

namespace blub {
namespace {

// Code of one component of a cell, 10 bits (component c at bits 10 c of the cell's word): bits 0-5 = the neighbour face at -x, +x, -y, +y,
// -z, +z is live (coupled), bit 6 = the face is live, bits 7-9 = m, the number of live and Dirichlet neighbours.
constexpr uint32_t VISC_LIVE = 1u << 6;
constexpr uint32_t VISC_LIVE_ANY = VISC_LIVE | (VISC_LIVE << 10) | (VISC_LIVE << 20);

__device__ __forceinline__ float voxel_component(const Voxel &v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : v.z); }

// Classifies face (x, y, z) of component C; a live face gets its right-hand side w + k * (sum of the Dirichlet values) in rhs[i].
template <int C>
__device__ __forceinline__ uint32_t viscosity_face_setup(const GridDim &g, const int8_t *__restrict__ marker, const uint2 *__restrict__ vox,
                                                         const float *__restrict__ u, float *__restrict__ rhs, int i, int x, int y, int z, int mi,
                                                         float k, float gravity_dt) {
    const int e[3] = {1, g.sy, g.sz}, dim[3] = {g.nx, g.ny, g.nz}, pos[3] = {x, y, z};
    const int mn = pos[C] + 1 < dim[C] ? marker[i + e[C]] : CELL_SOLID;
    if (!((mi == CELL_FLUID || mn == CELL_FLUID) && mi != CELL_SOLID && mn != CELL_SOLID)) return 0u;
    uint32_t code = VISC_LIVE, m = 0;
    float dirichlet = 0.0f;
#pragma unroll
    for (int d = 0; d < 3; ++d)
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            // the neighbour face lies between cells a = j and b = j + e_C
            const int pa = pos[d] + (side ? 1 : -1), j = i + (side ? e[d] : -e[d]);
            const bool in_a = pa >= 0 && pa < dim[d], in_b = in_a && (d == C ? pa : pos[C]) + 1 < dim[C];
            const int ma = in_a ? marker[j] : CELL_SOLID, mb = in_b ? marker[j + e[C]] : CELL_SOLID;
            if (ma == CELL_SOLID || mb == CELL_SOLID) { // no-slip: the solid's velocity, 0 outside the grid
                m += 1u;
                if (ma == CELL_SOLID ? in_a : in_b) dirichlet += voxel_component(load_voxel(vox, ma == CELL_SOLID ? j : j + e[C]), C);
            } else if (ma == CELL_FLUID || mb == CELL_FLUID) {
                code |= 1u << (2 * d + side);
                m += 1u;
            }
        }
    rhs[i] = (u[i] - gravity_dt) + k * dirichlet;
    return code | (m << 7);
}

__global__ void __launch_bounds__(PT) viscosity_setup_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params,
                                                             const BlubViscosity *__restrict__ vb, const int8_t *__restrict__ marker,
                                                             const uint2 *__restrict__ vox, const float *__restrict__ ux,
                                                             const float *__restrict__ uy, const float *__restrict__ uz, uint32_t *__restrict__ codes,
                                                             float *__restrict__ rx, float *__restrict__ ry, float *__restrict__ rz,
                                                             uint32_t *__restrict__ word_flags) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_word(g, b, p) : 0u; // a live face lies in a FLUID cell or at the low side of one
    const float k = vb->kinematic_viscosity * params->dt;
    const int lane = threadIdx.x & 31;
    uint32_t active = 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int src) {
        uint32_t code = 0u;
        const int i = lin(g, x, y, z);
        if (on) {
            const int mi = marker[i];
            code = viscosity_face_setup<0>(g, marker, vox, ux, rx, i, x, y, z, mi, k, params->gravity_dt[0]) |
                   viscosity_face_setup<1>(g, marker, vox, uy, ry, i, x, y, z, mi, k, params->gravity_dt[1]) << 10 |
                   viscosity_face_setup<2>(g, marker, vox, uz, rz, i, x, y, z, mi, k, params->gravity_dt[2]) << 20;
        }
        if (x < g.nx) codes[i] = code;
        const unsigned any = __ballot_sync(0xffffffffu, code != 0u);
        if (lane == src) active = any != 0u ? 1u : 0u;
    });
    const int w = blockIdx.x * PT + threadIdx.x;
    if (w <= b.wpr * g.ny * g.nz) word_flags[w] = active; // one entry beyond the words: the scan leaves the number of active words there
}

// flags scanned in place: word w is active when the scan steps behind it.  Also zeroes the solve's arrival counter.
__global__ void __launch_bounds__(PT) viscosity_list_kernel(int num_words, const uint32_t *__restrict__ scanned, uint32_t *__restrict__ words,
                                                            unsigned *__restrict__ barrier) {
    const int w = blockIdx.x * PT + threadIdx.x;
    if (w == 0) *barrier = 0u;
    if (w >= num_words) return;
    const uint32_t at = scanned[w];
    if (scanned[w + 1] != at) words[at] = (uint32_t)w;
}

struct ViscositySolveArgs {
    GridDim g;
    int wpr;
    const uint32_t *codes, *words, *num_words;
    float *u[3], *r[3], *s[3];
    float *partials;
    unsigned *barrier;
    const StepParams *params;
    const BlubViscosity *vb;
    ViscositySolveInfo *info;
};

// Row i of A applied to v - sub: (1 + k m) (v_i - sub) - k * (sum of the coupled neighbours, in the order -x, +x, -y, +y, -z, +z).  The
// neighbours are other threads' values of this solve: read from L2.
__device__ __forceinline__ float viscosity_row(uint32_t code, float k, float own, const float *v, int i, int sy, int sz, float sub) {
    float sum = 0.0f;
    if (code & 1u) sum += __ldcg(v + i - 1) - sub;
    if (code & 2u) sum += __ldcg(v + i + 1) - sub;
    if (code & 4u) sum += __ldcg(v + i - sy) - sub;
    if (code & 8u) sum += __ldcg(v + i + sy) - sub;
    if (code & 16u) sum += __ldcg(v + i - sz) - sub;
    if (code & 32u) sum += __ldcg(v + i + sz) - sub;
    return (1.0f + k * (float)((code >> 7) & 7u)) * own - k * sum;
}

// x is kept in the velocity volumes as u = x + gravity_dt: x_0 = w = u* - gravity_dt is what they hold on entry, x += alpha s is u += alpha s,
// and a face whose residual is zero from the start is never written.  s is stored, so an iteration has three grid-wide rounds: s . A s, then
// r . z with max |r| behind the update, then a plain one behind the new s.
__global__ void __launch_bounds__(PCG_THREADS, 4) viscosity_solve_kernel(ViscositySolveArgs a) {
    __shared__ ReduceScratchN<3> sc;
    const int lane = threadIdx.x & 31, warp0 = blockIdx.x * (PCG_THREADS / 32) + (threadIdx.x >> 5), warps = gridDim.x * (PCG_THREADS / 32);
    const int num_words = (int)*a.num_words, nx = a.g.nx, sy = a.g.sy, sz = a.g.sz, nb = (int)gridDim.x;
    const float k = a.vb->kinematic_viscosity * a.params->dt, tolerance = a.vb->error_tolerance;
    const int max_iterations = a.vb->max_num_iterations;
    const float gdt[3] = {a.params->gravity_dt[0], a.params->gravity_dt[1], a.params->gravity_dt[2]};
    unsigned round = 0u;
    // body(i, c, code of component c) for every live face of the words this warp walks
    auto walk = [&](auto &&body) {
        for (int w = warp0; w < num_words; w += warps) {
            const int word = (int)__ldg(a.words + w), row = word / a.wpr, x = (word - row * a.wpr) * 32 + lane, i = row * nx + x;
            const uint32_t code = x < nx ? __ldg(a.codes + i) : 0u;
            if (!(code & VISC_LIVE_ANY)) continue;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const uint32_t cc = (code >> (10 * c)) & 1023u;
                if (cc & VISC_LIVE) body(i, c, cc);
            }
        }
    };
    auto reduce = [&](const float (&acc)[3], const float (&err)[3], double (&tot)[3], float (&gmax)[3]) {
        grid_reduce_n<3>(a.barrier, round, a.partials + (round & 1u) * 6 * nb, acc, err, sc, tot, gmax);
    };
    const float zero[3] = {0.0f, 0.0f, 0.0f};
    float acc[3] = {0.0f, 0.0f, 0.0f}, err[3] = {0.0f, 0.0f, 0.0f}, sigma[3], alpha[3], beta[3], max_error[3];
    double tot[3];
    bool active[3];

    // r = b - A x_0 (the set-up left b in r), z = r / diagonal, s = z
    walk([&](int i, int c, uint32_t code) {
        const float diag = 1.0f + k * (float)((code >> 7) & 7u);
        const float r = a.r[c][i] - viscosity_row(code, k, a.u[c][i] - gdt[c], a.u[c], i, sy, sz, gdt[c]);
        const float z = r / diag;
        a.r[c][i] = r;
        a.s[c][i] = z;
        acc[c] += r * z;
        err[c] = fmaxf(err[c], fabsf(r));
    });
    reduce(acc, err, tot, max_error);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        sigma[c] = (float)tot[c];
        active[c] = max_error[c] > tolerance;
        alpha[c] = beta[c] = 0.0f;
    }
    int iterations = 0;
    while (iterations < max_iterations && (active[0] || active[1] || active[2])) {
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = err[c] = 0.0f;
        walk([&](int i, int c, uint32_t code) {
            if (!active[c]) return;
            const float s = a.s[c][i];
            acc[c] += s * viscosity_row(code, k, s, a.s[c], i, sy, sz, 0.0f);
        });
        float none[3];
        reduce(acc, zero, tot, none);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (active[c]) alpha[c] = guarded_div(sigma[c], (float)tot[c]);
            acc[c] = 0.0f;
        }
        walk([&](int i, int c, uint32_t code) {
            if (!active[c]) return;
            const float s = a.s[c][i];
            const float q = viscosity_row(code, k, s, a.s[c], i, sy, sz, 0.0f); // as the first pass formed it
            const float r = a.r[c][i] - alpha[c] * q;
            a.u[c][i] += alpha[c] * s;
            a.r[c][i] = r;
            acc[c] += r * (r / (1.0f + k * (float)((code >> 7) & 7u)));
            err[c] = fmaxf(err[c], fabsf(r));
        });
        float gmax[3];
        reduce(acc, err, tot, gmax);
        iterations += 1;
#pragma unroll
        for (int c = 0; c < 3; ++c)
            if (active[c]) {
                beta[c] = guarded_div((float)tot[c], sigma[c]);
                sigma[c] = (float)tot[c];
                max_error[c] = gmax[c];
                active[c] = gmax[c] > tolerance; // a component that has met the tolerance stops updating
            }
        if (iterations == max_iterations || !(active[0] || active[1] || active[2])) break;
        walk([&](int i, int c, uint32_t code) {
            if (!active[c]) return;
            a.s[c][i] = a.r[c][i] / (1.0f + k * (float)((code >> 7) & 7u)) + beta[c] * a.s[c][i];
        });
        reduce(zero, zero, tot, none); // everybody's s before anybody's A s
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.info->iterations = iterations;
        for (int c = 0; c < 3; ++c) a.info->max_error[c] = max_error[c];
    }
}

} // namespace

int viscosity_solve_blocks() {
    int per = 0;
    BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, viscosity_solve_kernel, PCG_THREADS, 0));
    int coop = 0, dev = 0;
    BLUB_CUDA_CHECK(cudaGetDevice(&dev));
    BLUB_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (per <= 0 || !coop) throw CudaError("the viscosity solve needs a cooperative launch, which this device does not offer");
    return device_sm_count() * per;
}

void launch_viscosity(cudaStream_t st, const GridDim &g, const StepParams *params, const FluidBits &bits, const int8_t *marker, const uint2 *vox,
                      float *const u[3], const ViscosityWork &w) {
    const int num_words = bits.wpr * g.ny * g.nz;
    BLUB_LAUNCH(viscosity_setup_kernel, (num_words + 1 + PT - 1) / PT, PT, 0, st, g, bits, params, w.block, marker, vox, u[0], u[1], u[2], w.codes, w.r[0], w.r[1],
                w.r[2], w.word_flags);
    launch_exclusive_scan(st, w.word_flags, (int64_t)num_words + 1, w.scan_sums);
    BLUB_LAUNCH(viscosity_list_kernel, (num_words + PT - 1) / PT, PT, 0, st, num_words, w.word_flags, w.words, w.barrier);
    ViscositySolveArgs a;
    a.g = g;
    a.wpr = bits.wpr;
    a.codes = w.codes;
    a.words = w.words;
    a.num_words = w.word_flags + num_words;
    for (int c = 0; c < 3; ++c) a.u[c] = u[c], a.r[c] = w.r[c], a.s[c] = w.s[c];
    a.partials = w.partials;
    a.barrier = w.barrier;
    a.params = params;
    a.vb = w.block;
    a.info = w.info;
    void *kargs[] = {&a};
    BLUB_CUDA_CHECK(cudaLaunchCooperativeKernel((const void *)viscosity_solve_kernel, dim3(w.blocks), dim3(PCG_THREADS), kargs, 0, st));
    g_kernel_launches.fetch_add(1, std::memory_order_relaxed);
}

} // namespace blub
