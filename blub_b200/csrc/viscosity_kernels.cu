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

// Per-pair coefficients (liquids of different viscosities): the cell viscosities, the step's dt and the outputs of the set-up.
struct PairSetup {
    const float *nu;
    float4 *k[3];
};

// nu of cell j when it is FLUID (m its marker), else 0
__device__ __forceinline__ float fluid_nu(const float *__restrict__ nu, int m, int j) { return m == CELL_FLUID ? __ldg(nu + j) : 0.0f; }

// Classifies face (x, y, z) of component C; a live face gets its right-hand side w + k * (sum of the Dirichlet values) in rhs[i].  PAIRS:
// every coupled or Dirichlet neighbour n has its own k_fn = float32(nu_fn dt), the right-hand side is w + sum k_fn g_n, the +x, +y, +z
// coefficients and 1 + sum k_fn go to ps.k[C][i]; a neighbour with k_fn = 0 is not coupled, and a face whose k_fn are all 0 is not live.
template <int C, bool PAIRS = false>
__device__ __forceinline__ uint32_t viscosity_face_setup(const GridDim &g, const int8_t *__restrict__ marker, const uint2 *__restrict__ vox,
                                                         const float *__restrict__ u, float *__restrict__ rhs, int i, int x, int y, int z, int mi,
                                                         float k, float gravity_dt, const PairSetup *ps = nullptr) {
    const int e[3] = {1, g.sy, g.sz}, dim[3] = {g.nx, g.ny, g.nz}, pos[3] = {x, y, z};
    const int mn = pos[C] + 1 < dim[C] ? marker[i + e[C]] : CELL_SOLID;
    if (!((mi == CELL_FLUID || mn == CELL_FLUID) && mi != CELL_SOLID && mn != CELL_SOLID)) return 0u;
    uint32_t code = VISC_LIVE, m = 0;
    float dirichlet = 0.0f, ksum = 0.0f, kplus[3] = {0.0f, 0.0f, 0.0f};
    // the face's own cells a = i and b = i + e_C, their nu summed once (float64, exact for the pair)
    const double nu_ab = PAIRS ? (double)fluid_nu(ps->nu, mi, i) + (double)fluid_nu(ps->nu, mn, i + e[C]) : 0.0;
#pragma unroll
    for (int d = 0; d < 3; ++d)
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            // the neighbour face lies between cells a = j and b = j + e_C
            const int pa = pos[d] + (side ? 1 : -1), j = i + (side ? e[d] : -e[d]);
            const bool in_a = pa >= 0 && pa < dim[d], in_b = in_a && (d == C ? pa : pos[C]) + 1 < dim[C];
            const int ma = in_a ? marker[j] : CELL_SOLID, mb = in_b ? marker[j + e[C]] : CELL_SOLID;
            if constexpr (PAIRS) {
                const bool solid = ma == CELL_SOLID || mb == CELL_SOLID;
                if (!solid && !(ma == CELL_FLUID || mb == CELL_FLUID)) continue; // a free-surface neighbour: dropped
                // nu_fn: along C the cell between the faces when it is FLUID, else (and across) the mean over the FLUID cells of both faces,
                // summed as (a + b) + (j + j + e_C) so that both faces of the pair form the same value
                const int mm = side ? mn : mi;
                float nu_fn;
                if (d == C && mm == CELL_FLUID) nu_fn = __ldg(ps->nu + (side ? i + e[C] : i));
                else {
                    const int cnt = (mi == CELL_FLUID) + (mn == CELL_FLUID) + (ma == CELL_FLUID) + (mb == CELL_FLUID);
                    const double sum = nu_ab + ((double)fluid_nu(ps->nu, ma, j) + (double)fluid_nu(ps->nu, mb, j + e[C]));
                    nu_fn = (float)(sum / (double)cnt);
                }
                const float kn = __fmul_rn(nu_fn, k);
                if (side) kplus[d] = kn;
                ksum = __fadd_rn(ksum, kn);
                if (solid) {
                    if (ma == CELL_SOLID ? in_a : in_b)
                        dirichlet = __fmaf_rn(kn, voxel_component(load_voxel(vox, ma == CELL_SOLID ? j : j + e[C]), C), dirichlet);
                } else if (kn != 0.0f) code |= 1u << (2 * d + side);
                m += 1u;
            } else {
                if (ma == CELL_SOLID || mb == CELL_SOLID) { // no-slip: the solid's velocity, 0 outside the grid
                    m += 1u;
                    if (ma == CELL_SOLID ? in_a : in_b) dirichlet += voxel_component(load_voxel(vox, ma == CELL_SOLID ? j : j + e[C]), C);
                } else if (ma == CELL_FLUID || mb == CELL_FLUID) {
                    code |= 1u << (2 * d + side);
                    m += 1u;
                }
            }
        }
    if constexpr (PAIRS) {
        if (ksum == 0.0f) return 0u; // no coupling at all: not an unknown, the face keeps its bits
        rhs[i] = (u[i] - gravity_dt) + dirichlet;
        ps->k[C][i] = make_float4(kplus[0], kplus[1], kplus[2], __fadd_rn(1.0f, ksum));
    } else {
        rhs[i] = (u[i] - gravity_dt) + k * dirichlet;
    }
    return code | (m << 7);
}

// PAIRS: k below is the step's dt, the per-pair coefficients are formed from the cell viscosities in ps.
template <bool PAIRS>
__global__ void __launch_bounds__(PT) viscosity_setup_kernel(GridDim g, FluidBits b, const StepParams *__restrict__ params,
                                                             const BlubViscosity *__restrict__ vb, const int8_t *__restrict__ marker,
                                                             const uint2 *__restrict__ vox, const float *__restrict__ ux,
                                                             const float *__restrict__ uy, const float *__restrict__ uz, uint32_t *__restrict__ codes,
                                                             float *__restrict__ rx, float *__restrict__ ry, float *__restrict__ rz,
                                                             uint32_t *__restrict__ word_flags, PairSetup ps) {
    const WordPos p = word_of_thread(g, b);
    const unsigned todo = p.inside ? near_fluid_word(g, b, p) : 0u; // a live face lies in a FLUID cell or at the low side of one
    const float k = PAIRS ? params->dt : vb->kinematic_viscosity * params->dt;
    const int lane = threadIdx.x & 31;
    uint32_t active = 0u;
    warp_walk(g, todo, p, [&](unsigned on, int x, int y, int z, int src) {
        uint32_t code = 0u;
        const int i = lin(g, x, y, z);
        if (on) {
            const int mi = marker[i];
            code = viscosity_face_setup<0, PAIRS>(g, marker, vox, ux, rx, i, x, y, z, mi, k, params->gravity_dt[0], &ps) |
                   viscosity_face_setup<1, PAIRS>(g, marker, vox, uy, ry, i, x, y, z, mi, k, params->gravity_dt[1], &ps) << 10 |
                   viscosity_face_setup<2, PAIRS>(g, marker, vox, uz, rz, i, x, y, z, mi, k, params->gravity_dt[2], &ps) << 20;
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
    const float4 *k[3]; // per-pair coefficients: TagViscosityWork::k
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

// The same with per-pair coefficients: diag (v_i - sub) - sum k_fn (v_n - sub), kc[i] = (+x, +y, +z, diagonal) of this component's face i;
// the -d coefficient is component d of kc[i - e_d].
__device__ __forceinline__ float viscosity_row_pairs(uint32_t code, float diag, const float4 *kc, float own, const float *v, int i, int sy, int sz,
                                                     float sub) {
    const float *k = reinterpret_cast<const float *>(kc + i);
    float sum = 0.0f;
    if (code & 1u) sum += __ldg(k - 4) * (__ldcg(v + i - 1) - sub);
    if (code & 2u) sum += __ldg(k) * (__ldcg(v + i + 1) - sub);
    if (code & 4u) sum += __ldg(k - 4 * sy + 1) * (__ldcg(v + i - sy) - sub);
    if (code & 8u) sum += __ldg(k + 1) * (__ldcg(v + i + sy) - sub);
    if (code & 16u) sum += __ldg(k - 4 * sz + 2) * (__ldcg(v + i - sz) - sub);
    if (code & 32u) sum += __ldg(k + 2) * (__ldcg(v + i + sz) - sub);
    return diag * own - sum;
}

// x is kept in the velocity volumes as u = x + gravity_dt: x_0 = w = u* - gravity_dt is what they hold on entry, x += alpha s is u += alpha s,
// and a face whose residual is zero from the start is never written.  s is stored, so an iteration has three grid-wide rounds: s . A s, then
// r . z with max |r| behind the update, then a plain one behind the new s.
// PAIRS: the rows of viscosity_row_pairs, z = r / diag.
template <bool PAIRS>
__global__ void __launch_bounds__(PCG_THREADS, 4) viscosity_solve_kernel(ViscositySolveArgs a) {
    __shared__ ReduceScratchN<3> sc;
    const int lane = threadIdx.x & 31, warp0 = blockIdx.x * (PCG_THREADS / 32) + (threadIdx.x >> 5), warps = gridDim.x * (PCG_THREADS / 32);
    const int num_words = (int)*a.num_words, nx = a.g.nx, sy = a.g.sy, sz = a.g.sz, nb = (int)gridDim.x;
    const float k = PAIRS ? 0.0f : a.vb->kinematic_viscosity * a.params->dt, tolerance = a.vb->error_tolerance;
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
    // the diagonal and A v of a row
    auto diagonal = [&](int i, int c, uint32_t code) {
        return PAIRS ? __ldg(reinterpret_cast<const float *>(a.k[c] + i) + 3) : 1.0f + k * (float)((code >> 7) & 7u);
    };
    auto row = [&](int i, int c, uint32_t code, float own, const float *v, float sub) {
        return PAIRS ? viscosity_row_pairs(code, diagonal(i, c, code), a.k[c], own, v, i, sy, sz, sub) : viscosity_row(code, k, own, v, i, sy, sz, sub);
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
        const float diag = diagonal(i, c, code);
        const float r = a.r[c][i] - row(i, c, code, a.u[c][i] - gdt[c], a.u[c], gdt[c]);
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
            acc[c] += s * row(i, c, code, s, a.s[c], 0.0f);
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
            const float q = row(i, c, code, s, a.s[c], 0.0f); // as the first pass formed it
            const float r = a.r[c][i] - alpha[c] * q;
            a.u[c][i] += alpha[c] * s;
            a.r[c][i] = r;
            acc[c] += r * (r / diagonal(i, c, code));
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
            a.s[c][i] = a.r[c][i] / diagonal(i, c, code) + beta[c] * a.s[c][i];
        });
        reduce(zero, zero, tot, none); // everybody's s before anybody's A s
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.info->iterations = iterations;
        for (int c = 0; c < 3; ++c) a.info->max_error[c] = max_error[c];
    }
}

} // namespace

int viscosity_solve_blocks(bool pairs) {
    int per = 0;
    BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, pairs ? (const void *)viscosity_solve_kernel<true>
                                                                                  : (const void *)viscosity_solve_kernel<false>, PCG_THREADS, 0));
    int coop = 0, dev = 0;
    BLUB_CUDA_CHECK(cudaGetDevice(&dev));
    BLUB_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (per <= 0 || !coop) throw CudaError("the viscosity solve needs a cooperative launch, which this device does not offer");
    return device_sm_count() * per;
}

void launch_viscosity(cudaStream_t st, const GridDim &g, const StepParams *params, const FluidBits &bits, const int8_t *marker, const uint2 *vox,
                      float *const u[3], const ViscosityWork &w, const TagViscosityWork *tag, bool device_count, uint32_t n_host, uint32_t np_upper,
                      const float4 *pos) {
    const int num_words = bits.wpr * g.ny * g.nz;
    PairSetup ps{};
    if (tag) {
        launch_tag_viscosity_cells(st, g, params, device_count, n_host, np_upper, pos, marker, *tag);
        ps.nu = tag->nu;
        for (int c = 0; c < 3; ++c) ps.k[c] = tag->k[c];
    }
    const int setup_blocks = (num_words + 1 + PT - 1) / PT;
    if (tag)
        BLUB_LAUNCH(viscosity_setup_kernel<true>, setup_blocks, PT, 0, st, g, bits, params, w.block, marker, vox, u[0], u[1], u[2], w.codes, w.r[0],
                    w.r[1], w.r[2], w.word_flags, ps);
    else
        BLUB_LAUNCH(viscosity_setup_kernel<false>, setup_blocks, PT, 0, st, g, bits, params, w.block, marker, vox, u[0], u[1], u[2], w.codes, w.r[0],
                    w.r[1], w.r[2], w.word_flags, ps);
    launch_exclusive_scan(st, w.word_flags, (int64_t)num_words + 1, w.scan_sums);
    BLUB_LAUNCH(viscosity_list_kernel, (num_words + PT - 1) / PT, PT, 0, st, num_words, w.word_flags, w.words, w.barrier);
    ViscositySolveArgs a{};
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
    for (int c = 0; c < 3; ++c) a.k[c] = ps.k[c];
    void *kargs[] = {&a};
    const void *solve = tag ? (const void *)viscosity_solve_kernel<true> : (const void *)viscosity_solve_kernel<false>;
    BLUB_CUDA_CHECK(cudaLaunchCooperativeKernel(solve, dim3(tag ? w.pair_blocks : w.blocks), dim3(PCG_THREADS), kargs, 0, st));
    g_kernel_launches.fetch_add(1, std::memory_order_relaxed);
}

} // namespace blub
