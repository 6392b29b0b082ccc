// pcg.cu -- preconditioned conjugate gradient pressure solve (sm_90a).
//
// Replaces PressureSolver::solve (src/simulation/pressure_solver.rs:591-729) and the seven compute pipelines under
// shader/simulation/pressure_solver/.  Same recurrence, same iteration schedule (error checks at i % freq == 0 and
// i == max, pressure_solver.rs:676-677), same epsilon guards (pressure_reduce.comp:73-80) -- but not the same pass
// structure: the reference records 9 dispatches + 3 two-level reductions per iteration (313 dispatches per solve,
// ~85 B/cell/iteration).  Here a solve is
//     prepare  (once): marker -> 1-byte codes (diag, fluid) + tile activity; p, r, s <- 0 off-fluid ("zero invariant": the
//              7-point stencil, the dot products and the maxima then need no masks at all)
//     solve    ONE persistent cooperative kernel (pcg_solve_columns_kernel by default): per iteration
//                 phase A  s' = z + beta s fused with s'.A s'   (pressure_update_search.comp + pressure_apply_coeff.comp)
//                 phase B  p += a s', r -= a A s', z.r, max|r|  (pressure_update_pressure_and_residual.comp + both
//                          preconditioner passes + the BETA / MAX_ERROR reductions)
//              with two grid barriers per iteration, redundant fixed-order fp64 reductions (deterministic), the diagonal
//              ("diag2") preconditioner evaluated on the fly so that z is never stored, an immediate stop on convergence
//              (the reference zeroes its indirect-dispatch arguments instead, pressure_reduce.comp:89-92), per-thread
//              skipping of fluid-free quads in sparsely filled tiles, and -- for z-slab sharded fluids -- the halo
//              exchange and the scalar all-reduce INSIDE the kernel (P2P stores, mailboxes).
// The three persistent kernels run one solve loop (pcg_solve) and differ only in their walker -- how a phase deals its work: the
// column solver's dense tiles plus a list of fluid columns, the tile kernel's active tiles (pcg_solve_persistent_kernel, solver paths 4
// and 6), or tensor-map boxes staged in shared memory (pcg_solve_tma_kernel, path 2; bit-compatible, measured slower -- see DESIGN.md
// 3.1) -- and in their reducer: an arrival counter (grid_reduce / grid_allreduce), or cooperative_groups grid barriers.
// Also kept and tested: a three-kernel-per-iteration path (dot / update / search with last-block-done reductions; used for
// precond_mode 1 and when cooperative launch is unavailable).
//
// Layout: four cells per thread along x (128-bit loads) marching 4 z-planes with the z-neighbours kept in registers and
// the x-neighbours exchanged by warp shuffles; fp32 vectors, 1-byte cell codes, padded arrays (common.cuh); tiles without
// any FLUID cell are never visited.
#include <cooperative_groups.h>
#include <cuda.h>          // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cudaTypedefs.h>  // PFN_cuTensorMapEncodeTiled

#include <cstdlib>
#include <type_traits>

#include "blub_core.hpp"
#include "grid_reduce.cuh"

namespace blub {

std::atomic<uint64_t> g_kernel_launches{0};

namespace {

constexpr int PCG_TZ = 4;             // z planes marched by one block

// Per-cell code, built once per solve from the marker volume (pcg_prepare_kernel):
//   bits 0..2  number of non-SOLID neighbours = diagonal of A (pressure.glsl:44-53)
//   bit  3     cell is FLUID
// INVARIANT kept by every kernel of a solve: p, r and s are exactly 0 on every non-FLUID cell (and in the padding).
// Then "subtract the FLUID neighbours" (pressure.glsl:56-73) is "subtract all six neighbours", so the stencil needs no
// neighbour masks:  (A x)_i = diag_i x_i - sum_6 x_nbr  on fluid cells.
constexpr unsigned CODE_FLUID = 8u;
constexpr int TILE_DENSE_BIT = 1 << 30; // in tile_list_flagged: the tile is at least 3/4 full

// Block = (bx, by) threads, bx * by = 256; thread (lx, ly) owns the quad of 4 x-consecutive cells at
// x = 4 * (blockIdx.x * bx + lx), y = blockIdx.y * by + ly and marches PCG_TZ planes in z from blockIdx.z * PCG_TZ.
struct TileMap {
    int bx, by;
    int tiles_x, tiles_y, tiles_z;
    int qx; // quads per row
    int ntiles;
    dim3 grid() const { return dim3(tiles_x, tiles_y, tiles_z); }
    dim3 block() const { return dim3(bx, by, 1); }
};

TileMap make_tilemap(const GridDim &g) {
    TileMap t;
    t.qx = g.nx / 4;
    t.bx = t.qx > 16 ? 32 : (t.qx > 8 ? 16 : 8);
    t.by = PCG_THREADS / t.bx;
    t.tiles_x = (t.qx + t.bx - 1) / t.bx;
    t.tiles_y = (g.ny + t.by - 1) / t.by;
    t.tiles_z = g.nz / PCG_TZ;
    t.ntiles = t.tiles_x * t.tiles_y * t.tiles_z;
    return t;
}

struct TileCtx {
    int tile, tz;
    bool valid, first, last; // first/last quad of the block's row segment (x neighbours come from memory there)
    int i;                   // linear index of the quad in the block's first plane (fits: n < 2^31)
};
__device__ __forceinline__ TileCtx tile_ctx_at(const GridDim &g, const TileMap &t, int tx, int ty, int tz) {
    TileCtx c;
    const int q = tx * t.bx + threadIdx.x;
    const int y = ty * t.by + threadIdx.y;
    c.tile = (tz * t.tiles_y + ty) * t.tiles_x + tx;
    c.tz = tz;
    c.valid = q < t.qx && y < g.ny;
    c.first = threadIdx.x == 0;
    c.last = threadIdx.x == t.bx - 1 || q == t.qx - 1;
    c.i = c.valid ? (tz * PCG_TZ * g.ny + y) * g.nx + 4 * q : 0;
    return c;
}
__device__ __forceinline__ TileCtx tile_ctx(const GridDim &g, const TileMap &t) { return tile_ctx_at(g, t, blockIdx.x, blockIdx.y, blockIdx.z); }
__device__ __forceinline__ TileCtx tile_ctx_id(const GridDim &g, const TileMap &t, int tile) {
    const int tx = tile % t.tiles_x, rest = tile / t.tiles_x;
    return tile_ctx_at(g, t, tx, rest % t.tiles_y, rest / t.tiles_y);
}

__device__ __forceinline__ float4 ld4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ void st4(float *p, const float4 &v) { *reinterpret_cast<float4 *>(p) = v; }
__device__ __forceinline__ uchar4 ldcode(const uint8_t *p) { return *reinterpret_cast<const uchar4 *>(p); }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// x-neighbours of a quad: from the adjacent lanes, or from memory at the ends of the block's row segment.
// Must be called by all 32 lanes of a warp.
__device__ __forceinline__ void x_neighbours(const float *x, int i, const float4 &c, const TileCtx &t, float &left, float &right) {
    left = __shfl_up_sync(0xffffffffu, c.w, 1);
    right = __shfl_down_sync(0xffffffffu, c.x, 1);
    if (t.valid && t.first) left = x[i - 1];
    if (t.valid && t.last) right = x[i + 4];
}

// A x for a quad under the zero invariant (MultiplyWithCoefficientMatrix, pressure.glsl:34-75)
__device__ __forceinline__ float4 stencil_quad(const uchar4 &code, const float4 &c, float left, float right, const float4 &ym, const float4 &yp,
                                               const float4 &zm, const float4 &zp) {
    float4 o;
    o.x = (float)(code.x & 7u) * c.x - (((left + c.y) + (ym.x + yp.x)) + (zm.x + zp.x));
    o.y = (float)(code.y & 7u) * c.y - (((c.x + c.z) + (ym.y + yp.y)) + (zm.y + zp.y));
    o.z = (float)(code.z & 7u) * c.z - (((c.y + c.w) + (ym.z + yp.z)) + (zm.z + zp.z));
    o.w = (float)(code.w & 7u) * c.w - (((c.z + right) + (ym.w + yp.w)) + (zm.w + zp.w));
    return o;
}

// z = P(P(r)) with the LOD-1 neighbour fetches reading 0: z = (r / d) / d, d = max(diag, 1)
// (pressure_apply_preconditioner.comp:48-77, SURVEY B1).  1/d^2 by table: <= 1.5 ulp from the two divisions.
__constant__ float c_inv_diag2[8] = {1.0f, 1.0f, 0.25f, 1.0f / 9.0f, 0.0625f, 0.04f, 1.0f / 36.0f, 1.0f};
__device__ __forceinline__ float precond_diag2(float r, unsigned code) { return r * c_inv_diag2[code & 7u]; }

__device__ __forceinline__ float block_sum(float v, float *sh) {
    v = warp_sum(v);
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5;
    if (lane == 0) sh[w] = v;
    __syncthreads();
    float r = 0.0f;
    if (w == 0) {
        r = lane < (PCG_THREADS / 32) ? sh[lane] : 0.0f;
        r = warp_sum(r);
    }
    __syncthreads();
    return r; // valid in warp 0
}
__device__ __forceinline__ float block_max(float v, float *sh) {
    v = warp_max(v);
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5;
    if (lane == 0) sh[w] = v;
    __syncthreads();
    float r = 0.0f;
    if (w == 0) {
        r = lane < (PCG_THREADS / 32) ? sh[lane] : 0.0f;
        r = warp_max(r);
    }
    __syncthreads();
    return r;
}

// Publishes this block's partial(s) and returns true in exactly one block: the last one to arrive.
__device__ __forceinline__ bool publish_and_elect(PcgScalars *scal, unsigned nblocks) {
    __shared__ bool last;
    if (linear_tid() == 0) {
        __threadfence();
        unsigned t = atomicAdd(&scal->ticket, 1u);
        last = (t == nblocks - 1);
        __threadfence(); // acquire side: the partials of all earlier arrivals are visible to this block from here on
    }
    __syncthreads();
    return last;
}

// Final reduction by the elected block, in fixed order and double precision => bit-reproducible run to run.
__device__ __forceinline__ double final_sum(const float *partials, int n) {
    __shared__ double shd[PCG_THREADS / 32];
    const int tid = linear_tid();
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int k = tid;
    for (; k + 3 * PCG_THREADS < n; k += 4 * PCG_THREADS) { // four independent loads in flight
        a0 += (double)__ldcg(partials + k);
        a1 += (double)__ldcg(partials + k + PCG_THREADS);
        a2 += (double)__ldcg(partials + k + 2 * PCG_THREADS);
        a3 += (double)__ldcg(partials + k + 3 * PCG_THREADS);
    }
    for (; k < n; k += PCG_THREADS) a0 += (double)__ldcg(partials + k);
    double acc = warp_sum((a0 + a1) + (a2 + a3));
    const int lane = tid & 31, w = tid >> 5;
    if (lane == 0) shd[w] = acc;
    __syncthreads();
    double r = 0.0;
    if (w == 0) {
        r = lane < (PCG_THREADS / 32) ? shd[lane] : 0.0;
        r = warp_sum(r);
    }
    __syncthreads();
    return r;
}
__device__ __forceinline__ float final_max(const float *partials, int n, float *sh) {
    float acc = 0.0f;
    for (int k = linear_tid(); k < n; k += PCG_THREADS) acc = fmaxf(acc, __ldcg(partials + k));
    return block_max(acc, sh);
}

// ---------------------------------------------------------------------------------------------------------------
// prepare (once per solve): marker -> codes + per-tile activity; establish the zero invariant:
// p <- 0 and rhs <- 0 off-fluid (pressure_init.comp:37-43 zeroes p there), s, s1 <- 0 everywhere (s1 may be null).
// Sparse set-up (dense_flags non-null and both flags of this solve clear): a tile that holds no FLUID cell now, was inactive in the
// previous solve (tile_active: codes, r, s, s1 are all 0 there) and was not active in this field's previous solve (p_tiles: p is 0
// there) is left as it is -- it is all zeros already.  The column solver writes only inside active tiles, and the rhs kernels write
// FLUID cells of the marker the solve is prepared from.
__global__ void __launch_bounds__(PCG_THREADS) pcg_prepare_kernel(GridDim g, TileMap t, const int8_t *__restrict__ m, uint8_t *__restrict__ codes,
                                                                  uint8_t *__restrict__ tile_active, int *__restrict__ tile_cols, uint8_t *__restrict__ p_tiles,
                                                                  const int *__restrict__ dense_flags, int which, float *__restrict__ p, float *__restrict__ r,
                                                                  float *__restrict__ s, float *__restrict__ s1) {
    __shared__ int sh_units;
    const TileCtx c = tile_ctx(g, t);
    const bool sparse = dense_flags && !dense_flags[0] && !dense_flags[1 + which];
    if (sparse && !tile_active[c.tile] && !p_tiles[c.tile]) { // block-uniform
        bool fluid = false;
        if (c.valid) {
#pragma unroll
            for (int k = 0; k < PCG_TZ; ++k) {
                const char4 cc = *reinterpret_cast<const char4 *>(m + c.i + k * g.sz);
                fluid = fluid || cc.x == CELL_FLUID || cc.y == CELL_FLUID || cc.z == CELL_FLUID || cc.w == CELL_FLUID;
            }
        }
        if (!__syncthreads_or(fluid)) {
            if (linear_tid() == 0) tile_cols[c.tile] = 0;
            return;
        }
    }
    if (linear_tid() == 0) sh_units = 0;
    __syncthreads();
    int any = 0; // planes of this thread's column whose quad holds a FLUID cell
    if (c.valid) {
        int i = c.i;
#pragma unroll
        for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
            const char4 cc = *reinterpret_cast<const char4 *>(m + i);
            uchar4 out = make_uchar4(0, 0, 0, 0);
            if (cc.x == CELL_FLUID || cc.y == CELL_FLUID || cc.z == CELL_FLUID || cc.w == CELL_FLUID) {
                any += 1;
                const char4 ym = *reinterpret_cast<const char4 *>(m + i - g.sy), yp = *reinterpret_cast<const char4 *>(m + i + g.sy);
                const char4 zm = *reinterpret_cast<const char4 *>(m + i - g.sz), zp = *reinterpret_cast<const char4 *>(m + i + g.sz);
                const int cx[6] = {m[i - 1], cc.x, cc.y, cc.z, cc.w, m[i + 4]};
                const int cym[4] = {ym.x, ym.y, ym.z, ym.w}, cyp[4] = {yp.x, yp.y, yp.z, yp.w};
                const int czm[4] = {zm.x, zm.y, zm.z, zm.w}, czp[4] = {zp.x, zp.y, zp.z, zp.w};
                unsigned code[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const unsigned d = (cx[e] != CELL_SOLID) + (cx[e + 2] != CELL_SOLID) + (cym[e] != CELL_SOLID) + (cyp[e] != CELL_SOLID) +
                                       (czm[e] != CELL_SOLID) + (czp[e] != CELL_SOLID);
                    code[e] = cx[e + 1] == CELL_FLUID ? (CODE_FLUID | d) : 0u;
                }
                out = make_uchar4((unsigned char)code[0], (unsigned char)code[1], (unsigned char)code[2], (unsigned char)code[3]);
                float4 p4 = ld4(p + i), r4 = ld4(r + i);
                if (!code[0]) { p4.x = 0.f; r4.x = 0.f; }
                if (!code[1]) { p4.y = 0.f; r4.y = 0.f; }
                if (!code[2]) { p4.z = 0.f; r4.z = 0.f; }
                if (!code[3]) { p4.w = 0.f; r4.w = 0.f; }
                st4(p + i, p4);
                st4(r + i, r4);
            } else {
                st4(p + i, zero4());
                st4(r + i, zero4());
            }
            *reinterpret_cast<uchar4 *>(codes + i) = out;
            st4(s + i, zero4());
            if (s1) st4(s1 + i, zero4());
        }
    }
    const int ncols = __syncthreads_count(any > 0); // columns (thread's quad x PCG_TZ planes) that hold a FLUID cell
    any = (int)__reduce_add_sync(0xffffffffu, (unsigned)any);
    if ((linear_tid() & 31) == 0 && any) atomicAdd(&sh_units, any);
    __syncthreads();
    // 0 = no fluid, 1 = some, 2 = at least 3/4 of the (thread, plane) quads hold fluid: the persistent solver runs such a tile
    // with its branch-free body
    if (linear_tid() == 0) {
        const int flag = sh_units == 0 ? 0 : (4 * sh_units >= 3 * PCG_THREADS * PCG_TZ ? 2 : 1);
        tile_active[c.tile] = (uint8_t)flag;
        tile_cols[c.tile] = flag == 1 ? ncols : 0; // the column solver walks sparsely filled tiles column by column
        p_tiles[c.tile] = (uint8_t)(flag != 0);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// init: r <- b - A p (warm start) and, for the diag2 preconditioner, s <- z, sigma <- z.r
// (pressure_init.comp:45-83 + the init block of pressure_solver.rs:625-649)
template <int MODE>
__global__ void __launch_bounds__(PCG_THREADS) pcg_init_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                               const uint8_t *__restrict__ tile_active, const float *__restrict__ p,
                                                               float *__restrict__ r, float *__restrict__ s, PcgScalars *scal, float *partials) {
    __shared__ float sh[PCG_THREADS / 32];
    const TileCtx c = tile_ctx(g, t);
    float acc = 0.0f;
    if (tile_active[c.tile]) {
        int i = c.i;
        float4 pm = zero4(), p0 = zero4(), pp = zero4();
        if (c.valid) { pm = ld4(p + i - g.sz); p0 = ld4(p + i); }
#pragma unroll
        for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
            float left, right;
            x_neighbours(p, i, p0, c, left, right);
            if (c.valid) {
                pp = ld4(p + i + g.sz);
                const uchar4 code = ldcode(codes + i);
                const float4 ym = ld4(p + i - g.sy), yp = ld4(p + i + g.sy);
                float4 r4 = ld4(r + i);
                const float4 Ap = stencil_quad(code, p0, left, right, ym, yp, pm, pp);
                r4.x -= code.x ? Ap.x : 0.0f;
                r4.y -= code.y ? Ap.y : 0.0f;
                r4.z -= code.z ? Ap.z : 0.0f;
                r4.w -= code.w ? Ap.w : 0.0f;
                st4(r + i, r4);
                if (MODE == 0) {
                    const float4 z = make_float4(precond_diag2(r4.x, code.x), precond_diag2(r4.y, code.y), precond_diag2(r4.z, code.z),
                                                 precond_diag2(r4.w, code.w));
                    st4(s + i, z);
                    acc += (z.x * r4.x + z.y * r4.y) + (z.z * r4.z + z.w * r4.w);
                }
            }
            pm = p0;
            p0 = pp;
        }
    }
    if (MODE != 0) return;
    const float bs = block_sum(acc, sh);
    if (linear_tid() == 0) partials[c.tile] = bs;
    if (publish_and_elect(scal, t.ntiles)) {
        const double tot = final_sum(partials, t.ntiles);
        if (linear_tid() == 0) {
            scal->alpha = 0.0f; // RESULTMODE_INIT, pressure_reduce.comp:68-71
            scal->beta = 0.0f;
            scal->sigma = (float)tot;
            scal->ticket = 0u;
        }
    }
}

// One half-pass of the preconditioner as literally written with the LOD clamped to 0 (MODE 1 only):
// out = (in - sum over FLUID -x,-y,-z neighbours of in) / diag;  pass 1 also reduces out . r
// (pressure_apply_preconditioner.comp:36-82).  `in` obeys the zero invariant.  result_mode: 1 = INIT (sigma), 3 = BETA.
__global__ void __launch_bounds__(PCG_THREADS) pcg_precond_pass_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                                       const uint8_t *__restrict__ tile_active, const float *__restrict__ in,
                                                                       float *__restrict__ out, const float *__restrict__ r, int pass1,
                                                                       int result_mode, PcgScalars *scal, float *partials) {
    __shared__ float sh[PCG_THREADS / 32];
    if (scal->done) return;
    const TileCtx c = tile_ctx(g, t);
    float acc = 0.0f;
    if (tile_active[c.tile] && c.valid) {
        int i = c.i;
        for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
            const uchar4 code = ldcode(codes + i);
            const float4 c4 = ld4(in + i), ym = ld4(in + i - g.sy), zm = ld4(in + i - g.sz);
            const float xl = in[i - 1];
            float4 o;
            o.x = code.x ? (c4.x - ((xl + ym.x) + zm.x)) : 0.0f;
            o.y = code.y ? (c4.y - ((c4.x + ym.y) + zm.y)) : 0.0f;
            o.z = code.z ? (c4.z - ((c4.y + ym.z) + zm.z)) : 0.0f;
            o.w = code.w ? (c4.w - ((c4.z + ym.w) + zm.w)) : 0.0f;
            if (code.x & 7u) o.x /= (float)(code.x & 7u);
            if (code.y & 7u) o.y /= (float)(code.y & 7u);
            if (code.z & 7u) o.z /= (float)(code.z & 7u);
            if (code.w & 7u) o.w /= (float)(code.w & 7u);
            st4(out + i, o);
            if (pass1) {
                const float4 r4 = ld4(r + i);
                acc += (o.x * r4.x + o.y * r4.y) + (o.z * r4.z + o.w * r4.w);
            }
        }
    }
    if (!pass1) return;
    const float bs = block_sum(acc, sh);
    if (linear_tid() == 0) partials[c.tile] = bs;
    if (publish_and_elect(scal, t.ntiles)) {
        const double tot = final_sum(partials, t.ntiles);
        if (linear_tid() == 0) {
            const float zr = (float)tot;
            if (result_mode == 1) {
                scal->alpha = 0.0f;
                scal->beta = 0.0f;
                scal->sigma = zr;
            } else {
                scal->beta = guarded_div(zr, scal->sigma);
                scal->sigma = zr;
            }
            scal->ticket = 0u;
        }
    }
}

// dot: alpha <- sigma / (s . A s)   (pressure_apply_coeff.comp:19-30 + RESULTMODE_ALPHA)
__global__ void __launch_bounds__(PCG_THREADS) pcg_dot_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                              const uint8_t *__restrict__ tile_active, const float *__restrict__ s,
                                                              PcgScalars *scal, float *partials) {
    __shared__ float sh[PCG_THREADS / 32];
    if (scal->done) return;
    const TileCtx c = tile_ctx(g, t);
    float acc = 0.0f;
    if (tile_active[c.tile]) {
        int i = c.i;
        float4 sm = zero4(), s0 = zero4(), sp = zero4();
        if (c.valid) { sm = ld4(s + i - g.sz); s0 = ld4(s + i); }
#pragma unroll
        for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
            float left, right;
            x_neighbours(s, i, s0, c, left, right);
            if (c.valid) {
                sp = ld4(s + i + g.sz);
                const uchar4 code = ldcode(codes + i);
                const float4 ym = ld4(s + i - g.sy), yp = ld4(s + i + g.sy);
                const float4 As = stencil_quad(code, s0, left, right, ym, yp, sm, sp);
                acc += (s0.x * As.x + s0.y * As.y) + (s0.z * As.z + s0.w * As.w); // s == 0 off-fluid: no mask needed
            }
            sm = s0;
            s0 = sp;
        }
    }
    const float bs = block_sum(acc, sh);
    if (linear_tid() == 0) partials[c.tile] = bs;
    if (publish_and_elect(scal, t.ntiles)) {
        const double tot = final_sum(partials, t.ntiles);
        if (linear_tid() == 0) {
            scal->alpha = guarded_div(scal->sigma, (float)tot);
            scal->ticket = 0u;
        }
    }
}

// update: p += alpha s; r -= alpha A s; [MODE 0: beta, sigma <- z.r]; [WITH_ERR: max|r| -> statistics / done]
// (pressure_update_pressure_and_residual.comp:23-59, reduce MAX_ERROR pressure_reduce.comp:82-94, and for MODE 0
//  both preconditioner passes + reduce BETA)
template <int MODE, bool WITH_ERR>
__global__ void __launch_bounds__(PCG_THREADS) pcg_update_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                                 const uint8_t *__restrict__ tile_active, float *__restrict__ p,
                                                                 float *__restrict__ r, const float *__restrict__ s, PcgScalars *scal,
                                                                 float *partials, const StepParams *__restrict__ params, int which,
                                                                 int iteration, int max_iterations) {
    __shared__ float sh[PCG_THREADS / 32];
    if (scal->done) return;
    const float alpha = scal->alpha;
    const TileCtx c = tile_ctx(g, t);
    float acc = 0.0f, err = 0.0f;
    if (tile_active[c.tile]) {
        int i = c.i;
        float4 sm = zero4(), s0 = zero4(), sp = zero4();
        if (c.valid) { sm = ld4(s + i - g.sz); s0 = ld4(s + i); }
#pragma unroll
        for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
            float left, right;
            x_neighbours(s, i, s0, c, left, right);
            if (c.valid) {
                sp = ld4(s + i + g.sz);
                const uchar4 code = ldcode(codes + i);
                const float4 ym = ld4(s + i - g.sy), yp = ld4(s + i + g.sy);
                float4 p4 = ld4(p + i), r4 = ld4(r + i);
                const float4 As = stencil_quad(code, s0, left, right, ym, yp, sm, sp);
                p4.x += alpha * s0.x; p4.y += alpha * s0.y; p4.z += alpha * s0.z; p4.w += alpha * s0.w; // s == 0 off-fluid
                r4.x -= alpha * (code.x ? As.x : 0.0f);
                r4.y -= alpha * (code.y ? As.y : 0.0f);
                r4.z -= alpha * (code.z ? As.z : 0.0f);
                r4.w -= alpha * (code.w ? As.w : 0.0f);
                st4(p + i, p4);
                st4(r + i, r4);
                if (MODE == 0) // r == 0 off-fluid: no mask needed
                    acc += (precond_diag2(r4.x, code.x) * r4.x + precond_diag2(r4.y, code.y) * r4.y) +
                           (precond_diag2(r4.z, code.z) * r4.z + precond_diag2(r4.w, code.w) * r4.w);
                if (WITH_ERR) err = fmaxf(fmaxf(err, fmaxf(fabsf(r4.x), fabsf(r4.y))), fmaxf(fabsf(r4.z), fabsf(r4.w)));
            }
            sm = s0;
            s0 = sp;
        }
    }
    if (MODE != 0 && !WITH_ERR) return;
    float *pmax = partials + t.ntiles;
    if (MODE == 0) {
        const float bs = block_sum(acc, sh);
        if (linear_tid() == 0) partials[c.tile] = bs;
    }
    if (WITH_ERR) {
        const float bm = block_max(err, sh);
        if (linear_tid() == 0) pmax[c.tile] = bm;
    }
    if (publish_and_elect(scal, t.ntiles)) {
        double tot = 0.0;
        float e = 0.0f;
        if (MODE == 0) tot = final_sum(partials, t.ntiles);
        if (WITH_ERR) e = final_max(pmax, t.ntiles, sh);
        if (linear_tid() == 0) {
            if (WITH_ERR) {
                const float tol = params->tolerance[which];
                if (scal->num_iterations == 0 && (iteration == max_iterations || e < tol)) {
                    scal->max_error = e;
                    scal->num_iterations = iteration;
                    scal->done = 1;
                }
            }
            if (MODE == 0) {
                const float zr = (float)tot;
                scal->beta = guarded_div(zr, scal->sigma);
                scal->sigma = zr;
            }
            scal->ticket = 0u;
        }
    }
}

// search: s <- z + beta s (pressure_update_search.comp:13-24); MODE 0 recomputes z = r / diag^2.  r, z, s are 0
// off-fluid, so the update needs no mask.
template <int MODE>
__global__ void __launch_bounds__(PCG_THREADS) pcg_search_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                                 const uint8_t *__restrict__ tile_active, float *__restrict__ s,
                                                                 const float *__restrict__ r_or_z, const PcgScalars *scal) {
    if (scal->done) return;
    const float beta = scal->beta;
    const TileCtx c = tile_ctx(g, t);
    if (!tile_active[c.tile] || !c.valid) return;
    int i = c.i;
    float4 s4[PCG_TZ], r4[PCG_TZ];
    uchar4 code[PCG_TZ];
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k) {
        s4[k] = ld4(s + i + k * g.sz);
        r4[k] = ld4(r_or_z + i + k * g.sz);
        if (MODE == 0) code[k] = ldcode(codes + i + k * g.sz);
    }
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k) {
        float4 o;
        if (MODE == 0) {
            o.x = precond_diag2(r4[k].x, code[k].x) + beta * s4[k].x;
            o.y = precond_diag2(r4[k].y, code[k].y) + beta * s4[k].y;
            o.z = precond_diag2(r4[k].z, code[k].z) + beta * s4[k].z;
            o.w = precond_diag2(r4[k].w, code[k].w) + beta * s4[k].w;
        } else {
            o.x = r4[k].x + beta * s4[k].x;
            o.y = r4[k].y + beta * s4[k].y;
            o.z = r4[k].z + beta * s4[k].z;
            o.w = r4[k].w + beta * s4[k].w;
        }
        st4(s + i + k * g.sz, o);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Persistent solver: the WHOLE solve in one cooperative launch (diag2 preconditioner).
//
//   for every iteration:   phase A  s' = z + beta s  fused with  s'.A s'   (search + dot; s ping-pongs between two
//                                   buffers because neighbours' s' are recomputed from r, s, code instead of waited for)
//                          grid.sync -> alpha
//                          phase B  p += alpha s', r -= alpha A s', z.r, max|r|
//                          grid.sync -> beta, convergence
//
// Two grid-wide barriers per iteration instead of three kernel launches; every block sums the per-block partials
// redundantly in the same fixed order (bit-identical scalars everywhere, no broadcast, deterministic); converged solves
// stop at once instead of running out a recorded launch list.  Blocks walk the compacted list of active tiles with a
// fixed stride, so a tile is processed by the same SM in every phase.  24 B/cell/iteration of DRAM traffic at most
// (A: r, s, code in + s' out = 13; B: p, r, s', code in + p, r out = 21 ... minus what stays in the 50 MB L2 of an H100).
struct PcgSolveArgs {
    GridDim g;
    TileMap t;
    const uint8_t *codes;
    const int *tile_list;   // compacted active tiles
    const int *tile_list_flagged; // the same with bit 30 set on tiles that are at least 3/4 full (pcg_prepare_kernel)
    const int *num_active;
    unsigned *barrier;      // column solver: arrival counter of its grid-wide reductions (0 at the start of a solve)
    const int *col_list;    // column solver: compacted quad columns (4 cells x PCG_TZ planes) of the sparsely filled tiles, see pcg_solve_columns_kernel
    const int *num_cols;
    int code_slots;         // column solver: passes per thread whose code words stay in shared memory (see pass_codes)
    int p_slots;            // column solver: passes per thread whose p stays in shared memory (see p_slot); 0 on the other paths
    float *p, *r, *s0, *s1;
    PcgScalars *scal;
    float *partials;        // 3 x gridDim.x
    const StepParams *params;
    int which, max_iterations, check_frequency;
    SlabComm comm;          // world == 1: single GPU
    // the variable-density solve (pcg_solve_weighted_kernel): TagDensityWork's face coefficients, diagonal and 1 / D^2; null on the other paths
    const float *wbeta[3], *wdiag, *winv;
};

// ---- cross-GPU all-reduce through peer-mapped mailboxes (z-slab sharding, protocol in common.cuh) ----------------
// Every block of every rank polls its OWN mailbox until all `world` entries carry `seq` and adds them in rank order: identical
// result on every rank and in every block, no second barrier.  The system-scope fences of the post and the poll also publish /
// acquire the ghost planes pushed before.
__device__ __forceinline__ void mailbox_gather(const SlabComm &c, unsigned seq, double &sum, float &mx, double *sh_sum, float *sh_max, int *sh_dead) {
    const int tid = linear_tid();
    if (tid < c.world) {
        unsigned long long v0, v1;
        // the fence ending the poll is the acquire, by the threads that saw the flags (the block follows through the barrier below): it
        // orders the block's later loads of the ghost planes after the peers' pushes and drops stale L1 lines of this SM
        mailbox_poll(mailbox_entry(c.mailbox[c.rank], seq, tid), seq, MAILBOX_SPIN_LIMIT, sh_dead, v0, v1);
        sh_sum[tid] = (double)__uint_as_float((unsigned)v0);
        sh_max[tid] = __uint_as_float((unsigned)v1);
    }
    __syncthreads();
    double t = 0.0;
    float m = 0.0f;
    for (int k = 0; k < c.world; ++k) {
        t += sh_sum[k];
        m = fmaxf(m, sh_max[k]);
    }
    __syncthreads(); // the mailbox copies are reused by the next round
    sum = t;
    mx = m;
}
// Block 0 posts this rank's values; everything this GPU wrote before is ordered before the post by the preceding grid barrier (all
// blocks) and the post's system-scope fence.
__device__ __forceinline__ void comm_allreduce(const SlabComm &c, unsigned seq, double &sum, float &mx, double *sh_sum, float *sh_max,
                                               int *sh_dead) {
    const int tid = linear_tid();
    if (blockIdx.x == 0 && tid < c.world)
        mailbox_post(mailbox_entry(c.mailbox[tid], seq, c.rank), seq, __float_as_uint((float)sum), __float_as_uint(mx));
    mailbox_gather(c, seq, sum, mx, sh_sum, sh_max, sh_dead);
}


// every thread of every block returns the same value
__device__ __forceinline__ double grid_sum(cooperative_groups::grid_group &grid, float *partials, float acc, float *sh, double *shd) {
    const float bs = block_sum(acc, sh);
    if (linear_tid() == 0) partials[blockIdx.x] = bs;
    grid.sync();
    const double tot = final_sum(partials, gridDim.x);
    if (linear_tid() == 0) *shd = tot;
    __syncthreads();
    const double v = *shd;
    __syncthreads();
    return v;
}

// Sparsity (SKIP): the FLUID set of a real scene is a thin, ragged body -- at step 110 of the 256^3 dam break 64 % of the
// 128x8x4 tiles hold fluid but only 16 % of the 4x1x4 thread columns do (tools/sparsity.py).  A thread of a
// sparse tile therefore reads the six code words of its column first and touches p, r, s only on planes whose quad holds a
// FLUID cell: under the zero invariant everything it would have loaded, added or stored elsewhere is exactly 0, so the
// result is bit-identical to the dense form.  Tiles that are at least 3/4 full (flagged by pcg_prepare_kernel, the flag
// travels with the tile id) run the branch-free body, where no load waits for a code word: an all-fluid grid costs what it
// cost before (3.72 vs 3.69 ms per 256^3 solve), the dam break's solves drop from 2.87 to 2.17 ms (step 110).
// SKIP = false (solver path 4) keeps the branch-free body everywhere, for comparison.
__device__ __forceinline__ unsigned ldcw(const uint8_t *p) { return *reinterpret_cast<const unsigned *>(p); }
__device__ __forceinline__ uchar4 cw_code(unsigned w) {
    return make_uchar4((unsigned char)(w & 0xffu), (unsigned char)((w >> 8) & 0xffu), (unsigned char)((w >> 16) & 0xffu), (unsigned char)(w >> 24));
}
template <bool SKIP>
__device__ __forceinline__ float4 ld4w(const float *x, int i, unsigned w) {
    if (SKIP && w == 0u) return zero4();
    return ld4(x + i);
}

// The operator a tile body applies: the constant-density stencil (UnitOp: diagonal and preconditioner from the cell codes), or the
// variable-density one of liquids of different densities (WeightedOp: face coefficients, D and 1 / D^2 from launch_tag_density).  apply(code,
// i, ...) is A x for the quad at i, factors(code, i) the quad's preconditioner factors (z = r * factor).  With every coefficient 1 WeightedOp
// does, operation for operation, what stencil_quad does: the products with the coefficients are rounded on their own (exact for 1), the sums
// keep stencil_quad's order and D x - S is one fused multiply-add, as the compiler contracts it in stencil_quad (FFMA d, x, -S).
struct UnitOp {
    __device__ __forceinline__ UnitOp() {}
    __device__ __forceinline__ explicit UnitOp(const PcgSolveArgs &) {}
    __device__ __forceinline__ float4 apply(const uchar4 &code, int, const float4 &c, float left, float right, const float4 &ym, const float4 &yp,
                                            const float4 &zm, const float4 &zp) const {
        return stencil_quad(code, c, left, right, ym, yp, zm, zp);
    }
    __device__ __forceinline__ float4 factors(const uchar4 &code, int) const {
        return make_float4(c_inv_diag2[code.x & 7u], c_inv_diag2[code.y & 7u], c_inv_diag2[code.z & 7u], c_inv_diag2[code.w & 7u]);
    }
    __device__ __forceinline__ float4 factors_at(const uint8_t *__restrict__ codes, int i) const { return factors(ldcode(codes + i), i); }
    __device__ __forceinline__ float factor_at(const uint8_t *__restrict__ codes, int i) const { return c_inv_diag2[codes[i] & 7u]; }
};
struct WeightedOp {
    const PcgSolveArgs &a;
    __device__ __forceinline__ explicit WeightedOp(const PcgSolveArgs &args) : a(args) {}
    __device__ __forceinline__ float4 apply(const uchar4 &, int i, const float4 &c, float left, float right, const float4 &ym, const float4 &yp,
                                            const float4 &zm, const float4 &zp) const {
        const float *bx = a.wbeta[0], *by = a.wbeta[1], *bz = a.wbeta[2];
        const float4 d = ld4(a.wdiag + i), xp = ld4(bx + i), ymb = ld4(by + i - a.g.sy), ypb = ld4(by + i), zmb = ld4(bz + i - a.g.sz), zpb = ld4(bz + i);
        const float xm = bx[i - 1];
        float4 o;
        o.x = __fmaf_rn(d.x, c.x, -(((__fmul_rn(xm, left) + __fmul_rn(xp.x, c.y)) + (__fmul_rn(ymb.x, ym.x) + __fmul_rn(ypb.x, yp.x))) +
                                    (__fmul_rn(zmb.x, zm.x) + __fmul_rn(zpb.x, zp.x))));
        o.y = __fmaf_rn(d.y, c.y, -(((__fmul_rn(xp.x, c.x) + __fmul_rn(xp.y, c.z)) + (__fmul_rn(ymb.y, ym.y) + __fmul_rn(ypb.y, yp.y))) +
                                    (__fmul_rn(zmb.y, zm.y) + __fmul_rn(zpb.y, zp.y))));
        o.z = __fmaf_rn(d.z, c.z, -(((__fmul_rn(xp.y, c.y) + __fmul_rn(xp.z, c.w)) + (__fmul_rn(ymb.z, ym.z) + __fmul_rn(ypb.z, yp.z))) +
                                    (__fmul_rn(zmb.z, zm.z) + __fmul_rn(zpb.z, zp.z))));
        o.w = __fmaf_rn(d.w, c.w, -(((__fmul_rn(xp.z, c.z) + __fmul_rn(xp.w, right)) + (__fmul_rn(ymb.w, ym.w) + __fmul_rn(ypb.w, yp.w))) +
                                    (__fmul_rn(zmb.w, zm.w) + __fmul_rn(zpb.w, zp.w))));
        return o;
    }
    __device__ __forceinline__ float4 factors(const uchar4 &, int i) const { return ld4(a.winv + i); }
    __device__ __forceinline__ float4 factors_at(const uint8_t *__restrict__, int i) const { return ld4(a.winv + i); }
    __device__ __forceinline__ float factor_at(const uint8_t *__restrict__, int i) const { return a.winv[i]; }
};
// z = r * factor, and s' = z + beta s, under an operator
__device__ __forceinline__ float4 precond4(const float4 &r, const float4 &f) { return make_float4(r.x * f.x, r.y * f.y, r.z * f.z, r.w * f.w); }
__device__ __forceinline__ float4 snew4f(const float4 &r4, const float4 &s4, const float4 &f, float beta) {
    return make_float4(r4.x * f.x + beta * s4.x, r4.y * f.y + beta * s4.y, r4.z * f.z + beta * s4.z, r4.w * f.w + beta * s4.w);
}
template <bool SKIP, class Op>
__device__ __forceinline__ float4 snew4w_op(const Op &op, const float *r, const float *s, int i, float beta, unsigned w) {
    if (SKIP && w == 0u) return zero4();
    const float4 r4 = ld4(r + i), s4 = ld4(s + i);
    return snew4f(r4, s4, op.factors(cw_code(w), i), beta);
}
// NOTE: r, s, p are written by other blocks between grid barriers: no __restrict__/read-only (LDG.NC) path for them.
template <class Op> __device__ __forceinline__ float4 snew4_op(const Op &op, const float *r, const float *s, const uint8_t *__restrict__ codes, int i, float beta) {
    const float4 r4 = ld4(r + i), s4 = ld4(s + i);
    return snew4f(r4, s4, op.factors_at(codes, i), beta);
}
template <class Op> __device__ __forceinline__ float snew1_op(const Op &op, const float *r, const float *s, const uint8_t *__restrict__ codes, int i, float beta) {
    return r[i] * op.factor_at(codes, i) + beta * s[i];
}
// The same for WeightedOp, with the contraction of s' = r f + beta s written out: the one nvcc picks for UnitOp in the tile kernel of
// solver path 6 (read from its SASS), so that with every coefficient 1 the weighted solve is path 6 bit for bit.  fma(beta, s, r f) for
// the y-quads and for the .y, .z and .w cells of the own column's quads; fma(r, f, beta s) for their .x cells and for the single cells left
// and right of a row segment.
__device__ __forceinline__ float snew_rf(float r, float f, float beta, float s) { return __fmaf_rn(beta, s, __fmul_rn(r, f)); }
__device__ __forceinline__ float snew_bs(float r, float f, float beta, float s) { return __fmaf_rn(r, f, __fmul_rn(beta, s)); }
template <bool SKIP>
__device__ __forceinline__ float4 snew4w_op(const WeightedOp &op, const float *r, const float *s, int i, float beta, unsigned w) {
    if (SKIP && w == 0u) return zero4();
    const float4 r4 = ld4(r + i), s4 = ld4(s + i), f = op.factors(cw_code(w), i);
    return make_float4(snew_bs(r4.x, f.x, beta, s4.x), snew_rf(r4.y, f.y, beta, s4.y), snew_rf(r4.z, f.z, beta, s4.z), snew_rf(r4.w, f.w, beta, s4.w));
}
__device__ __forceinline__ float4 snew4_op(const WeightedOp &op, const float *r, const float *s, const uint8_t *__restrict__ codes, int i, float beta) {
    const float4 r4 = ld4(r + i), s4 = ld4(s + i), f = op.factors_at(codes, i);
    return make_float4(snew_rf(r4.x, f.x, beta, s4.x), snew_rf(r4.y, f.y, beta, s4.y), snew_rf(r4.z, f.z, beta, s4.z), snew_rf(r4.w, f.w, beta, s4.w));
}
__device__ __forceinline__ float snew1_op(const WeightedOp &op, const float *r, const float *s, const uint8_t *__restrict__ codes, int i, float beta) {
    return snew_bs(r[i], op.factor_at(codes, i), beta, s[i]);
}

// What the tile bodies need besides their operands.
struct TileEnv {
    GridDim g;
    const uint8_t *codes;
    bool sharded;
    int tz_first, tz_last, push;
    float *peer_r_lo, *peer_r_hi;
};

// Code words of the thread's column (planes -1 .. PCG_TZ)
__device__ __forceinline__ void load_column_codes(const TileEnv &e, const TileCtx &c, unsigned (&w)[PCG_TZ + 2]) {
#pragma unroll
    for (int k = 0; k < PCG_TZ + 2; ++k) w[k] = c.valid ? ldcw(e.codes + c.i + (k - 1) * e.g.sz) : 0u;
}

// A warp none of whose columns holds a FLUID cell in the tile's planes or in the two planes around them has nothing to do in any tile
// body: every value it would load is 0 (zero invariant), it would store nothing and add 0 to the partial sums -- and nobody else
// depends on it (x-neighbours live in the same warp, y / z neighbours are read from memory).  In a dam break most warps of the
// "active" tiles along the free surface are like that: skipping them at warp granularity removes the body's instruction skeleton,
// which is what the sparse solve is bound by.
__device__ __forceinline__ bool warp_has_no_fluid(const unsigned (&w)[PCG_TZ + 2]) {
    unsigned any = 0;
#pragma unroll
    for (int k = 0; k < PCG_TZ + 2; ++k) any |= w[k];
    return !__any_sync(0xffffffffu, any != 0u);
}

// r <- b - A p, partial z.r  (pressure_init.comp:45-83).  ps (column solver, see p_slot): the thread's slot that keeps its own p quads
// on chip for the rest of the solve, filled here with the quads of planes 0 .. PCG_TZ - 1.
template <bool SKIP, class Op = UnitOp>
__device__ __forceinline__ void init_tile(const TileEnv &e, const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], const float *p, float *r, float &acc,
                                          float4 *ps = nullptr, const Op &op = Op()) {
    const GridDim &g = e.g;
    int i = c.i;
    float4 pm = zero4(), p0 = zero4(), pp = zero4();
    if (c.valid) { pm = ld4w<SKIP>(p, i - g.sz, w[0]); p0 = ld4w<SKIP>(p, i, w[1]); }
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
        float left = __shfl_up_sync(0xffffffffu, p0.w, 1), right = __shfl_down_sync(0xffffffffu, p0.x, 1);
        if (ps) ps[k * PCG_THREADS] = p0;
        if (c.valid) pp = ld4w<SKIP>(p, i + g.sz, w[k + 2]);
        if (c.valid && (!SKIP || w[k + 1] != 0u)) {
            if (c.first) left = p[i - 1];
            if (c.last) right = p[i + 4];
            const uchar4 code = cw_code(w[k + 1]);
            const float4 ym = ld4(p + i - g.sy), yp = ld4(p + i + g.sy);
            float4 r4 = ld4(r + i);
            const float4 Ap = op.apply(code, i, p0, left, right, ym, yp, pm, pp);
            r4.x -= code.x ? Ap.x : 0.0f;
            r4.y -= code.y ? Ap.y : 0.0f;
            r4.z -= code.z ? Ap.z : 0.0f;
            r4.w -= code.w ? Ap.w : 0.0f;
            st4(r + i, r4);
            if (e.sharded) { // boundary planes go straight into the neighbour's ghost planes (NVLink P2P stores)
                if (k == 0 && c.tz == e.tz_first && e.peer_r_lo) st4(e.peer_r_lo + i + e.push, r4);
                if (k == PCG_TZ - 1 && c.tz == e.tz_last && e.peer_r_hi) st4(e.peer_r_hi + i - e.push, r4);
            }
            const float4 z = precond4(r4, op.factors(code, i));
            acc += (z.x * r4.x + z.y * r4.y) + (z.z * r4.z + z.w * r4.w);
        }
        pm = p0;
        p0 = pp;
    }
}

// phase A: s' = z + beta s (pressure_update_search.comp) fused with s'.A s' (pressure_apply_coeff.comp)
template <bool SKIP, class Op = UnitOp>
__device__ __forceinline__ void search_tile(const TileEnv &e, const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], const float *r, const float *s_in,
                                            float *s_out, float beta, float &acc, const Op &op = Op()) {
    const GridDim &g = e.g;
    const uint8_t *codes = e.codes;
    int i = c.i;
    float4 cm = zero4(), c0 = zero4(), cp = zero4();
    if (c.valid) {
        cm = snew4w_op<SKIP>(op, r, s_in, i - g.sz, beta, w[0]);
        c0 = snew4w_op<SKIP>(op, r, s_in, i, beta, w[1]);
        // ghost plane below an owned boundary tile: keep the recomputed s' so that phase B and the next
        // iteration find it locally (bit-identical to what the neighbour computes for its own plane)
        if (e.sharded && c.tz == e.tz_first && (!SKIP || w[0] != 0u)) st4(s_out + i - g.sz, cm);
    }
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
        float left = __shfl_up_sync(0xffffffffu, c0.w, 1), right = __shfl_down_sync(0xffffffffu, c0.x, 1);
        if (c.valid) cp = snew4w_op<SKIP>(op, r, s_in, i + g.sz, beta, w[k + 2]);
        const bool act = c.valid && (!SKIP || w[k + 1] != 0u);
        float4 ym = zero4(), yp = zero4();
        if (act) { // operand loads only: short enough to be predicated, so that the planes' loads can overlap
            ym = snew4_op(op, r, s_in, codes, i - g.sy, beta);
            yp = snew4_op(op, r, s_in, codes, i + g.sy, beta);
        }
        if (act) {
            if (c.first) left = snew1_op(op, r, s_in, codes, i - 1, beta);
            if (c.last) right = snew1_op(op, r, s_in, codes, i + 4, beta);
            const float4 As = op.apply(cw_code(w[k + 1]), i, c0, left, right, ym, yp, cm, cp);
            acc += (c0.x * As.x + c0.y * As.y) + (c0.z * As.z + c0.w * As.w);
            st4(s_out + i, c0);
        }
        if (c.valid && e.sharded && k == PCG_TZ - 1 && c.tz == e.tz_last && (!SKIP || w[k + 2] != 0u)) st4(s_out + i + g.sz, cp);
        cm = c0;
        c0 = cp;
    }
}

// phase B: p += alpha s', r -= alpha A s' (pressure_update_pressure_and_residual.comp), partial z.r and max|r|.  With a p slot (ps) the
// thread's p quads are read and updated there instead of in memory.
template <bool SKIP, class Op = UnitOp>
__device__ __forceinline__ void update_tile(const TileEnv &e, const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], const float *s, float *p, float *r,
                                            float alpha, float &acc, float &err, float4 *ps = nullptr, const Op &op = Op()) {
    const GridDim &g = e.g;
    int i = c.i;
    float4 sm = zero4(), s0 = zero4(), sp = zero4();
    if (c.valid) { sm = ld4w<SKIP>(s, i - g.sz, w[0]); s0 = ld4w<SKIP>(s, i, w[1]); }
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
        float left = __shfl_up_sync(0xffffffffu, s0.w, 1), right = __shfl_down_sync(0xffffffffu, s0.x, 1);
        if (c.valid) sp = ld4w<SKIP>(s, i + g.sz, w[k + 2]);
        const bool act = c.valid && (!SKIP || w[k + 1] != 0u);
        float4 ym = zero4(), yp = zero4(), p4 = zero4(), r4 = zero4();
        if (act) {
            ym = ld4(s + i - g.sy);
            yp = ld4(s + i + g.sy);
            p4 = ps ? ps[k * PCG_THREADS] : ld4(p + i);
            r4 = ld4(r + i);
        }
        if (act) {
            if (c.first) left = s[i - 1];
            if (c.last) right = s[i + 4];
            const uchar4 code = cw_code(w[k + 1]);
            const float4 As = op.apply(code, i, s0, left, right, ym, yp, sm, sp);
            p4.x += alpha * s0.x; p4.y += alpha * s0.y; p4.z += alpha * s0.z; p4.w += alpha * s0.w;
            r4.x -= alpha * (code.x ? As.x : 0.0f);
            r4.y -= alpha * (code.y ? As.y : 0.0f);
            r4.z -= alpha * (code.z ? As.z : 0.0f);
            r4.w -= alpha * (code.w ? As.w : 0.0f);
            if (ps) ps[k * PCG_THREADS] = p4;
            else st4(p + i, p4);
            st4(r + i, r4);
            if (e.sharded) {
                if (k == 0 && c.tz == e.tz_first && e.peer_r_lo) st4(e.peer_r_lo + i + e.push, r4);
                if (k == PCG_TZ - 1 && c.tz == e.tz_last && e.peer_r_hi) st4(e.peer_r_hi + i - e.push, r4);
            }
            const float4 z = precond4(r4, op.factors(code, i));
            acc += (z.x * r4.x + z.y * r4.y) + (z.z * r4.z + z.w * r4.w);
            err = fmaxf(fmaxf(err, fmaxf(fabsf(r4.x), fabsf(r4.y))), fmaxf(fabsf(r4.z), fabsf(r4.w)));
        }
        sm = s0;
        s0 = sp;
    }
}

// End of a solve: the slotted p quads go to memory on exactly the planes update_tile stores, so that p is still written only inside
// the active tiles (the sparse set-up and PressureField::p_tiles rely on that)
template <bool SKIP>
__device__ __forceinline__ void store_p_tile(const TileEnv &e, const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], float *p, const float4 *ps) {
#pragma unroll
    for (int k = 0; k < PCG_TZ; ++k)
        if (c.valid && (!SKIP || w[k + 1] != 0u)) st4(p + c.i + k * e.g.sz, ps[k * PCG_THREADS]);
}

// Formed from the kernel parameters where a phase needs it, not kept in the walkers: values derived from parameters are re-read from the
// constant bank instead of holding registers through the whole solve (a TileEnv member made the TMA kernel spill three times as much).
__device__ __forceinline__ TileEnv make_tile_env(const PcgSolveArgs &a) {
    const SlabComm &cm = a.comm;
    TileEnv e;
    e.g = a.g;
    e.codes = a.codes;
    e.sharded = cm.world > 1;
    // slab geometry: tile layers tz_first..tz_last are owned; the planes just outside are ghost planes fed by the neighbours
    e.tz_first = cm.halo / PCG_TZ;
    e.tz_last = a.t.tiles_z - 1 - cm.halo / PCG_TZ;
    e.push = cm.owned_nz * a.g.sz; // index distance between an owned boundary plane and its image in the neighbour
    e.peer_r_lo = cm.peer_r[0];
    e.peer_r_hi = cm.peer_r[1];
    return e;
}

// ---------------------------------------------------------------------------------------------------------------
// The solve, written once for the three persistent kernels.  A kernel hands it
//   a walker:  init(acc), search(it, beta, acc) = phase A, update(it, alpha, acc, err) = phase B -- the kernel's share of the work of a
//              phase --, store_p(), which writes back the p kept on chip (column solver), and each_tile(f), which calls f(c) for every
//              tile (and column) of that share;
//   a reducer: the grid-wide sums, on z-slab ranks followed by or fused with the all-rank round: open(psum) and close(psum) are empty
//              rounds, sum(psum, acc, tot) a sum, sum_max(psum, pmax, acc, err, tot, gmax) a sum and a maximum.
// Partial buffers (gridDim.x floats each): init on 1, phase A on 0, phase B on 1 + 2 for the maximum (a fast block never overwrites
// what a slow one still reads), the empty rounds of a sharded solve on 0.
struct SlabRounds {
    const SlabComm &c;
    unsigned seq; // all-reduce rounds done so far
    double *sh_sum;
    float *sh_max;
    int *sh_dead; // set when a peer did not answer (or a TMA transaction was lost): the solve ends with done = -1
};

template <class Walker, class Reducer>
__device__ __forceinline__ void pcg_solve(const PcgSolveArgs &a, Walker &wk, Reducer &rd) {
    SlabRounds &sr = rd.sr;
    const bool sharded = sr.c.world > 1;
    // partial buffers, formed where they are used: three pointers kept across the loop cost registers the phases need
    auto partials = [&](int k) { return a.partials + k * gridDim.x; };
    if (linear_tid() == 0) *sr.sh_dead = 0;
    if (sharded) sr.seq = *sr.c.seq;
    __syncthreads();
    // First thing a sharded solve does: one empty round.  A rank that has entered its solver kernel has finished its prepare kernel
    // (stream order), which zeroes r and p off-fluid in ALL its planes -- ghost planes included -- with read-modify-write; without the
    // round a fast neighbour's first ghost-plane push could land in the middle of that and be lost.
    if (sharded) rd.open(partials(0));

    // ---- init: r <- b - A p, sigma <- z.r (pressure_init.comp:45-83, pressure_solver.rs:625-649); s stays 0
    float acc = 0.0f;
    wk.init(acc);
    double tot;
    rd.sum(partials(1), acc, tot);
    float sigma = (float)tot;
    float alpha = 0.0f, beta = 0.0f, max_error = 0.0f, gmax;
    int num_iterations = 0;

    for (int it = 0;; ++it) {
        acc = 0.0f;
        wk.search(it, beta, acc);
        rd.sum(partials(0), acc, tot);
        alpha = guarded_div(sigma, (float)tot); // RESULTMODE_ALPHA, pressure_reduce.comp:73-75

        acc = 0.0f;
        float err = 0.0f;
        wk.update(it, alpha, acc, err);
        rd.sum_max(partials(1), partials(2), acc, err, tot, gmax);
        const float zr = (float)tot;
        const bool with_err = (a.max_iterations == it) || (it > 0 && it % a.check_frequency == 0); // pressure_solver.rs:676-677
        if (with_err) {
            const float tol = a.params->tolerance[a.which];
            if (a.max_iterations == it || gmax < tol) { // pressure_reduce.comp:82-94: statistics + stop everything
                max_error = gmax;
                num_iterations = it;
                break;
            }
        }
        beta = guarded_div(zr, sigma); // RESULTMODE_BETA, pressure_reduce.comp:77-80
        sigma = zr;
    }
    wk.store_p();
    if (sharded) {
        // hand the boundary planes of the solution to the neighbours (warm start of their next init, pressure gradient across the slab
        // face), then one more round so that nobody leaves before its ghost planes are complete
        float *const peer_p_lo = sr.c.peer_p[a.which][0], *const peer_p_hi = sr.c.peer_p[a.which][1];
        const TileEnv e = make_tile_env(a);
        wk.each_tile([&](const TileCtx &c) {
            if (!c.valid) return;
            if (c.tz == e.tz_first && peer_p_lo) st4(peer_p_lo + c.i + e.push, ld4(a.p + c.i));
            if (c.tz == e.tz_last && peer_p_hi) {
                const int i = c.i + (PCG_TZ - 1) * e.g.sz;
                st4(peer_p_hi + i - e.push, ld4(a.p + i));
            }
        });
        rd.close(partials(0));
        if (blockIdx.x == 0 && linear_tid() == 0) *sr.c.seq = sr.seq;
    }
    if (blockIdx.x == 0 && linear_tid() == 0) {
        a.scal->alpha = alpha;
        a.scal->beta = beta;
        a.scal->sigma = sigma;
        a.scal->max_error = max_error;
        a.scal->num_iterations = num_iterations;
        a.scal->done = *sr.sh_dead ? -1 : 1;
    }
}

// Reducer of the tile and TMA kernels: cooperative_groups grid barrier, every block re-reads the partials (block_sum / final_sum /
// final_max); on z-slab ranks a mailbox round after it.
struct SyncReduce {
    SlabRounds sr;
    cooperative_groups::grid_group grid;
    float *sh;
    double *shd;
    float *shf;
    __device__ __forceinline__ void open(float *) {
        double none = 0.0;
        float nomax = 0.0f;
        comm_allreduce(sr.c, ++sr.seq, none, nomax, sr.sh_sum, sr.sh_max, sr.sh_dead);
    }
    __device__ __forceinline__ void close(float *psum) {
        grid.sync(); // every block's pushes before block 0 posts
        open(psum);
    }
    __device__ __forceinline__ void sum(float *psum, float acc, double &tot) {
        tot = grid_sum(grid, psum, acc, sh, shd);
        float nomax = 0.0f;
        if (sr.c.world > 1) comm_allreduce(sr.c, ++sr.seq, tot, nomax, sr.sh_sum, sr.sh_max, sr.sh_dead);
    }
    __device__ __forceinline__ void sum_max(float *psum, float *pmax, float acc, float err, double &tot, float &gmax) {
        {
            const float bm = block_max(err, sh);
            if (linear_tid() == 0) pmax[blockIdx.x] = bm;
        }
        tot = grid_sum(grid, psum, acc, sh, shd); // the barrier inside also publishes pmax
        {
            const float em = final_max(pmax, gridDim.x, sh);
            if (linear_tid() == 0) *shf = em;
            __syncthreads();
            gmax = *shf;
            __syncthreads();
        }
        if (sr.c.world > 1) comm_allreduce(sr.c, ++sr.seq, tot, gmax, sr.sh_sum, sr.sh_max, sr.sh_dead);
    }
};

// Tiles are dealt round robin: all blocks sweep the volume as one front, so the z-neighbour planes of a layer of tiles are still
// in L2 when the next layer needs them.  (Grouping sparse tiles into equal-"work" slots was tried and is slower: a tile pass
// costs a chain of dependent memory latencies whatever its fill.)  The id of the next tile is fetched one pass ahead.
#define PCG_FOR_EACH_TILE(tile)                                                                                                      \
    for (int li_ = blockIdx.x, tile = li_ < nact ? a.tile_list_flagged[li_] : 0, next_ = 0; li_ < nact; li_ += gridDim.x, tile = next_) \
        if ((next_ = li_ + (int)gridDim.x < nact ? a.tile_list_flagged[li_ + gridDim.x] : 0), true)

// Phases of the register-marching kernels (tile and column solver): Walk::passes(fill, body) calls body(c, w, sparse, ps) for every pass
// of the thread -- a tile or a column with its code words w; sparse: std::true_type for the sparse body; ps: the pass's p slot or null --
// and fill is set in the first phase of a solve.
// Op: the operator of the tile bodies (UnitOp, or WeightedOp for the variable-density solve).
template <class Walk, class Op = UnitOp>
struct MarchWalker : Walk {
    __device__ __forceinline__ void init(float &acc) const {
        const TileEnv e = make_tile_env(this->a);
        const Op op(this->a);
        this->passes(true, [&](const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], auto sparse, float4 *ps) {
            init_tile<decltype(sparse)::value>(e, c, w, this->a.p, this->a.r, acc, ps, op);
        });
    }
    __device__ __forceinline__ void search(int it, float beta, float &acc) const {
        const float *s_in = (it & 1) ? this->a.s1 : this->a.s0;
        float *s_out = (it & 1) ? this->a.s0 : this->a.s1;
        const TileEnv e = make_tile_env(this->a);
        const Op op(this->a);
        this->passes(false, [&](const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], auto sparse, float4 *) {
            search_tile<decltype(sparse)::value>(e, c, w, this->a.r, s_in, s_out, beta, acc, op);
        });
    }
    __device__ __forceinline__ void update(int it, float alpha, float &acc, float &err) const {
        const float *s = (it & 1) ? this->a.s0 : this->a.s1;
        const TileEnv e = make_tile_env(this->a);
        const Op op(this->a);
        this->passes(false, [&](const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], auto sparse, float4 *ps) {
            update_tile<decltype(sparse)::value>(e, c, w, s, this->a.p, this->a.r, alpha, acc, err, ps, op);
        });
    }
    __device__ __forceinline__ void store_p() const {
        if (this->a.p_slots == 0) return;
        const TileEnv e = make_tile_env(this->a);
        this->passes(false, [&](const TileCtx &c, const unsigned (&w)[PCG_TZ + 2], auto sparse, float4 *ps) {
            if (ps) store_p_tile<decltype(sparse)::value>(e, c, w, this->a.p, ps);
        });
    }
};

// Work of the tile kernel: the active tiles; SKIP: sparse bodies in tiles that are not flagged dense, and warps without fluid skipped
template <bool SKIP>
struct TileWalk {
    const PcgSolveArgs &a;
    int nact;
    template <class F> __device__ __forceinline__ void each_tile(F f) const {
        PCG_FOR_EACH_TILE(tile) f(tile_ctx_id(a.g, a.t, tile & (TILE_DENSE_BIT - 1)));
    }
    template <class Body> __device__ __forceinline__ void passes(bool, Body body) const {
        const TileEnv e = make_tile_env(a);
        PCG_FOR_EACH_TILE(tile) {
            const TileCtx c = tile_ctx_id(e.g, a.t, tile & (TILE_DENSE_BIT - 1));
            unsigned w[PCG_TZ + 2];
            load_column_codes(e, c, w);
            if (SKIP && warp_has_no_fluid(w)) continue;
            if (!SKIP || (tile & TILE_DENSE_BIT)) body(c, w, std::false_type{}, nullptr);
            else body(c, w, std::true_type{}, nullptr);
        }
    }
};

template <bool SKIP>
__global__ void __launch_bounds__(PCG_THREADS, 4) pcg_solve_persistent_kernel(PcgSolveArgs a) {
    __shared__ float sh[PCG_THREADS / 32];
    __shared__ double shd;
    __shared__ float shf;
    __shared__ double sh_csum[SLAB_MAX_WORLD];
    __shared__ float sh_cmax[SLAB_MAX_WORLD];
    __shared__ int sh_dead;
    MarchWalker<TileWalk<SKIP>> wk{{a, *a.num_active}};
    SyncReduce rd{{a.comm, 0u, sh_csum, sh_cmax, &sh_dead}, cooperative_groups::this_grid(), sh, &shd, &shf};
    pcg_solve(a, wk, rd);
}

// The variable-density velocity solve of liquids of different densities: the tile kernel of solver path 6 (same tiles, sparse bodies, blocks,
// reductions and recurrence) with the weighted operator.
__global__ void __launch_bounds__(PCG_THREADS, 4) pcg_solve_weighted_kernel(PcgSolveArgs a) {
    __shared__ float sh[PCG_THREADS / 32];
    __shared__ double shd;
    __shared__ float shf;
    __shared__ double sh_csum[SLAB_MAX_WORLD];
    __shared__ float sh_cmax[SLAB_MAX_WORLD];
    __shared__ int sh_dead;
    MarchWalker<TileWalk<true>, WeightedOp> wk{{a, *a.num_active}};
    SyncReduce rd{{a.comm, 0u, sh_csum, sh_cmax, &sh_dead}, cooperative_groups::this_grid(), sh, &shd, &shf};
    pcg_solve(a, wk, rd);
}

// ---------------------------------------------------------------------------------------------------------------
// The column solver's grid-wide reduction (grid_reduce.cuh) on a z-slab rank, fused with the cross-GPU all-reduce: the block that arrives LAST on the local counter (atomicAdd returns
// the ticket) adds this GPU's partials and publishes the total straight into every rank's mailbox -- its own included -- and ALL blocks of all
// ranks wait on their own mailbox only.  The local "everybody waits for the counter, everybody re-reads the partials" step is off the critical
// path: a round is one local arrival + one NVLink store + one poll (round 1: grid barrier, then block 0 publishes, then everybody polls).
// Ordering of the ghost planes pushed during the phase: their writers release on the counter (gpu scope), the last block acquires, fences at
// system scope and only then stores the flags; a reader polls the flag, fences at system scope and passes the block barrier.
template <bool WITH_MAX>
__device__ __forceinline__ void grid_allreduce(const SlabComm &c, unsigned seq, unsigned *counter, unsigned &round, float *psum, float *pmax, float acc, float err,
                                               ReduceScratch &sc, double *sh_sum, float *sh_max, int *sh_dead, int *sh_last, double &tot, float &gmax) {
    if (publish_and_arrive<WITH_MAX, true>(counter, round, psum, pmax, acc, err, sc, sh_last)) { // this block adds the GPU's partials and posts
        double t;
        float mm;
        read_partials<WITH_MAX>(psum, pmax, sc, t, mm);
        // the post's system-scope fence covers everything this GPU wrote before, cumulatively through the ticket
        if (linear_tid() < c.world) mailbox_post(mailbox_entry(c.mailbox[linear_tid()], seq, c.rank), seq, __float_as_uint((float)t), __float_as_uint(mm));
    }
    mailbox_gather(c, seq, tot, gmax, sh_sum, sh_max, sh_dead);
}

// Reducer of the column solver: grid_reduce on one GPU, grid_allreduce on z-slab ranks.
struct CounterReduce {
    SlabRounds sr;
    unsigned *counter;
    unsigned round; // counter rounds done by this solve (the counter is 0 at its start)
    ReduceScratch &sc;
    int *sh_last;
    template <bool WITH_MAX> __device__ __forceinline__ void reduce(float *psum, float *pmax, float acc, float err, double &tot, float &gmax) {
        if (sr.c.world > 1) grid_allreduce<WITH_MAX>(sr.c, ++sr.seq, counter, round, psum, pmax, acc, err, sc, sr.sh_sum, sr.sh_max, sr.sh_dead, sh_last, tot, gmax);
        else grid_reduce<WITH_MAX>(counter, round, psum, pmax, acc, err, sc, tot, gmax);
    }
    __device__ __forceinline__ void open(float *psum) {
        double none;
        float nomax;
        reduce<false>(psum, nullptr, 0.0f, 0.0f, none, nomax);
    }
    __device__ __forceinline__ void close(float *psum) { open(psum); } // the counter's release orders the pushes before the post
    __device__ __forceinline__ void sum(float *psum, float acc, double &tot) {
        float nomax;
        reduce<false>(psum, nullptr, acc, 0.0f, tot, nomax);
    }
    __device__ __forceinline__ void sum_max(float *psum, float *pmax, float acc, float err, double &tot, float &gmax) { reduce<true>(psum, pmax, acc, err, tot, gmax); }
};

// ---------------------------------------------------------------------------------------------------------------
// Column solver (default on one GPU): the persistent solver with a work list that follows the fluid.
//
// Why: at step 110 of the 256^3 dam break (12.6 % of the cells FLUID) the sparsely filled tiles of the tile kernel have only 4-5 of 32
// lanes doing anything -- a warp pays the
// whole instruction skeleton of a plane as soon as ONE of its lanes has a FLUID quad there.  The solve is bound by that skeleton and by
// the 4-5 sequential tile passes per block and phase, not by bandwidth.
// Here tiles that are at least 3/4 full still run the branch-free tile body (an all-fluid grid costs what it cost: the roofline
// microbench), but everything else is flattened into ONE list of active quad columns (4 cells x PCG_TZ planes, ascending index:
// deterministic) and dealt to the warps 32 columns at a time: every lane has work, x-adjacent quads still sit in adjacent lanes
// (coalesced loads), and a phase is ~one pass.  The column body IS the sparse tile body with "first" and "last" set: the x-neighbours
// come from memory instead of the neighbouring lanes, so every cell sees the operands it saw before and the iterates agree with the
// tile kernel up to the grouping of the partial sums.  Same phases, barriers, reductions and statistics as pcg_solve_persistent_kernel.
__global__ void __launch_bounds__(PCG_THREADS) pcg_column_fill_kernel(GridDim g, TileMap t, const uint8_t *__restrict__ codes,
                                                                      const uint8_t *__restrict__ tile_active, const int *__restrict__ col_offset,
                                                                      int tile_lo, int tile_hi, int *__restrict__ col_list) {
    __shared__ int sh_warp[PCG_THREADS / 32];
    const TileCtx c = tile_ctx(g, t);
    if (c.tile < tile_lo || c.tile >= tile_hi || tile_active[c.tile] != 1) return; // block-uniform; [tile_lo, tile_hi): the owned tiles of a slab
    bool active = false;
    if (c.valid) {
#pragma unroll
        for (int k = 0; k < PCG_TZ; ++k) active = active || ldcw(codes + c.i + k * g.sz) != 0u;
    }
    const int tid = linear_tid(), lane = tid & 31, w = tid >> 5;
    const unsigned ballot = __ballot_sync(0xffffffffu, active);
    if (lane == 0) sh_warp[w] = __popc(ballot);
    __syncthreads();
    int before = 0;
    for (int k = 0; k < w; ++k) before += sh_warp[k];
    if (active) col_list[col_offset[c.tile] + before + __popc(ballot & ((1u << lane) - 1u))] = c.i; // ascending thread order inside a tile
}

// One block: compacts the tiles the tile loop walks (all active tiles, or only the dense ones when the columns take the rest) and
// scans the per-tile column counts.  Deterministic (ascending tile id).  Runs after the prepare kernel: clears the set-up flags of the
// solve (dense_flags[0], dense_flags[1 + which]) when it is given them.
__global__ void __launch_bounds__(1024) pcg_compact_kernel(const uint8_t *__restrict__ tile_active, const int *__restrict__ tile_cols, int tile_lo, int ntiles,
                                                           int dense_only, int *__restrict__ tile_list, int *__restrict__ tile_list_flagged,
                                                           int *__restrict__ num_active, int *__restrict__ col_offset, int *__restrict__ num_cols,
                                                           int *__restrict__ dense_flags, int which) {
    __shared__ int sh[1024], shc[1024];
    __shared__ int carry, carry_c;
    if (threadIdx.x == 0) { carry = 0; carry_c = 0; }
    if (dense_flags && threadIdx.x == 0) {
        dense_flags[0] = 0;
        dense_flags[1 + which] = 0;
    }
    __syncthreads();
    for (int base = tile_lo; base < ntiles; base += 1024) { // [tile_lo, ntiles): the owned tiles of a slab, else all
        const int idx = base + threadIdx.x;
        const int flag = idx < ntiles ? tile_active[idx] : 0;
        const int v = (dense_only ? flag == 2 : flag != 0) ? 1 : 0;
        const int nc = dense_only && idx < ntiles ? tile_cols[idx] : 0;
        sh[threadIdx.x] = v;
        shc[threadIdx.x] = nc;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            const int tmp = threadIdx.x >= o ? sh[threadIdx.x - o] : 0, tmpc = threadIdx.x >= o ? shc[threadIdx.x - o] : 0;
            __syncthreads();
            sh[threadIdx.x] += tmp;
            shc[threadIdx.x] += tmpc;
            __syncthreads();
        }
        const int incl = sh[threadIdx.x], inclc = shc[threadIdx.x];
        if (v) {
            tile_list[carry + incl - 1] = idx;
            tile_list_flagged[carry + incl - 1] = idx | (flag == 2 ? TILE_DENSE_BIT : 0);
        }
        if (dense_only && idx < ntiles) col_offset[idx] = carry_c + inclc - nc;
        __syncthreads();
        if (threadIdx.x == 1023) { carry += incl; carry_c += inclc; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { *num_active = carry; *num_cols = carry_c; }
}

// 32 consecutive list entries per warp and pass; the index of the next pass is fetched one pass ahead.  All 32 lanes stay in the loop
// (the bodies shuffle): lanes beyond the end of the list carry valid = false.
#define PCG_FOR_EACH_COLUMN(c)                                                                                                            \
    for (int cb_ = warp_first, ci_ = cb_ + lane < ncols ? a.col_list[cb_ + lane] : -1, cn_ = -1; cb_ < ncols; cb_ += col_stride, ci_ = cn_) \
        if ((cn_ = cb_ + col_stride + lane < ncols ? a.col_list[cb_ + col_stride + lane] : -1), true)                                      \
            if (const TileCtx c = column_ctx(ci_, sz); true)
__device__ __forceinline__ TileCtx column_ctx(int i, int sz) {
    TileCtx c;
    c.tile = 0;
    c.valid = i >= 0;
    c.first = true; // x-neighbours from memory: the neighbouring lanes hold unrelated columns
    c.last = true;
    c.i = i >= 0 ? i : 0;
    c.tz = (c.i / sz) / PCG_TZ; // tile layer of the column (z-slab ranks: which columns touch a ghost plane)
    return c;
}

// Code words of a thread's pass (tile or column) number `pass` of a phase.  They do not change during a solve, but the acquire of every
// grid-wide reduction invalidates L1, so reloading them costs an L2 round trip at the head of every pass, before any operand load can
// start.  The first phase (init) loads them and keeps the first `slots` passes of each thread in a slot of dynamic shared memory that
// only this thread uses ([pass][plane][thread]: conflict-free); later phases read them from there.  Passes beyond the slots reload.
__device__ __forceinline__ void pass_codes(const TileEnv &e, const TileCtx &c, unsigned (&w)[PCG_TZ + 2], unsigned *sh_cw, int slots, int pass, bool fill) {
    if (pass >= slots) {
        load_column_codes(e, c, w);
        return;
    }
    unsigned *slot = sh_cw + pass * (PCG_TZ + 2) * PCG_THREADS + linear_tid();
    if (fill) {
        load_column_codes(e, c, w);
#pragma unroll
        for (int k = 0; k < PCG_TZ + 2; ++k) slot[k * PCG_THREADS] = w[k];
    } else {
#pragma unroll
        for (int k = 0; k < PCG_TZ + 2; ++k) w[k] = slot[k * PCG_THREADS];
    }
}
constexpr int PCG_CODE_SLOT_BYTES = (PCG_TZ + 2) * PCG_THREADS * 4; // 6 KB

// p of a thread's pass (tile or column) number `pass`, for the whole solve.  Nobody else reads a cell's p during a solve: init reads the
// neighbours' p before any of it changes, phase B reads and writes the thread's own quads only, and only the closing push of a z-slab rank
// (no p slots there) reads p after the loop.  So init keeps the p quads of its own planes in a slot of dynamic shared memory that only
// this thread uses ([pass][plane][thread] float4: conflict-free), phase B updates them there, and store_p writes them back once at the
// end: 24 instead of 32 B of own-cell traffic per cell and iteration, and one operand load less in phase B.  Passes beyond the slots
// keep p in memory.
// The p slots follow the code slots (sh_cw: 6 KB slots, so 16-byte aligned).
__device__ __forceinline__ float4 *p_slot(unsigned *sh_cw, const PcgSolveArgs &a, int pass) {
    return pass < a.p_slots ? reinterpret_cast<float4 *>(sh_cw + a.code_slots * (PCG_TZ + 2) * PCG_THREADS) + pass * PCG_TZ * PCG_THREADS + linear_tid()
                            : nullptr;
}
constexpr int PCG_P_SLOT_BYTES = PCG_TZ * PCG_THREADS * 16; // 16 KB

// Slots per block, code words and p (PressureSolver searches down from this pair for one that keeps the resident blocks per SM).  2 + 2 =
// 44 KB per block ran the 256^3 dam break fastest of the pairs measured: 153.3 steps/s, 150.0-150.2 for 4 + 2 and 2 + 3, 139.3-140.1 for
// 8 or 4 code slots without p slots (H100 SXM at 700 W, profiles/h100_pcg_onchip.json).  12 code slots alone (72 KB) shrink L1 to ~28 KB
// and ran 112.9 against 126.7 steps/s for 8 (400 W, profiles/h100_pcg_setup.json).
constexpr int PCG_CODE_SLOTS = 2, PCG_P_SLOTS = 2;
constexpr int PCG_MAX_CODE_SLOTS = 8, PCG_MAX_P_SLOTS = 4; // largest counts the test hooks may ask for

// Work of the column solver: the dense tiles by the tile body, then the column list by the sparse body, code words and p of the first
// passes kept in shared memory (pass_codes, p_slot)
struct ColumnWalk {
    const PcgSolveArgs &a;
    int nact, ncols;
    int lane, col_stride, warp_first, sz;
    unsigned *sh_cw;
    template <class F> __device__ __forceinline__ void each_tile(F f) const {
        PCG_FOR_EACH_TILE(tile) f(tile_ctx_id(a.g, a.t, tile & (TILE_DENSE_BIT - 1)));
        PCG_FOR_EACH_COLUMN(c) f(c);
    }
    template <class Body> __device__ __forceinline__ void passes(bool fill, Body body) const {
        const TileEnv e = make_tile_env(a);
        int pass = 0;
        PCG_FOR_EACH_TILE(tile) {
            const TileCtx c = tile_ctx_id(e.g, a.t, tile & (TILE_DENSE_BIT - 1));
            unsigned w[PCG_TZ + 2];
            pass_codes(e, c, w, sh_cw, a.code_slots, pass, fill);
            body(c, w, std::false_type{}, p_slot(sh_cw, a, pass++));
        }
        PCG_FOR_EACH_COLUMN(c) {
            unsigned w[PCG_TZ + 2];
            pass_codes(e, c, w, sh_cw, a.code_slots, pass, fill);
            body(c, w, std::true_type{}, p_slot(sh_cw, a, pass++));
        }
    }
};

// Three resident blocks per SM (up to 85 registers): for sm_90a, a four-block bound (64 registers) spills the column body to local memory,
// and on an H100 SXM (700 W limit) the 256^3 dam break runs 100.9 instead of 97.7 steps/s with three blocks (profiles/h100_choices.json).
__global__ void __launch_bounds__(PCG_THREADS, 3) pcg_solve_columns_kernel(PcgSolveArgs a) {
    extern __shared__ unsigned sh_cw[]; // a.code_slots x (PCG_TZ + 2) x PCG_THREADS code words, then a.p_slots x PCG_TZ x PCG_THREADS p quads
    __shared__ ReduceScratch sc;
    __shared__ double sh_csum[SLAB_MAX_WORLD];
    __shared__ float sh_cmax[SLAB_MAX_WORLD];
    __shared__ int sh_dead, sh_last;
    // Tiles are dealt to the blocks from block 0 upwards, columns to the warps from the LAST warp of the last block downwards: when there are
    // fewer dense tiles than blocks (or a remainder), the blocks without a tile take the columns first and a phase is one pass, not two.
    const int col_stride = gridDim.x * PCG_THREADS;
    const int warp_first = col_stride - 32 - (blockIdx.x * (PCG_THREADS / 32) + (linear_tid() >> 5)) * 32;
    MarchWalker<ColumnWalk> wk{{a, *a.num_active, *a.num_cols, linear_tid() & 31, col_stride, warp_first, a.g.sz, sh_cw}};
    CounterReduce rd{{a.comm, 0u, sh_csum, sh_cmax, &sh_dead}, a.barrier, 0u, sc, &sh_last};
    pcg_solve(a, wk, rd);
}

// ---------------------------------------------------------------------------------------------------------------
// TMA-tiled variant of the persistent solver (grids whose x extent is a multiple of 128 cells).
//
// Same algorithm, phases, barriers and multi-GPU protocol as pcg_solve_persistent_kernel; what changes is how a tile's
// stencil operands reach the SM.  One elected thread issues 3-D tensor-map bulk loads (cp.async.bulk.tensor.3d, SASS
// UTMALDG) of the tile PLUS its halo -- box (128+8) x (8+2) x (4+2) of r, s and (128+32) x 10 x 6 of the codes -- into
// shared memory; completion is an mbarrier transaction count, out-of-range parts of a box are zero-filled by the TMA
// unit (== SOLID / 0, the same convention as the padded arrays).  Phase A then evaluates s' = z + beta s ONCE per box
// cell in shared memory (the register-marching kernel re-derives it for the y and z neighbours of every thread: 9
// global vector loads per 4 cells and plane instead of 3 here), and both phases take all seven stencil operands from
// shared memory.  Three blocks per SM, each single-buffered: while one block waits for its boxes the others compute.
constexpr int TMA_BX = 136, TMA_BY = 10, TMA_BZ = 6; // float box: x0-4 .. x0+131, y0-1 .. y0+8, z0-1 .. z0+4
constexpr int TMA_CX = 160;                           // code box:  x0-16 .. x0+143 (inner extent must be a multiple of 16 bytes)
constexpr int TMA_F32_BYTES = TMA_BX * TMA_BY * TMA_BZ * 4; // 32,640 (multiple of 128)
constexpr int TMA_U8_BYTES = TMA_CX * TMA_BY * TMA_BZ;      // 9,600
constexpr int TMA_SMEM_BYTES = 2 * TMA_F32_BYTES + TMA_U8_BYTES; // 74,880 per block
constexpr long long TMA_SPIN_LIMIT = 1LL << 26;

struct PcgTmaMaps {
    CUtensorMap r, s0, s1, codes;
};

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// r and s are written with ordinary (generic-proxy) stores and later read by TMA (async proxy): every writer orders its
// global stores before later async-proxy accesses with this fence, then the grid barrier makes them visible device-wide.
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// all threads: wait for the boxes of the current tile; a lost transaction ends the solve instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity, int *sh_dead) {
    long long spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > TMA_SPIN_LIMIT) { *sh_dead = 1; break; }
    }
}

// Work of the TMA kernel: the active tiles, operands staged in shared memory by tensor-map box loads.  Every phase ends with
// fence_proxy_async_global(): its generic-proxy stores of r, s and p come before the async-proxy (TMA) reads after the grid barrier.
struct TmaWalk {
    const PcgSolveArgs &a;
    const PcgTmaMaps &maps;
    int nact;
    float *shR, *shS;
    uint8_t *shC;
    uint64_t *bar;
    int *sh_dead;
    unsigned parity; // of the mbarrier phase the next box load completes
    template <class F> __device__ __forceinline__ void each_tile(F f) const {
        for (int li = blockIdx.x; li < nact; li += gridDim.x) f(tile_ctx_id(a.g, a.t, a.tile_list[li]));
    }
    __device__ __forceinline__ void store_p() const {} // p stays in memory
    // init as in the register-marching kernels (runs once, plain loads)
    __device__ __forceinline__ void init(float &acc) const {
        const TileEnv e = make_tile_env(a);
        each_tile([&](const TileCtx &c) {
            unsigned w[PCG_TZ + 2];
            load_column_codes(e, c, w);
            init_tile<false>(e, c, w, a.p, a.r, acc);
        });
        fence_proxy_async_global();
    }
    // phase A: boxes of r, s, codes -> smem; s' once per box cell; s'.A s' from smem
    __device__ __forceinline__ void search(int it, float beta, float &acc) {
        const TileEnv e = make_tile_env(a);
        const GridDim &g = e.g;
        const TileMap &t = a.t;
        const CUtensorMap *map_in = (it & 1) ? &maps.s1 : &maps.s0;
        float *s_out = (it & 1) ? a.s0 : a.s1;
        const int tid = linear_tid(), lx = threadIdx.x, ly = threadIdx.y;
        // offsets of this thread's quad inside a box: row (ly + 1), columns 4 + 4 lx .. 7 + 4 lx
        const int qoff = (ly + 1) * TMA_BX + 4 + 4 * lx;
        const int coff = (ly + 1) * TMA_CX + 16 + 4 * lx;
        constexpr int PLANE = TMA_BX * TMA_BY, CPLANE = TMA_CX * TMA_BY;
        for (int li = blockIdx.x; li < nact; li += gridDim.x) {
            const TileCtx c = tile_ctx_id(g, t, a.tile_list[li]);
            const int tile = c.tile, tx = tile % t.tiles_x, rest = tile / t.tiles_x, ty = rest % t.tiles_y, tz = rest / t.tiles_y;
            const int x0 = tx * 128, y0 = ty * 8, z0 = tz * PCG_TZ;
            __syncthreads(); // every thread is done with the previous tile's boxes
            if (tid == 0) {
                fence_proxy_async_global();
                fence_proxy_async(); // generic-proxy reads of the boxes above happen-before the async writes below
                mbar_arrive_expect_tx(bar, 2 * TMA_F32_BYTES + TMA_U8_BYTES);
                tma_load_3d(shR, &maps.r, x0 - 4, y0 - 1, z0 - 1, bar);
                tma_load_3d(shS, map_in, x0 - 4, y0 - 1, z0 - 1, bar);
                tma_load_3d(shC, &maps.codes, x0 - 16, y0 - 1, z0 - 1, bar);
            }
            mbar_wait(bar, parity, sh_dead);
            parity ^= 1u;
            // s' = z + beta s for the whole box, in place over s (60 rows x 34 quads)
            for (int qd = tid; qd < TMA_BY * TMA_BZ * (TMA_BX / 4); qd += PCG_THREADS) {
                const int row = qd / (TMA_BX / 4), col = (qd - row * (TMA_BX / 4)) * 4;
                const float4 r4 = *reinterpret_cast<const float4 *>(shR + row * TMA_BX + col);
                float4 s4 = *reinterpret_cast<const float4 *>(shS + row * TMA_BX + col);
                const uchar4 cd = *reinterpret_cast<const uchar4 *>(shC + row * TMA_CX + col + 12);
                s4.x = precond_diag2(r4.x, cd.x) + beta * s4.x;
                s4.y = precond_diag2(r4.y, cd.y) + beta * s4.y;
                s4.z = precond_diag2(r4.z, cd.z) + beta * s4.z;
                s4.w = precond_diag2(r4.w, cd.w) + beta * s4.w;
                *reinterpret_cast<float4 *>(shS + row * TMA_BX + col) = s4;
            }
            __syncthreads();
            int i = c.i;
            if (e.sharded && c.tz == e.tz_first) st4(s_out + i - g.sz, *reinterpret_cast<const float4 *>(shS + qoff));
#pragma unroll
            for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
                const float *S = shS + (k + 1) * PLANE + qoff;
                const float4 c0 = *reinterpret_cast<const float4 *>(S);
                const float4 ym = *reinterpret_cast<const float4 *>(S - TMA_BX), yp = *reinterpret_cast<const float4 *>(S + TMA_BX);
                const float4 zm = *reinterpret_cast<const float4 *>(S - PLANE), zp = *reinterpret_cast<const float4 *>(S + PLANE);
                const uchar4 code = *reinterpret_cast<const uchar4 *>(shC + (k + 1) * CPLANE + coff);
                const float4 As = stencil_quad(code, c0, S[-1], S[4], ym, yp, zm, zp);
                acc += (c0.x * As.x + c0.y * As.y) + (c0.z * As.z + c0.w * As.w);
                st4(s_out + i, c0);
                if (e.sharded && k == PCG_TZ - 1 && c.tz == e.tz_last) st4(s_out + i + g.sz, zp);
            }
        }
        fence_proxy_async_global();
    }
    // phase B: box of s' -> smem (p, r, codes: plain loads issued before the wait); update; z.r, max|r|
    __device__ __forceinline__ void update(int it, float alpha, float &acc, float &err) {
        const TileEnv e = make_tile_env(a);
        const GridDim &g = e.g;
        const TileMap &t = a.t;
        const CUtensorMap *map_out = (it & 1) ? &maps.s0 : &maps.s1;
        const uint8_t *__restrict__ codes = e.codes;
        const int tid = linear_tid(), lx = threadIdx.x, ly = threadIdx.y;
        const int qoff = (ly + 1) * TMA_BX + 4 + 4 * lx;
        constexpr int PLANE = TMA_BX * TMA_BY;
        for (int li = blockIdx.x; li < nact; li += gridDim.x) {
            const TileCtx c = tile_ctx_id(g, t, a.tile_list[li]);
            const int tile = c.tile, tx = tile % t.tiles_x, rest = tile / t.tiles_x, ty = rest % t.tiles_y, tz = rest / t.tiles_y;
            __syncthreads();
            if (tid == 0) {
                fence_proxy_async_global();
                fence_proxy_async();
                mbar_arrive_expect_tx(bar, TMA_F32_BYTES);
                tma_load_3d(shS, map_out, tx * 128 - 4, ty * 8 - 1, tz * PCG_TZ - 1, bar);
            }
            float4 p4[PCG_TZ], r4[PCG_TZ];
            uchar4 code[PCG_TZ];
#pragma unroll
            for (int k = 0; k < PCG_TZ; ++k) { // independent of the box: in flight while the TMA load lands
                p4[k] = ld4(a.p + c.i + k * g.sz);
                r4[k] = ld4(a.r + c.i + k * g.sz);
                code[k] = ldcode(codes + c.i + k * g.sz);
            }
            mbar_wait(bar, parity, sh_dead);
            parity ^= 1u;
            int i = c.i;
#pragma unroll
            for (int k = 0; k < PCG_TZ; ++k, i += g.sz) {
                const float *S = shS + (k + 1) * PLANE + qoff;
                const float4 s0 = *reinterpret_cast<const float4 *>(S);
                const float4 ym = *reinterpret_cast<const float4 *>(S - TMA_BX), yp = *reinterpret_cast<const float4 *>(S + TMA_BX);
                const float4 zm = *reinterpret_cast<const float4 *>(S - PLANE), zp = *reinterpret_cast<const float4 *>(S + PLANE);
                const float4 As = stencil_quad(code[k], s0, S[-1], S[4], ym, yp, zm, zp);
                float4 pq = p4[k], rq = r4[k];
                pq.x += alpha * s0.x; pq.y += alpha * s0.y; pq.z += alpha * s0.z; pq.w += alpha * s0.w;
                rq.x -= alpha * (code[k].x ? As.x : 0.0f);
                rq.y -= alpha * (code[k].y ? As.y : 0.0f);
                rq.z -= alpha * (code[k].z ? As.z : 0.0f);
                rq.w -= alpha * (code[k].w ? As.w : 0.0f);
                st4(a.p + i, pq);
                st4(a.r + i, rq);
                if (e.sharded) {
                    if (k == 0 && c.tz == e.tz_first && e.peer_r_lo) st4(e.peer_r_lo + i + e.push, rq);
                    if (k == PCG_TZ - 1 && c.tz == e.tz_last && e.peer_r_hi) st4(e.peer_r_hi + i - e.push, rq);
                }
                acc += (precond_diag2(rq.x, code[k].x) * rq.x + precond_diag2(rq.y, code[k].y) * rq.y) +
                       (precond_diag2(rq.z, code[k].z) * rq.z + precond_diag2(rq.w, code[k].w) * rq.w);
                err = fmaxf(fmaxf(err, fmaxf(fabsf(rq.x), fabsf(rq.y))), fmaxf(fabsf(rq.z), fabsf(rq.w)));
            }
        }
        fence_proxy_async_global();
    }
};

__global__ void __launch_bounds__(PCG_THREADS, 3) pcg_solve_tma_kernel(const __grid_constant__ PcgSolveArgs a, const __grid_constant__ PcgTmaMaps maps) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bar;
    __shared__ float sh[PCG_THREADS / 32];
    __shared__ double shd;
    __shared__ float shf;
    __shared__ double sh_csum[SLAB_MAX_WORLD];
    __shared__ float sh_cmax[SLAB_MAX_WORLD];
    __shared__ int sh_dead;
    if (linear_tid() == 0) {
        mbar_init(&bar, 1);
        fence_proxy_async(); // make the initialised barrier visible to the async (TMA) proxy (the solve's first block barrier follows)
    }
    TmaWalk wk{a, maps, *a.num_active, reinterpret_cast<float *>(smem_raw), reinterpret_cast<float *>(smem_raw + TMA_F32_BYTES),
               smem_raw + 2 * TMA_F32_BYTES, &bar, &sh_dead, 0u};
    SyncReduce rd{{a.comm, 0u, sh_csum, sh_cmax, &sh_dead}, cooperative_groups::this_grid(), sh, &shd, &shf};
    pcg_solve(a, wk, rd);
}
#undef PCG_FOR_EACH_COLUMN
#undef PCG_FOR_EACH_TILE

__global__ void pcg_reset_scalars_kernel(PcgScalars *scal, unsigned *barrier) {
    if (barrier) *barrier = 0u;
    scal->alpha = 0.0f; scal->beta = 0.0f; scal->sigma = 0.0f;
    scal->max_error = 0.0f; scal->num_iterations = 0; scal->done = 0; scal->ticket = 0u;
}

} // namespace

// ---------------------------------------------------------------------------------------------------------------
PressureField::PressureField(const GridDim &grid, const SolverConfig &cfg, void *external_volume) : config(cfg) {
    if (external_volume) pressure_.place(grid, external_volume);
    else pressure_.alloc(grid);
    BLUB_CUDA_CHECK(cudaMalloc(&scalars, sizeof(PcgScalars)));
    BLUB_CUDA_CHECK(cudaMemset(scalars, 0, sizeof(PcgScalars)));
    const int ntiles = make_tilemap(grid).ntiles;
    BLUB_CUDA_CHECK(cudaMalloc(&p_tiles, (size_t)ntiles));
    BLUB_CUDA_CHECK(cudaMemset(p_tiles, 0, (size_t)ntiles));
    BLUB_CUDA_CHECK(cudaMallocHost(&pinned_, sizeof(float) * 2 * NUM_PRESSURE_ERROR_BUFFER));
    ring_.resize(NUM_PRESSURE_ERROR_BUFFER);
    for (int k = 0; k < NUM_PRESSURE_ERROR_BUFFER; ++k) {
        BLUB_CUDA_CHECK(cudaEventCreateWithFlags(&ring_[k].event, cudaEventDisableTiming));
        ring_[k].host = pinned_ + 2 * k;
        ring_[k].in_flight = false;
        unused_.push_back(k);
    }
}

PressureField::~PressureField() {
    for (auto &p : ring_) cudaEventDestroy(p.event);
    if (pinned_) cudaFreeHost(pinned_);
    if (scalars) cudaFree(scalars);
    if (p_tiles) cudaFree(p_tiles);
    pressure_.release();
}

void PressureField::retrieve_new_error_samples() {
    while (!pending_.empty()) {
        Pending &pb = ring_[pending_.front()];
        if (cudaEventQuery(pb.event) != cudaSuccess) break; // oldest first; later ones cannot be done either
        SolverStatisticSample smp;
        // "We always deal with pressure * dt / density": scale the error by dt for display (pressure_solver.rs:158-163)
        smp.error = pb.host[0] * pb.dt;
        smp.iteration_count = (int32_t)pb.host[1];
        stats.push_back(smp);
        while (stats.size() > SOLVER_STATISTIC_HISTORY_LENGTH) stats.pop_front();
        pb.in_flight = false;
        unused_.push_back(pending_.front());
        pending_.pop_front();
    }
}

namespace {
__global__ void pcg_export_stats_kernel(const PcgScalars *scal, float *out) {
    out[0] = scal->max_error;
    out[1] = (float)scal->num_iterations;
}
} // namespace

void PressureField::enqueue_error_buffer_read(cudaStream_t stream, float simulation_delta) {
    if (unused_.empty()) return; // "No more error buffer available for async copy" (pressure_solver.rs:188-190)
    int k = unused_.back();
    unused_.pop_back();
    Pending &pb = ring_[k];
    // pinned host memory is device-accessible under UVA: the 8-byte result is stored straight into it
    BLUB_LAUNCH(pcg_export_stats_kernel, 1, 1, 0, stream, scalars, pb.host);
    BLUB_CUDA_CHECK(cudaEventRecord(pb.event, stream));
    pb.dt = simulation_delta;
    pb.in_flight = true;
    pending_.push_back(k);
}

void PressureField::read_last_solve(cudaStream_t stream, float *max_error, int *iterations) {
    PcgScalars h;
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&h, scalars, sizeof(h), cudaMemcpyDeviceToHost, stream));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream));
    *max_error = h.max_error;
    *iterations = h.num_iterations;
}

void PressureField::read_last_scalars(cudaStream_t stream, float out[3]) {
    PcgScalars h;
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&h, scalars, sizeof(h), cudaMemcpyDeviceToHost, stream));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream));
    out[0] = h.alpha;
    out[1] = h.beta;
    out[2] = h.sigma;
}

namespace {
// 3-D tensor maps (x fastest).  The encoder lives in libcuda; it is fetched through the runtime so that libblubcore.so
// does not link against the driver library.
bool encode_map(PFN_cuTensorMapEncodeTiled encode, CUtensorMap *map, CUtensorMapDataType type, size_t elem, void *base, const GridDim &g, unsigned bx,
                unsigned by, unsigned bz) {
    const cuuint64_t dims[3] = {(cuuint64_t)g.nx, (cuuint64_t)g.ny, (cuuint64_t)g.nz};
    const cuuint64_t strides[2] = {(cuuint64_t)g.nx * elem, (cuuint64_t)g.nx * g.ny * elem};
    const cuuint32_t box[3] = {bx, by, bz}, estr[3] = {1, 1, 1};
    return encode(map, type, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
bool make_tma_maps(const GridDim &g, float *r, float *s0, float *s1, uint8_t *codes, PcgTmaMaps &m) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
        cudaGetLastError();
        return false;
    }
    auto encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
    return encode_map(encode, &m.r, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, r, g, TMA_BX, TMA_BY, TMA_BZ) &&
           encode_map(encode, &m.s0, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, s0, g, TMA_BX, TMA_BY, TMA_BZ) &&
           encode_map(encode, &m.s1, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, s1, g, TMA_BX, TMA_BY, TMA_BZ) &&
           encode_map(encode, &m.codes, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, codes, g, TMA_CX, TMA_BY, TMA_BZ);
}
} // namespace

PressureSolver::PressureSolver(const GridDim &grid, void *external_residual) : grid_(grid) {
    if (external_residual) residual_.place(grid, external_residual);
    else residual_.alloc(grid);
    search_.alloc(grid);
    aux_.alloc(grid);
    aux_temp_.alloc(grid);
    codes_.alloc(grid);
    TileMap t = make_tilemap(grid);
    num_blocks_ = t.ntiles;
    BLUB_CUDA_CHECK(cudaMalloc(&partials_, sizeof(float) * (2 * (size_t)num_blocks_ + 8192)));
    BLUB_CUDA_CHECK(cudaMalloc(&tile_active_, (size_t)num_blocks_));
    BLUB_CUDA_CHECK(cudaMemset(tile_active_, 0, (size_t)num_blocks_));
    BLUB_CUDA_CHECK(cudaMalloc(&tile_list_, sizeof(int) * (2 * (size_t)num_blocks_ + 1))); // ids | count | ids with the dense flag
    num_active_ = tile_list_ + num_blocks_;
    BLUB_CUDA_CHECK(cudaMalloc(&dense_flags_, 3 * sizeof(int)));
    BLUB_CUDA_CHECK(cudaMemset(dense_flags_, 1, 3 * sizeof(int))); // the first solve of each field prepares every tile
    // persistent cooperative solver: as many blocks as can be co-resident
    int dev = 0, coop = 0, sms = 0, per_sm = 0;
    BLUB_CUDA_CHECK(cudaGetDevice(&dev));
    BLUB_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    BLUB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pcg_solve_persistent_kernel<true>, PCG_THREADS, 0));
    persistent_blocks_ = coop ? sms * per_sm : 0;
    if (persistent_blocks_ > 2048) persistent_blocks_ = 2048;
    const char *env = std::getenv("BLUB_PCG");
    if (env && std::string(env) == "multikernel") persistent_blocks_ = 0;
    // TMA-tiled variant: 128-cell-wide tiles, tensor maps over r, both s buffers and the codes
    tma_blocks_ = 0;
    if (persistent_blocks_ > 0 && grid.nx % 128 == 0 && !(env && std::string(env) == "registers")) {
        tma_maps_ = new PcgTmaMaps();
        if (make_tma_maps(grid, residual_.ptr, search_.ptr, aux_.ptr, codes_.ptr, *static_cast<PcgTmaMaps *>(tma_maps_))) {
            BLUB_CUDA_CHECK(cudaFuncSetAttribute(pcg_solve_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TMA_SMEM_BYTES));
            int per = 0;
            BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, pcg_solve_tma_kernel, PCG_THREADS, TMA_SMEM_BYTES));
            tma_blocks_ = sms * per;
        }
    }
    use_tma = tma_blocks_ > 0 && env && std::string(env) == "tma";
    // column solver (default on one GPU): list of the active quad columns of the sparsely filled tiles
    column_blocks_ = 0;
    if (persistent_blocks_ > 0) {
        const size_t max_cols = (size_t)t.ntiles * PCG_THREADS;
        BLUB_CUDA_CHECK(cudaMalloc(&tile_cols_, sizeof(int) * (2 * (size_t)t.ntiles + 2))); // counts | offsets | total
        BLUB_CUDA_CHECK(cudaMemset(tile_cols_, 0, sizeof(int) * (2 * (size_t)t.ntiles + 2)));
        BLUB_CUDA_CHECK(cudaMalloc(&col_list_, sizeof(int) * max_cols));
        BLUB_CUDA_CHECK(cudaMalloc(&barrier_, 256));
        BLUB_CUDA_CHECK(cudaMemset(barrier_, 0, 256));
        int per = 0;
        BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, pcg_solve_columns_kernel, PCG_THREADS, 0));
        column_blocks_ = sms * per;
        if (column_blocks_ > 2048) column_blocks_ = 2048;
        // as many code and p slots as leave the number of resident blocks (and with it the grouping of the partial sums) unchanged: p slots
        // are kept longest, code slots give way first.  The attribute is the largest size any solver asks for, so that solvers with
        // different slot counts can live in one process.  Test hooks BLUB_PCG_CODE_SLOTS=N (0..8) and BLUB_PCG_P_SLOTS=N (0..4) start the
        // search at N: the grid and every sum stay the same, passes beyond the slots reload their code words / keep p in memory.
        auto hook = [](const char *name, int dflt, int most) {
            const char *v = std::getenv(name);
            return v && v[0] >= '0' && v[0] <= '0' + most && v[1] == '\0' ? v[0] - '0' : dflt;
        };
        const int max_code = hook("BLUB_PCG_CODE_SLOTS", PCG_CODE_SLOTS, PCG_MAX_CODE_SLOTS), max_p = hook("BLUB_PCG_P_SLOTS", PCG_P_SLOTS, PCG_MAX_P_SLOTS);
        BLUB_CUDA_CHECK(cudaFuncSetAttribute(pcg_solve_columns_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             PCG_MAX_CODE_SLOTS * PCG_CODE_SLOT_BYTES + PCG_MAX_P_SLOTS * PCG_P_SLOT_BYTES));
        code_slots_ = p_slots_ = 0;
        for (int ps = max_p, found = 0; ps >= 0 && !found; --ps) {
            for (int cs = max_code; cs >= 0; --cs) {
                int per_slots = 0;
                BLUB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_slots, pcg_solve_columns_kernel, PCG_THREADS,
                                                                              cs * PCG_CODE_SLOT_BYTES + ps * PCG_P_SLOT_BYTES));
                if (per_slots == per) {
                    code_slots_ = cs;
                    p_slots_ = ps;
                    found = 1;
                    break;
                }
            }
        }
    }
    use_columns = column_blocks_ > 0 && !(env && std::string(env) == "tiles");
    // BLUB_PCG_SETUP=dense (test hook): the column solver prepares every tile on every solve, as the other paths do -- the comparator
    // of the set-up sized by the fluid, with the same arithmetic
    const char *setup_env = std::getenv("BLUB_PCG_SETUP");
    dense_setup_ = setup_env && std::string(setup_env) == "dense";
}

PressureSolver::~PressureSolver() {
    residual_.release(); search_.release(); aux_.release(); aux_temp_.release(); codes_.release();
    if (partials_) cudaFree(partials_);
    if (tile_active_) cudaFree(tile_active_);
    if (tile_list_) cudaFree(tile_list_);
    if (tile_cols_) cudaFree(tile_cols_);
    if (col_list_) cudaFree(col_list_);
    if (barrier_) cudaFree(barrier_);
    if (dense_flags_) cudaFree(dense_flags_);
    delete static_cast<PcgTmaMaps *>(tma_maps_);
}

void PressureSolver::prepare_dense_next(cudaStream_t stream) { BLUB_CUDA_CHECK(cudaMemsetAsync(dense_flags_, 1, 3 * sizeof(int), stream)); }

void PressureSolver::read_work(cudaStream_t stream, uint32_t out[4]) {
    const TileMap t = make_tilemap(grid_);
    int tiles = 0, cols = 0;
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&tiles, num_active_, sizeof(int), cudaMemcpyDeviceToHost, stream));
    if (tile_cols_) BLUB_CUDA_CHECK(cudaMemcpyAsync(&cols, tile_cols_ + 2 * t.ntiles, sizeof(int), cudaMemcpyDeviceToHost, stream));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream));
    out[0] = (uint32_t)tiles;
    out[1] = (uint32_t)cols;
    out[2] = (uint32_t)(4 * t.bx * t.by * PCG_TZ);
    out[3] = (uint32_t)(4 * PCG_TZ);
}

void PressureSolver::set_path(int path) {
    // validate first: a refused request leaves the solver exactly as it was
    if (path < 0 || path > 6 || path == 3 || path == 5)
        throw std::invalid_argument("solver path must be 0 (three kernels), 1 (persistent, default), 2 (TMA-staged), 4 (dense) or 6 (tiles only)");
    if (path == 2 && !tma_available()) throw std::invalid_argument("TMA solver needs nx % 128 == 0 and cooperative launch");
    use_persistent = path != 0;
    use_tma = path == 2;
    use_dense = path == 4;
    use_columns = path == 1;
}

void PressureSolver::solve(cudaStream_t stream, PressureField &field, int which, const int8_t *marker, const StepParams *dparams,
                           const Quirks &quirks, const TagDensityWork *weights) {
    const GridDim g = grid_;
    const TileMap t = make_tilemap(g);
    const dim3 grid = t.grid(), block = t.block();
    float *p = field.pressure(), *r = residual_.ptr, *s = search_.ptr;
    const uint8_t *st = codes_.ptr;
    const uint8_t *ta = tile_active_;
    PcgScalars *scal = field.scalars;
    const int mode = quirks.precond_mode;
    const int max_it = field.config.max_num_iterations;
    const int freq = field.config.error_check_frequency > 0 ? field.config.error_check_frequency : 1;

    field.touched = true; // the volume is zero-initialised at allocation (pressure_solver.rs:601-603)

    if (comm.world > 1 && !(mode == 0 && persistent_blocks_ > 0 && use_persistent))
        throw std::invalid_argument("the z-slab sharded solve needs the persistent solver with precond_mode 0");
    // the variable-density solve runs pcg_solve_weighted_kernel whatever the solver path
    if (weights && (mode != 0 || persistent_blocks_ == 0 || comm.world > 1))
        throw std::invalid_argument("the variable-density solve needs cooperative launch, precond_mode 0 and one GPU");
    const bool persistent = weights || (mode == 0 && persistent_blocks_ > 0 && use_persistent);
    // Set-up sized by the fluid: only the tiles that hold FLUID now or were active in the previous solve (p: this field's previous
    // solve) are prepared.  Kept to the single-GPU column solver, whose kernels write inside the active tiles only; everything else,
    // the first solve and any solve after a write from outside the step prepare every tile, and so does the solve after them.
    // The choice is made on the device (dense_flags_), so that a captured step graph follows writes from outside the step.
    const bool columns = !weights && persistent && use_columns && column_blocks_ > 0 && !use_tma && !use_dense;
    int *const flags = columns && comm.world == 1 && !dense_setup_ ? dense_flags_ : nullptr;

    BLUB_LAUNCH(pcg_reset_scalars_kernel, 1, 1, 0, stream, scal, barrier_);
    int *const scratch_cols = tile_cols_ ? tile_cols_ : num_active_; // (no cooperative launch: the counts are not used)
    // the persistent solvers ping-pong s between search_ and aux_: both zero off the fluid
    BLUB_LAUNCH(pcg_prepare_kernel, grid, block, 0, stream, g, t, marker, codes_.ptr, tile_active_, scratch_cols, field.p_tiles, flags, which, p, r, s,
                persistent ? aux_.ptr : nullptr);
    if (!flags) prepare_dense_next(stream);
    if (mode != 0) { // the stored preconditioner vectors must obey the zero invariant as well
        BLUB_CUDA_CHECK(cudaMemsetAsync(aux_.ptr, 0, (size_t)g.n * sizeof(float), stream));
        BLUB_CUDA_CHECK(cudaMemsetAsync(aux_temp_.ptr, 0, (size_t)g.n * sizeof(float), stream));
    }
    if (persistent) {
        // one cooperative launch for the whole solve
        const int ghost_tiles = (comm.halo / PCG_TZ) * t.tiles_x * t.tiles_y; // ghost planes are whole tiles (SLAB_HALO == PCG_TZ)
        int *col_offset = tile_cols_ + t.ntiles, *num_cols = tile_cols_ + 2 * t.ntiles;
        BLUB_LAUNCH(pcg_compact_kernel, 1, 1024, 0, stream, tile_active_, tile_cols_, ghost_tiles, t.ntiles - ghost_tiles, columns ? 1 : 0, tile_list_, num_active_ + 1,
                    num_active_, col_offset, num_cols, flags, which);
        PcgSolveArgs args;
        args.g = g; args.t = t; args.codes = st; args.tile_list = tile_list_; args.tile_list_flagged = num_active_ + 1; args.num_active = num_active_;
        args.p = p; args.r = r; args.s0 = s; args.s1 = aux_.ptr; args.scal = scal; args.partials = partials_;
        args.params = dparams; args.which = which; args.max_iterations = max_it; args.check_frequency = freq;
        args.comm = comm;
        args.col_list = col_list_; args.num_cols = num_cols; args.barrier = barrier_; args.code_slots = code_slots_;
        // z-slab ranks keep p in memory: their closing push reads it
        args.p_slots = columns && comm.world == 1 ? p_slots_ : 0;
        for (int c = 0; c < 3; ++c) args.wbeta[c] = weights ? weights->beta[c] : nullptr;
        args.wdiag = weights ? weights->diag : nullptr;
        args.winv = weights ? weights->inv_diag2 : nullptr;
        void *args_only[] = {&args}, *args_and_maps[] = {&args, tma_maps_};
        void **kargs = args_only;
        const void *kernel;
        int nblocks;
        size_t smem;
        if (weights) { // as many blocks as path 6 launches: the same grouping of every sum
            kernel = (const void *)pcg_solve_weighted_kernel;
            nblocks = persistent_blocks_ < t.ntiles ? persistent_blocks_ : t.ntiles;
            smem = 0;
        } else if (columns) { // dense tiles by the tile body, everything else column by column
            BLUB_LAUNCH(pcg_column_fill_kernel, grid, block, 0, stream, g, t, st, ta, col_offset, ghost_tiles, t.ntiles - ghost_tiles, col_list_);
            kernel = (const void *)pcg_solve_columns_kernel;
            nblocks = column_blocks_;
            smem = (size_t)code_slots_ * PCG_CODE_SLOT_BYTES + (size_t)args.p_slots * PCG_P_SLOT_BYTES;
        } else if (use_tma && tma_blocks_ > 0) {
            kernel = (const void *)pcg_solve_tma_kernel;
            kargs = args_and_maps;
            nblocks = tma_blocks_ < t.ntiles ? tma_blocks_ : t.ntiles;
            smem = TMA_SMEM_BYTES;
        } else {
            kernel = use_dense ? (const void *)pcg_solve_persistent_kernel<false> : (const void *)pcg_solve_persistent_kernel<true>;
            nblocks = persistent_blocks_ < t.ntiles ? persistent_blocks_ : t.ntiles;
            smem = 0;
        }
        BLUB_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(nblocks), t.block(), kargs, smem, stream));
        g_kernel_launches.fetch_add(1, std::memory_order_relaxed);
        return;
    }
    if (mode == 0) {
        BLUB_LAUNCH(pcg_init_kernel<0>, grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_);
    } else {
        BLUB_LAUNCH(pcg_init_kernel<1>, grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_);
        BLUB_LAUNCH(pcg_precond_pass_kernel, grid, block, 0, stream, g, t, st, ta, r, aux_temp_.ptr, r, 0, 0, scal, partials_);
        BLUB_LAUNCH(pcg_precond_pass_kernel, grid, block, 0, stream, g, t, st, ta, aux_temp_.ptr, s, r, 1, 1, scal, partials_);
    }
    for (int i = 0;; ++i) {
        BLUB_LAUNCH(pcg_dot_kernel, grid, block, 0, stream, g, t, st, ta, s, scal, partials_);
        const bool with_err = (max_it == i) || (i > 0 && i % freq == 0); // pressure_solver.rs:676-677
        if (mode == 0) {
            if (with_err)
                BLUB_LAUNCH((pcg_update_kernel<0, true>), grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_, dparams, which, i, max_it);
            else
                BLUB_LAUNCH((pcg_update_kernel<0, false>), grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_, dparams, which, i, max_it);
        } else {
            if (with_err)
                BLUB_LAUNCH((pcg_update_kernel<1, true>), grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_, dparams, which, i, max_it);
            else
                BLUB_LAUNCH((pcg_update_kernel<1, false>), grid, block, 0, stream, g, t, st, ta, p, r, s, scal, partials_, dparams, which, i, max_it);
        }
        if (i >= max_it) break; // :699-701
        if (mode == 0) {
            BLUB_LAUNCH(pcg_search_kernel<0>, grid, block, 0, stream, g, t, st, ta, s, r, scal);
        } else {
            BLUB_LAUNCH(pcg_precond_pass_kernel, grid, block, 0, stream, g, t, st, ta, r, aux_temp_.ptr, r, 0, 0, scal, partials_);
            BLUB_LAUNCH(pcg_precond_pass_kernel, grid, block, 0, stream, g, t, st, ta, aux_temp_.ptr, aux_.ptr, r, 1, 3, scal, partials_);
            BLUB_LAUNCH(pcg_search_kernel<1>, grid, block, 0, stream, g, t, st, ta, s, aux_.ptr, scal);
        }
    }
}

} // namespace blub
