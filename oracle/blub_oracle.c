/*
 * blub_oracle.c -- CPU restatement of the Wumpf/blub APIC/FLIP fluid step.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The shipped library
 * (blub_b200/csrc -> libblubcore.so) never links, loads or calls anything in oracle/.
 *
 * PARITY UNPINNED: the reference (Rust + wgpu/Vulkan + GLSL) cannot be built or run in this
 * environment (no cargo/rustc/Vulkan/shaderc, 258 un-vendored crates, windowed app) and it
 * ships no tests, golden vectors or known-answer fixtures for this path.  This file follows
 * the reference's shaders and host code line by line (citations below, relative to
 * the reference checkout) and is pinned only by analytic known-answer tests (tests/test_oracle_kat.py, tests/test_transfer_kat.py).
 *
 * Conventions (shader/simulation/hybrid_fluid.glsl:20-23):
 *   marker: SOLID = 0, FLUID = 1, AIR = -1; any out-of-domain texel/image read returns 0.
 *   grids are linear x-fastest; face value U_c[g] lives on the +c face of cell g
 *   (shader/simulation/bindings_write_volume.glsl:10).
 *   linked-list pointers on the grid are stored +1 so that 0 == empty (particles.glsl:1-3).
 * All arithmetic is IEEE fp32 (compile with -ffp-contract=off).
 *
 * Quirk switches (SURVEY.md Appendix B):
 *   precond_mode   0 = "diag2": neighbour fetch at LOD 1 of a 1-mip texture returns 0
 *                      (pressure_apply_preconditioner.comp:58,61,64) => z = r / diag^2   [default]
 *                  1 = "clamped": LOD clamped to 0 => z = (D^-1 (I - L))^2 r (as literally written)
 *   cap_p2g / cap_density   max list entries walked per dual cell (reference: 12 / 32;
 *                      transfer_gather_velocity.comp:61, density_projection_gather_error.comp:69);
 *                      0 = no cap [default]
 *   binning_mode   0 = fixed stable counting sort [default], 1 = as written (off-by-one, unguarded)
 *   reduce_mode    0 = every partial of the first reduce level is summed [default]
 *                  1 = as written: the final pass reads N / 16384 (FLOOR, pressure_solver.rs:571) partials although
 *                      ceil(N / 16384) groups wrote one (pressure_init.comp:27-30), so the last group's partial is dropped
 *                      whenever N is not a multiple of 16384.  Every shipped scene has N % 16384 == 0, where both modes
 *                      coincide (B16).
 * Followed as written without a switch: the in-cell RK4 of advect_particles.comp:116-125 advances component k's three interpolants by
 * step[k] (element-wise vec3 addition on component-indexed vectors, B17).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define CELL_SOLID 0
#define CELL_FLUID 1
#define CELL_AIR (-1)
#define INVALID_PTR 0xFFFFFFFFu

typedef struct {
    float error_tolerance;
    int max_num_iterations;
    int error_check_frequency;
} OrcSolverConfig;

typedef struct {
    float error; /* max|r| (NOT yet multiplied by dt) */
    int iteration_count;
} OrcSolveResult;

typedef struct OrcFluid {
    int nx, ny, nz;
    size_t n;
    uint32_t max_particles, num_particles;
    float gravity[3];
    /* particle state: hybrid_fluid.rs:76-85, particles.glsl:5-16 */
    float *pos;     /* 4 floats / particle: xyz + (uint32 next) */
    float *pos_tmp; /* binning scratch */
    float *row[3];  /* vec4(C_col.xyz, v_c) per particle per axis */
    /* grid */
    float *u[3];
    uint32_t *ll;
    int8_t *marker;
    float *voxel; /* RGBA per cell: xyz = solid velocity (cells/s), w != 0 => solid */
    /* solver scratch (pressure_solver.rs:228-529) */
    float *residual, *aux, *aux_temp, *search, *reduce0, *reduce1;
    float *pressure[2]; /* 0 = from velocity, 1 = from density */
    int pressure_touched[2];
    OrcSolverConfig cfg[2];
    OrcSolveResult last[2];
    uint32_t rebin_frequency, step_counter;
    int precond_mode, cap_p2g, cap_density, binning_mode, reduce_mode;
} OrcFluid;

/* ------------------------------------------------------------------ helpers */
static inline size_t lin(const OrcFluid *f, int x, int y, int z) { return ((size_t)z * f->ny + y) * f->nx + x; }
static inline int inb(const OrcFluid *f, int x, int y, int z) {
    return x >= 0 && y >= 0 && z >= 0 && x < f->nx && y < f->ny && z < f->nz;
}
static inline int mk(const OrcFluid *f, int x, int y, int z) { return inb(f, x, y, z) ? f->marker[lin(f, x, y, z)] : 0; }
static inline float ldf(const OrcFluid *f, const float *a, int x, int y, int z) { return inb(f, x, y, z) ? a[lin(f, x, y, z)] : 0.0f; }
static inline float vox(const OrcFluid *f, int x, int y, int z, int c) { return inb(f, x, y, z) ? f->voxel[lin(f, x, y, z) * 4 + c] : 0.0f; }
static inline float satf(float x) { return x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x); }
static inline float mixf(float a, float b, float t) { return a * (1.0f - t) + b * t; } /* GLSL mix */
static inline float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
static inline float fractf(float x) { return x - floorf(x); }
static inline float signf(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
static inline uint32_t *pnext(OrcFluid *f, uint32_t i) { return (uint32_t *)&f->pos[4 * (size_t)i + 3]; }

/* ------------------------------------------------------------------ lifecycle */
OrcFluid *orc_create(int nx, int ny, int nz, uint32_t max_particles) {
    OrcFluid *f = (OrcFluid *)calloc(1, sizeof(OrcFluid));
    f->nx = nx; f->ny = ny; f->nz = nz;
    f->n = (size_t)nx * ny * nz;
    f->max_particles = max_particles;
    size_t np = (size_t)max_particles + 64; /* slack for the as-written binning overrun */
    f->pos = (float *)calloc(np * 4, sizeof(float));
    f->pos_tmp = (float *)calloc(np * 4, sizeof(float));
    for (int c = 0; c < 3; ++c) {
        f->row[c] = (float *)calloc(np * 4, sizeof(float));
        f->u[c] = (float *)calloc(f->n, sizeof(float));
    }
    f->ll = (uint32_t *)calloc(f->n, sizeof(uint32_t));
    f->marker = (int8_t *)calloc(f->n, 1);
    f->voxel = (float *)calloc(f->n * 4, sizeof(float));
    f->residual = (float *)calloc(f->n, sizeof(float));
    f->aux = (float *)calloc(f->n, sizeof(float));
    f->aux_temp = (float *)calloc(f->n, sizeof(float));
    f->search = (float *)calloc(f->n, sizeof(float));
    f->reduce0 = (float *)calloc(f->n, sizeof(float));
    f->reduce1 = (float *)calloc(f->n / 16384 + 1024, sizeof(float));
    for (int k = 0; k < 2; ++k) {
        f->pressure[k] = (float *)calloc(f->n, sizeof(float));
        /* defaults: hybrid_fluid.rs:253-257 */
        f->cfg[k].error_tolerance = 0.1f;
        f->cfg[k].error_check_frequency = 4;
        f->cfg[k].max_num_iterations = 32;
    }
    f->rebin_frequency = 60; /* hybrid_fluid.rs:603-605 */
    return f;
}

void orc_destroy(OrcFluid *f) {
    if (!f) return;
    free(f->pos); free(f->pos_tmp);
    for (int c = 0; c < 3; ++c) { free(f->row[c]); free(f->u[c]); }
    free(f->ll); free(f->marker); free(f->voxel);
    free(f->residual); free(f->aux); free(f->aux_temp); free(f->search); free(f->reduce0); free(f->reduce1);
    free(f->pressure[0]); free(f->pressure[1]);
    free(f);
}

/* ------------------------------------------------------------------ particle seeding
 * hybrid_fluid.rs:609-678.  RNG = rand 0.8.5 SmallRng (xoshiro256++ seeded through SplitMix64),
 * cgmath 0.18 Standard -> Vector3<f32> draws x,y,z; f32 = (next_u32 >> 8) * 2^-24 with
 * next_u32 = high half of next_u64.  Third-party crates are absent from the reference checkout
 * (Cargo.lock pins rand 0.8.5, rand_core 0.6.4, cgmath 0.18.0): restated from the published
 * algorithms, unverifiable offline. */
typedef struct { uint64_t s[4]; } Xo;
static inline uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static void xo_seed(Xo *r, uint64_t state) {
    for (int i = 0; i < 4; ++i) {
        state += 0x9e3779b97f4a7c15ull;
        uint64_t z = state;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        r->s[i] = z ^ (z >> 31);
    }
}
static inline uint64_t xo_next(Xo *r) {
    uint64_t *s = r->s;
    uint64_t result = rotl64(s[0] + s[3], 23) + s[0];
    uint64_t t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
    s[2] ^= t;
    s[3] = rotl64(s[3], 45);
    return result;
}
static inline float xo_f32(Xo *r) { return (float)((uint32_t)(xo_next(r) >> 32) >> 8) * (1.0f / 16777216.0f); }

static uint32_t clamp_to_grid(uint32_t dim, float v) { /* hybrid_fluid.rs:609-617 */
    uint32_t u = v <= 0.0f ? 0u : (v >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)v); /* Rust `as u32` saturates */
    uint32_t m = dim - 1 < u ? dim - 1 : u;
    return m < 1 ? 1 : m;
}

/* returns number of particles added; -1-based truncation is reported via *truncated */
uint32_t orc_add_fluid_cube(OrcFluid *f, const float min_grid[3], const float max_grid[3], int *truncated) {
    uint32_t dim[3] = {(uint32_t)f->nx, (uint32_t)f->ny, (uint32_t)f->nz};
    uint32_t mn[3], mx[3], ext[3];
    for (int k = 0; k < 3; ++k) {
        mn[k] = clamp_to_grid(dim[k], min_grid[k]);
        mx[k] = clamp_to_grid(dim[k], max_grid[k]);
        ext[k] = mx[k] - mn[k]; /* max corner is exclusive */
    }
    uint32_t num_new = ext[0] * ext[1] * ext[2] * 8u;
    if (truncated) *truncated = 0;
    if (f->max_particles < num_new + f->num_particles) { /* hybrid_fluid.rs:627-633 */
        num_new = f->max_particles - f->num_particles;
        if (truncated) *truncated = 1;
    }
    Xo rng;
    xo_seed(&rng, (uint64_t)(f->num_particles + num_new)); /* hybrid_fluid.rs:637 */
    for (uint32_t i = 0; i < num_new; ++i) {
        float cell[3] = {(float)(mn[0] + i / 8u % ext[0]), (float)(mn[1] + i / 8u / ext[0] % ext[1]),
                         (float)(mn[2] + i / 8u / ext[0] / ext[1])};
        uint32_t s = i % 8u;
        float strat[3] = {(float)(s % 2u), (float)(s / 2u % 2u), (float)(s / 4u % 2u)};
        float *p = &f->pos[4 * (size_t)(f->num_particles + i)];
        for (int k = 0; k < 3; ++k) {
            float r = xo_f32(&rng);
            float off = strat[k] * 0.5f + r * 0.5f; /* hybrid_fluid.rs:664-665 */
            p[k] = cell[k] + off;
        }
        *(uint32_t *)&p[3] = INVALID_PTR;
    }
    f->num_particles += num_new;
    return num_new;
}

void orc_set_particles(OrcFluid *f, uint32_t n, const float *pos4, const float *rx, const float *ry, const float *rz) {
    if (n > f->max_particles) n = f->max_particles;
    f->num_particles = n;
    memcpy(f->pos, pos4, (size_t)n * 16);
    if (rx) memcpy(f->row[0], rx, (size_t)n * 16); else memset(f->row[0], 0, (size_t)n * 16);
    if (ry) memcpy(f->row[1], ry, (size_t)n * 16); else memset(f->row[1], 0, (size_t)n * 16);
    if (rz) memcpy(f->row[2], rz, (size_t)n * 16); else memset(f->row[2], 0, (size_t)n * 16);
}

void orc_set_gravity(OrcFluid *f, const float g[3]) { memcpy(f->gravity, g, 12); }
void orc_set_solver_config(OrcFluid *f, int which, float tol, int max_it, int freq) {
    f->cfg[which].error_tolerance = tol; f->cfg[which].max_num_iterations = max_it; f->cfg[which].error_check_frequency = freq;
}
void orc_set_rebin_frequency(OrcFluid *f, uint32_t fr) { f->rebin_frequency = fr; }
void orc_set_quirks(OrcFluid *f, int precond_mode, int cap_p2g, int cap_density, int binning_mode) {
    f->precond_mode = precond_mode; f->cap_p2g = cap_p2g; f->cap_density = cap_density; f->binning_mode = binning_mode;
}
void orc_set_reduce_mode(OrcFluid *f, int mode) { f->reduce_mode = mode; }
void orc_set_voxels(OrcFluid *f, const float *rgba) { memcpy(f->voxel, rgba, f->n * 16); }
uint32_t orc_num_particles(const OrcFluid *f) { return f->num_particles; }
uint32_t orc_step_counter(const OrcFluid *f) { return f->step_counter; }
void orc_last_solve(const OrcFluid *f, int which, float *err, int *iters) { *err = f->last[which].error; *iters = f->last[which].iteration_count; }

/* array accessor for the Python harness */
void *orc_array(OrcFluid *f, int which) {
    switch (which) {
    case 0: return f->pos;
    case 1: return f->row[0];
    case 2: return f->row[1];
    case 3: return f->row[2];
    case 4: return f->u[0];
    case 5: return f->u[1];
    case 6: return f->u[2];
    case 7: return f->marker;
    case 8: return f->pressure[0];
    case 9: return f->pressure[1];
    case 10: return f->residual;
    case 11: return f->ll;
    case 12: return f->voxel;
    case 13: return f->search;
    case 14: return f->aux;
    default: return NULL;
    }
}

/* ------------------------------------------------------------------ A1: P2G */
/* transfer_clear.comp:10-15 */
void orc_transfer_clear(OrcFluid *f, int c) {
    memset(f->ll, 0, f->n * sizeof(uint32_t));
    if (c == 0) memset(f->marker, CELL_AIR, f->n);
}

/* transfer_build_linkedlist.comp:10-27 -- particles in index order; the atomic exchange then makes
 * each dual-cell list run in DESCENDING particle index (the GPU's arrival order is arbitrary). */
void orc_transfer_build_linkedlist(OrcFluid *f, int c) {
    float off[3] = {0.5f, 0.5f, 0.5f};
    off[c] = 1.0f;
    for (uint32_t i = 0; i < f->num_particles; ++i) {
        const float *p = &f->pos[4 * (size_t)i];
        if (c == 0) {
            int x = (int)p[0], y = (int)p[1], z = (int)p[2];
            if (inb(f, x, y, z)) f->marker[lin(f, x, y, z)] = CELL_FLUID;
        }
        int dx = (int)(p[0] - off[0]), dy = (int)(p[1] - off[1]), dz = (int)(p[2] - off[2]);
        uint32_t prev = 0;
        if (inb(f, dx, dy, dz)) { /* imageAtomicExchange out of bounds: no store, returns 0 */
            size_t d = lin(f, dx, dy, dz);
            prev = f->ll[d];
            f->ll[d] = i + 1;
        }
        *pnext(f, i) = prev - 1u;
    }
}

/* transfer_set_boundary_marker.comp:11-20 */
void orc_set_boundary_marker(OrcFluid *f) {
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                size_t g = lin(f, x, y, z);
                if (x == 0 || y == 0 || z == 0 || x == f->nx - 1 || y == f->ny - 1 || z == f->nz - 1)
                    f->marker[g] = CELL_SOLID;
                else if (f->voxel[g * 4 + 3] != 0.0f)
                    f->marker[g] = CELL_SOLID;
            }
}

/* transfer_gather_velocity.comp:39-127.  Round i visits the i-th list entry of the thread's own dual
 * cell first (:63-72) and then those of the seven neighbours in the order of :85-91. */
static const int GATHER_ORDER[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {1, 1, 0}, {0, 0, 1}, {1, 0, 1}, {0, 1, 1}, {1, 1, 1}};

void orc_transfer_gather_velocity(OrcFluid *f, int c, float dt) {
    const float *rowc = f->row[c];
    const int cap = f->cap_p2g;
#pragma omp parallel for collapse(2) schedule(dynamic, 4)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                int n[3] = {x, y, z};
                n[c] += 1;
                int ma = mk(f, x, y, z), mb = mk(f, n[0], n[1], n[2]);
                int writes = (ma == CELL_FLUID || mb == CELL_FLUID);
                if (!writes) continue; /* stale value stays (B6) */
                int computes = (ma != CELL_SOLID && mb != CELL_SOLID);
                float q[3] = {(float)x + 0.5f, (float)y + 0.5f, (float)z + 0.5f};
                q[c] += 0.5f;
                float num = 0.0f, den = 0.0f;
                if (computes) {
                    uint32_t cur[8];
                    for (int k = 0; k < 8; ++k) {
                        int dx = x - GATHER_ORDER[k][0], dy = y - GATHER_ORDER[k][1], dz = z - GATHER_ORDER[k][2];
                        cur[k] = (inb(f, dx, dy, dz) ? f->ll[lin(f, dx, dy, dz)] : 0u) - 1u;
                    }
                    for (int round = 0; cap == 0 || round < cap; ++round) {
                        int any = 0;
                        for (int k = 0; k < 8; ++k) {
                            uint32_t i = cur[k];
                            if (i == INVALID_PTR) continue;
                            any = 1;
                            const float *p = &f->pos[4 * (size_t)i];
                            const float *r = &rowc[4 * (size_t)i];
                            cur[k] = *(const uint32_t *)&p[3];
                            float tx = q[0] - p[0], ty = q[1] - p[1], tz = q[2] - p[2];
                            float w = satf(1.0f - fabsf(tx)) * satf(1.0f - fabsf(ty)) * satf(1.0f - fabsf(tz));
                            float d = r[0] * tx + r[1] * ty + r[2] * tz + r[3] * 1.0f;
                            num += w * d;
                            den += w;
                        }
                        if (!any) break;
                    }
                    if (den > 0.0f) num /= den;
                    num += f->gravity[c] * dt;
                } else {
                    num = 0.0f;
                }
                f->u[c][lin(f, x, y, z)] = num;
            }
}

/* hybrid_fluid.rs:806-833 */
void orc_stage_p2g(OrcFluid *f, float dt) {
    for (int c = 0; c < 3; ++c) {
        orc_transfer_clear(f, c);
        orc_transfer_build_linkedlist(f, c);
        if (c == 0) orc_set_boundary_marker(f);
        orc_transfer_gather_velocity(f, c, dt);
    }
}

/* ------------------------------------------------------------------ A2: rhs of solve 1
 * divergence_compute.comp:28-86 (result goes into the PCG residual volume, hybrid_fluid.rs:836-838) */
void orc_divergence_compute(OrcFluid *f) {
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                if (mk(f, x, y, z) != CELL_FLUID) continue;
                float px = ldf(f, f->u[0], x, y, z), py = ldf(f, f->u[1], x, y, z), pz = ldf(f, f->u[2], x, y, z);
                float nx_ = ldf(f, f->u[0], x - 1, y, z), ny_ = ldf(f, f->u[1], x, y - 1, z), nz_ = ldf(f, f->u[2], x, y, z - 1);
                float d = px - nx_;
                d += py - ny_;
                d += pz - nz_;
                if (mk(f, x - 1, y, z) == CELL_SOLID) d += nx_ - vox(f, x - 1, y, z, 0);
                if (mk(f, x, y - 1, z) == CELL_SOLID) d += ny_ - vox(f, x, y - 1, z, 1);
                if (mk(f, x, y, z - 1) == CELL_SOLID) d += nz_ - vox(f, x, y, z - 1, 2);
                if (mk(f, x + 1, y, z) == CELL_SOLID) d -= px - vox(f, x + 1, y, z, 0);
                if (mk(f, x, y + 1, z) == CELL_SOLID) d -= py - vox(f, x, y + 1, z, 1);
                if (mk(f, x, y, z + 1) == CELL_SOLID) d -= pz - vox(f, x, y, z + 1, 2);
                f->residual[lin(f, x, y, z)] = d;
            }
}

/* ------------------------------------------------------------------ A3: PCG
 * pressure.glsl:34-75 */
static float mul_coeff(const OrcFluid *f, const float *t, int x, int y, int z, float v) {
    int m0 = mk(f, x - 1, y, z), m1 = mk(f, x + 1, y, z), m2 = mk(f, x, y - 1, z), m3 = mk(f, x, y + 1, z), m4 = mk(f, x, y, z - 1),
        m5 = mk(f, x, y, z + 1);
    float nn = 0.0f;
    nn += fabsf((float)m0); nn += fabsf((float)m1); nn += fabsf((float)m2);
    nn += fabsf((float)m3); nn += fabsf((float)m4); nn += fabsf((float)m5);
    float r = 0.0f;
    r += nn * v;
    if (m0 == CELL_FLUID) r -= ldf(f, t, x - 1, y, z);
    if (m1 == CELL_FLUID) r -= ldf(f, t, x + 1, y, z);
    if (m2 == CELL_FLUID) r -= ldf(f, t, x, y - 1, z);
    if (m3 == CELL_FLUID) r -= ldf(f, t, x, y + 1, z);
    if (m4 == CELL_FLUID) r -= ldf(f, t, x, y, z - 1);
    if (m5 == CELL_FLUID) r -= ldf(f, t, x, y, z + 1);
    return r;
}

/* GetReduceBufferAddress(): 8x8x1 work groups, pressure_apply_coeff.comp:13-17 */
static inline size_t reduce_addr(const OrcFluid *f, int x, int y, int z) {
    int ngx = (f->nx + 7) / 8, ngy = (f->ny + 7) / 8;
    size_t group = ((size_t)z * ngy + (y >> 3)) * ngx + (x >> 3);
    return (size_t)((y & 7) * 8 + (x & 7)) + 64u * group;
}

/* pressure_reduce.comp:35-61 -- one 1024-thread group with `groups` groups dispatched */
static float reduce_group(const float *src, size_t src_size, uint32_t group, uint32_t groups, int is_max) {
    float sh[1024];
    size_t dispatch = (size_t)1024 * groups;
    for (uint32_t t = 0; t < 1024; ++t) {
        size_t a = (size_t)group * 1024 + t;
        float v = 0.0f;
        for (int i = 0; i < 16; ++i) {
            if (a < src_size) v = is_max ? fmaxf(v, src[a]) : v + src[a];
            a += dispatch;
        }
        sh[t] = v;
    }
    for (uint32_t i = 512; i > 1; i /= 2)
        for (uint32_t t = 0; t < i; ++t) sh[t] = is_max ? fmaxf(sh[t], sh[t + i]) : sh[t] + sh[t + i];
    return is_max ? fmaxf(sh[0], sh[1]) : sh[0] + sh[1];
}

/* PressureSolver::reduce, pressure_solver.rs:543-589: strided passes while remaining > 16384, then 1 group */
static float reduce_all(OrcFluid *f, int is_max) {
    size_t remaining = f->n;
    float *src = f->reduce0, *dst = f->reduce1;
    while (remaining > 16384) {
        uint32_t groups = (uint32_t)((remaining / 16 + 1023) / 1024);
#pragma omp parallel for
        for (uint32_t g = 0; g < groups; ++g) dst[g] = reduce_group(src, remaining, g, groups, is_max);
        float *t = src; src = dst; dst = t;
        remaining = f->reduce_mode == 1 ? remaining / 16384 : (size_t)groups; /* B16 */
    }
    float r = reduce_group(src, remaining, 0, 1, is_max);
    return r;
}

/* pressure_apply_preconditioner.comp:36-82 */
static void precond_pass(OrcFluid *f, const float *in, float *out, int pass1) {
    const int lod1_is_zero = (f->precond_mode == 0);
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                size_t ra = reduce_addr(f, x, y, z);
                if (mk(f, x, y, z) != CELL_FLUID) {
                    if (pass1) f->reduce0[ra] = 0.0f;
                    continue;
                }
                size_t g = lin(f, x, y, z);
                float res = in[g];
                int m0 = mk(f, x - 1, y, z), m1 = mk(f, x + 1, y, z), m2 = mk(f, x, y - 1, z), m3 = mk(f, x, y + 1, z),
                    m4 = mk(f, x, y, z - 1), m5 = mk(f, x, y, z + 1);
                if (!lod1_is_zero) {
                    if (m0 == CELL_FLUID) res -= ldf(f, in, x - 1, y, z);
                    if (m2 == CELL_FLUID) res -= ldf(f, in, x, y - 1, z);
                    if (m4 == CELL_FLUID) res -= ldf(f, in, x, y, z - 1);
                }
                float nn = 0.0f;
                nn += (float)(m0 != CELL_SOLID); nn += (float)(m1 != CELL_SOLID); nn += (float)(m2 != CELL_SOLID);
                nn += (float)(m3 != CELL_SOLID); nn += (float)(m4 != CELL_SOLID); nn += (float)(m5 != CELL_SOLID);
                if (nn > 0.0f) res /= nn;
                out[g] = res;
                if (pass1) f->reduce0[ra] = res * f->residual[g];
            }
}

/* PressureSolver::solve, pressure_solver.rs:591-729.  The rhs must already be in f->residual. */
void orc_solve(OrcFluid *f, int which, float dt) {
    float *p = f->pressure[which];
    const OrcSolverConfig cfg = f->cfg[which];
    const float tol = cfg.error_tolerance / dt; /* pressure_solver.rs:193-201 */
    const float EPS = 1e-10f;
    if (!f->pressure_touched[which]) { /* :601-603 */
        memset(p, 0, f->n * sizeof(float));
        f->pressure_touched[which] = 1;
    }
    /* pressure_init.comp:37-83 (in place on p: a non-fluid cell is zeroed, a fluid cell only reads FLUID neighbours) */
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                size_t g = lin(f, x, y, z);
                if (mk(f, x, y, z) != CELL_FLUID) { p[g] = 0.0f; continue; }
                int m0 = mk(f, x - 1, y, z), m1 = mk(f, x + 1, y, z), m2 = mk(f, x, y - 1, z), m3 = mk(f, x, y + 1, z),
                    m4 = mk(f, x, y, z - 1), m5 = mk(f, x, y, z + 1);
                float r = f->residual[g];
                float nn = 0.0f;
                nn += fabsf((float)m0); nn += fabsf((float)m1); nn += fabsf((float)m2);
                nn += fabsf((float)m3); nn += fabsf((float)m4); nn += fabsf((float)m5);
                if (nn > 0.0f) r -= nn * p[g];
                if (m0 == CELL_FLUID) r += p[g - 1];
                if (m1 == CELL_FLUID) r += p[g + 1];
                if (m2 == CELL_FLUID) r += p[g - f->nx];
                if (m3 == CELL_FLUID) r += p[g + f->nx];
                if (m4 == CELL_FLUID) r += p[g - (size_t)f->nx * f->ny];
                if (m5 == CELL_FLUID) r += p[g + (size_t)f->nx * f->ny];
                f->residual[g] = r;
            }
    float max_error = 0.0f;
    int num_iterations = 0; /* NumIterations = 0 doubles as "no stats yet" (pressure_reduce.comp:84) */
    /* init: precondition r straight into the search vector, sigma = z.r (:625-649) */
    precond_pass(f, f->residual, f->aux_temp, 0);
    precond_pass(f, f->aux_temp, f->search, 1);
    float alphabeta = 0.0f;
    float sigma = reduce_all(f, 0);
    for (int i = 0;; ++i) {
        /* pressure_apply_coeff.comp:19-30 */
#pragma omp parallel for collapse(2)
        for (int z = 0; z < f->nz; ++z)
            for (int y = 0; y < f->ny; ++y)
                for (int x = 0; x < f->nx; ++x) {
                    float dp = 0.0f;
                    if (mk(f, x, y, z) == CELL_FLUID) {
                        float s = f->search[lin(f, x, y, z)];
                        dp = s * mul_coeff(f, f->search, x, y, z, s);
                    }
                    f->reduce0[reduce_addr(f, x, y, z)] = dp;
                }
        float sAs = reduce_all(f, 0);
        alphabeta = sigma / (sAs + (sAs < 0.0f ? -EPS : EPS)); /* pressure_reduce.comp:73-75 */
        int with_err = (cfg.max_num_iterations == i) || (i > 0 && i % cfg.error_check_frequency == 0);
        /* pressure_update_pressure_and_residual.comp:23-59 */
        const float alpha = alphabeta;
#pragma omp parallel for collapse(2)
        for (int z = 0; z < f->nz; ++z)
            for (int y = 0; y < f->ny; ++y)
                for (int x = 0; x < f->nx; ++x) {
                    size_t g = lin(f, x, y, z);
                    if (mk(f, x, y, z) != CELL_FLUID) {
                        if (with_err) f->reduce0[reduce_addr(f, x, y, z)] = 0.0f;
                        continue;
                    }
                    float s = f->search[g];
                    p[g] = p[g] + alpha * s;
                    float r = f->residual[g];
                    r -= alpha * mul_coeff(f, f->search, x, y, z, s);
                    if (with_err) f->reduce0[reduce_addr(f, x, y, z)] = fabsf(r);
                    f->residual[g] = r;
                }
        if (with_err) {
            float e = reduce_all(f, 1);
            if (num_iterations == 0 && (cfg.max_num_iterations == i || e < tol)) { /* pressure_reduce.comp:82-94 */
                max_error = e;
                num_iterations = i;
                break; /* indirect dispatch arguments are zeroed: nothing else touches p, r */
            }
            if (cfg.max_num_iterations == i) break;
        }
        precond_pass(f, f->residual, f->aux_temp, 0);
        precond_pass(f, f->aux_temp, f->aux, 1);
        float zr = reduce_all(f, 0);
        alphabeta = zr / (sigma + (sigma < 0.0f ? -EPS : EPS)); /* :77-80 */
        sigma = zr;
        const float beta = alphabeta;
        /* pressure_update_search.comp:13-24 */
#pragma omp parallel for
        for (size_t g = 0; g < f->n; ++g)
            if (f->marker[g] == CELL_FLUID) f->search[g] = f->aux[g] + beta * f->search[g];
    }
    f->last[which].error = max_error;
    f->last[which].iteration_count = num_iterations;
}

/* ------------------------------------------------------------------ A4: projection
 * divergence_remove.comp:19-49 */
void orc_divergence_remove(OrcFluid *f) {
    const float *p = f->pressure[0];
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                size_t g = lin(f, x, y, z);
                int mc = f->marker[g];
                float pc = mc == CELL_FLUID ? p[g] : 0.0f;
                for (int c = 0; c < 3; ++c) {
                    int n[3] = {x, y, z};
                    n[c] += 1;
                    int mn = mk(f, n[0], n[1], n[2]);
                    float v = 0.0f;
                    if (mc == CELL_FLUID || mn == CELL_FLUID) {
                        if (mc == CELL_SOLID) v = vox(f, x, y, z, c);
                        else if (mn == CELL_SOLID) v = vox(f, n[0], n[1], n[2], c);
                        else {
                            v = f->u[c][g];
                            float pn = mn == CELL_FLUID ? ldf(f, p, n[0], n[1], n[2]) : 0.0f;
                            v -= pc - pn;
                        }
                    }
                    f->u[c][g] = v;
                }
            }
}

/* ------------------------------------------------------------------ A5: extrapolation
 * extrapolate_velocity.comp:26-90.  In place: written faces are exactly the invalid ones, read faces the valid ones. */
static inline int valid_vel(const OrcFluid *f, int x, int y, int z, int c) {
    if (mk(f, x, y, z) == CELL_FLUID) return 1;
    int n[3] = {x, y, z};
    n[c] += 1;
    return mk(f, n[0], n[1], n[2]) == CELL_FLUID;
}
void orc_extrapolate_velocity(OrcFluid *f) {
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                if (mk(f, x, y, z) == CELL_FLUID) continue;
                for (int c = 0; c < 3; ++c) {
                    int n[3] = {x, y, z};
                    n[c] += 1;
                    if (mk(f, n[0], n[1], n[2]) == CELL_FLUID) continue;
                    int a = (c + 1) % 3, b = (c + 2) % 3;
                    if (c == 1) { a = 0; b = 2; } /* loop order of the shader: first listed axis fastest */
                    if (c == 0) { a = 1; b = 2; }
                    if (c == 2) { a = 0; b = 1; }
                    float numv = 0.0f, avg = 0.0f;
                    for (int ob = -1; ob <= 1; ++ob)
                        for (int oa = -1; oa <= 1; ++oa) {
                            if (oa == 0 && ob == 0) continue;
                            int h[3] = {x, y, z};
                            h[a] += oa;
                            h[b] += ob;
                            if (valid_vel(f, h[0], h[1], h[2], c)) {
                                numv += 1.0f;
                                avg += ldf(f, f->u[c], h[0], h[1], h[2]);
                            }
                        }
                    if (numv > 0.0f) f->u[c][lin(f, x, y, z)] = avg / numv;
                }
            }
}

/* ------------------------------------------------------------------ A6: binning
 * particle_binning_{count,prefixsum,rewrite_particles}.comp, hybrid_fluid.rs:854-894.
 * Only the position buffer is permuted: the velocity rows are dead here (advect rewrites them). */
void orc_binning(OrcFluid *f) {
    uint32_t *cnt = f->ll; /* the linked-list volume doubles as ParticleBinningVolume (hybrid_fluid.rs:857) */
    memset(cnt, 0, f->n * sizeof(uint32_t));
    const uint32_t np = f->num_particles;
    if (f->binning_mode == 1) {
        /* AS WRITTEN (B2): no `i < NumParticles` guard, destination = inclusive prefix - index in cell.
         * Block bases are taken in linear block order here (the GPU uses atomic arrival order). */
        uint32_t nthreads = (np + 63u) / 64u * 64u;
        for (uint32_t i = 0; i < nthreads; ++i) { /* particle_binning_count.comp:10-12 */
            const float *p = &f->pos[4 * (size_t)i];
            int x = (int)p[0], y = (int)p[1], z = (int)p[2];
            uint32_t idx = 0;
            if (inb(f, x, y, z)) idx = cnt[lin(f, x, y, z)]++;
            *pnext(f, i) = idx;
        }
        uint32_t run = 0; /* particle_binning_prefixsum.comp:37-60 */
        for (size_t g = 0; g < f->n; ++g) {
            run += cnt[g];
            if (run != 0) cnt[g] = run;
        }
        for (uint32_t i = 0; i < nthreads; ++i) { /* particle_binning_rewrite_particles.comp:9-15 */
            const float *p = &f->pos[4 * (size_t)i];
            int x = (int)p[0], y = (int)p[1], z = (int)p[2];
            uint32_t incl = inb(f, x, y, z) ? cnt[lin(f, x, y, z)] : 0u;
            size_t dst = (size_t)(uint32_t)(incl - *pnext(f, i));
            if (dst < (size_t)f->max_particles + 64) memcpy(&f->pos_tmp[4 * dst], p, 16);
        }
        memcpy(f->pos, f->pos_tmp, (size_t)f->max_particles * 16); /* hybrid_fluid.rs:884-892 */
        return;
    }
    /* FIXED (default): guarded, exclusive offsets, stable (ascending particle index inside a cell). */
    for (uint32_t i = 0; i < np; ++i) {
        const float *p = &f->pos[4 * (size_t)i];
        int x = (int)p[0], y = (int)p[1], z = (int)p[2];
        if (inb(f, x, y, z)) cnt[lin(f, x, y, z)]++;
    }
    uint32_t run = 0;
    for (size_t g = 0; g < f->n; ++g) {
        uint32_t c = cnt[g];
        cnt[g] = run; /* exclusive start, used as the cell's write cursor below */
        run += c;
    }
    for (uint32_t i = 0; i < np; ++i) {
        const float *p = &f->pos[4 * (size_t)i];
        int x = (int)p[0], y = (int)p[1], z = (int)p[2];
        size_t dst = inb(f, x, y, z) ? cnt[lin(f, x, y, z)]++ : i;
        memcpy(&f->pos_tmp[4 * dst], p, 16);
    }
    memcpy(f->pos, f->pos_tmp, (size_t)np * 16);
}

/* ------------------------------------------------------------------ A7: G2P / advection
 * advect_particles.comp:35-194 */
static inline float voxel_point_w(const OrcFluid *f, const float p[3], float out_xyz[3]) {
    /* texture(sampler3D(SceneVoxelization, SamplerPointClamp), pos / gridSize): nearest texel, clamp to edge */
    int x = (int)floorf(p[0]), y = (int)floorf(p[1]), z = (int)floorf(p[2]);
    x = x < 0 ? 0 : (x > f->nx - 1 ? f->nx - 1 : x);
    y = y < 0 ? 0 : (y > f->ny - 1 ? f->ny - 1 : y);
    z = z < 0 ? 0 : (z > f->nz - 1 ? f->nz - 1 : z);
    const float *v = &f->voxel[lin(f, x, y, z) * 4];
    if (out_xyz) { out_xyz[0] = v[0]; out_xyz[1] = v[1]; out_xyz[2] = v[2]; }
    return v[3];
}
/* SamplerTrilinearClamp on channel `ch` of a 4-channel volume / or a scalar volume; coordinate in texels */
static float trilinear_clamp(const OrcFluid *f, const float *vol, int stride, int ch, float ux, float uy, float uz) {
    float cx = ux - 0.5f, cy = uy - 0.5f, cz = uz - 0.5f;
    float fx0 = floorf(cx), fy0 = floorf(cy), fz0 = floorf(cz);
    float tx = cx - fx0, ty = cy - fy0, tz = cz - fz0;
    int x0 = (int)fx0, y0 = (int)fy0, z0 = (int)fz0;
    int xs[2] = {x0, x0 + 1}, ys[2] = {y0, y0 + 1}, zs[2] = {z0, z0 + 1};
    for (int k = 0; k < 2; ++k) {
        xs[k] = xs[k] < 0 ? 0 : (xs[k] > f->nx - 1 ? f->nx - 1 : xs[k]);
        ys[k] = ys[k] < 0 ? 0 : (ys[k] > f->ny - 1 ? f->ny - 1 : ys[k]);
        zs[k] = zs[k] < 0 ? 0 : (zs[k] > f->nz - 1 ? f->nz - 1 : zs[k]);
    }
#define TL(i, j, k) vol[lin(f, xs[i], ys[j], zs[k]) * stride + ch]
    float c00 = mixf(TL(0, 0, 0), TL(1, 0, 0), tx), c10 = mixf(TL(0, 1, 0), TL(1, 1, 0), tx);
    float c01 = mixf(TL(0, 0, 1), TL(1, 0, 1), tx), c11 = mixf(TL(0, 1, 1), TL(1, 1, 1), tx);
#undef TL
    return mixf(mixf(c00, c10, ty), mixf(c01, c11, ty), tz);
}

static void trilerp3(const float v[8][3], const float ix[3], const float iy[3], const float iz[3], float out[3]) {
    /* InterpolateTrilinear, advect_particles.comp:19-23; corner order 000,100,010,110,001,101,011,111 */
    for (int k = 0; k < 3; ++k) {
        float a = mixf(mixf(v[0][k], v[1][k], ix[k]), mixf(v[2][k], v[3][k], ix[k]), iy[k]);
        float b = mixf(mixf(v[4][k], v[5][k], ix[k]), mixf(v[6][k], v[7][k], ix[k]), iy[k]);
        out[k] = mixf(a, b, iz[k]);
    }
}

/* shared wall handling, advect_particles.comp:134-173 / density_projection_correct_particles.comp:48-70 */
static int wall_hit(const OrcFluid *f, const float np_[3], int use_marker) {
    float hi[3] = {(float)f->nx - 1.001f, (float)f->ny - 1.001f, (float)f->nz - 1.001f};
    for (int k = 0; k < 3; ++k)
        if (clampf(np_[k], 1.001f, hi[k]) != np_[k]) return 1;
    if (use_marker) {
        int x = (int)floorf(np_[0]), y = (int)floorf(np_[1]), z = (int)floorf(np_[2]);
        x = x < 0 ? 0 : (x > f->nx - 1 ? f->nx - 1 : x);
        y = y < 0 ? 0 : (y > f->ny - 1 ? f->ny - 1 : y);
        z = z < 0 ? 0 : (z > f->nz - 1 ? f->nz - 1 : z);
        return f->marker[lin(f, x, y, z)] == CELL_SOLID;
    }
    return voxel_point_w(f, np_, NULL) > 0.0f;
}

void orc_advect_particles(OrcFluid *f, float dt) {
    const int S[3] = {f->nx, f->ny, f->nz};
    /* Every particle is independent up to the marker / linked-list writes of :175-181, whose result depends on the particle order:
     * those run in a second, sequential pass over the new positions (identical outcome, the first pass can use all cores). */
#pragma omp parallel for schedule(static)
    for (uint32_t i = 0; i < f->num_particles; ++i) {
        float x0[3] = {f->pos[4 * (size_t)i], f->pos[4 * (size_t)i + 1], f->pos[4 * (size_t)i + 2]};
        { /* :45-64 "eaten" by a moving wall */
            float sv[3];
            float w = voxel_point_w(f, x0, sv);
            if (w > 0.0f) {
                float ax = fabsf(sv[0]), ay = fabsf(sv[1]), az = fabsf(sv[2]);
                if (ax > ay) {
                    if (ax > az) x0[0] += signf(sv[0]); else x0[2] += signf(sv[2]);
                } else {
                    if (ay > az) x0[1] += signf(sv[1]); else x0[2] += signf(sv[2]);
                }
            }
        }
        float v[8][3], ix[3], iy[3], iz[3];
        for (int c = 0; c < 3; ++c) { /* :73-92 */
            float o[3] = {0.5f, 0.5f, 0.5f};
            o[c] = 1.0f;
            float op[3];
            int lo[3], hi[3];
            for (int k = 0; k < 3; ++k) {
                op[k] = fmaxf(0.0f, x0[k] - o[k]);
                lo[k] = (int)op[k];
                hi[k] = lo[k] + 1 < S[k] - 1 ? lo[k] + 1 : S[k] - 1;
            }
            const float *U = f->u[c];
            v[0][c] = ldf(f, U, lo[0], lo[1], lo[2]); v[1][c] = ldf(f, U, hi[0], lo[1], lo[2]);
            v[2][c] = ldf(f, U, lo[0], hi[1], lo[2]); v[3][c] = ldf(f, U, hi[0], hi[1], lo[2]);
            v[4][c] = ldf(f, U, lo[0], lo[1], hi[2]); v[5][c] = ldf(f, U, hi[0], lo[1], hi[2]);
            v[6][c] = ldf(f, U, lo[0], hi[1], hi[2]); v[7][c] = ldf(f, U, hi[0], hi[1], hi[2]);
            ix[c] = fractf(op[0]); iy[c] = fractf(op[1]); iz[c] = fractf(op[2]);
        }
        float vx00[3], vx01[3], vx10[3], vx11[3], vxy0[3], vxy1[3], nv[3], cx[3], cy[3], cz[3];
        for (int k = 0; k < 3; ++k) { /* :96-112 */
            vx00[k] = mixf(v[0][k], v[1][k], ix[k]);
            vx01[k] = mixf(v[4][k], v[5][k], ix[k]);
            vx10[k] = mixf(v[2][k], v[3][k], ix[k]);
            vx11[k] = mixf(v[6][k], v[7][k], ix[k]);
            vxy0[k] = mixf(vx00[k], vx10[k], iy[k]);
            vxy1[k] = mixf(vx01[k], vx11[k], iy[k]);
            nv[k] = mixf(vxy0[k], vxy1[k], iz[k]);
            cx[k] = mixf(mixf(v[1][k], v[3][k], iy[k]), mixf(v[5][k], v[7][k], iy[k]), iz[k]) -
                    mixf(mixf(v[0][k], v[2][k], iy[k]), mixf(v[4][k], v[6][k], iy[k]), iz[k]);
            cy[k] = mixf(vx10[k], vx11[k], iz[k]) - mixf(vx00[k], vx01[k], iz[k]);
            cz[k] = vxy1[k] - vxy0[k];
        }
        /* RK4 inside the cell, :116-126.  AS WRITTEN (SURVEY quirk B17, found in review): interpolantsX/Y/Z are vec3s indexed by the velocity
         * COMPONENT and the shader adds the step vector to each of them element-wise (`saturate(interpolantsX + stepK2)`), so component k
         * is re-sampled at its own interpolants advanced by step[k] along x, y AND z -- not at the point moved by (step.x, step.y, step.z). */
        float k1[3] = {nv[0], nv[1], nv[2]}, k2[3], k3[3], k4[3], ax[3], ay[3], az[3], st[3];
        for (int k = 0; k < 3; ++k) st[k] = dt * 0.5f * k1[k];
        for (int k = 0; k < 3; ++k) { ax[k] = satf(ix[k] + st[k]); ay[k] = satf(iy[k] + st[k]); az[k] = satf(iz[k] + st[k]); }
        trilerp3(v, ax, ay, az, k2);
        for (int k = 0; k < 3; ++k) st[k] = dt * 0.5f * k2[k];
        for (int k = 0; k < 3; ++k) { ax[k] = satf(ix[k] + st[k]); ay[k] = satf(iy[k] + st[k]); az[k] = satf(iz[k] + st[k]); }
        trilerp3(v, ax, ay, az, k3);
        for (int k = 0; k < 3; ++k) st[k] = dt * k3[k];
        for (int k = 0; k < 3; ++k) { ax[k] = satf(ix[k] + st[k]); ay[k] = satf(iy[k] + st[k]); az[k] = satf(iz[k] + st[k]); }
        trilerp3(v, ax, ay, az, k4);
        float mv[3], x1[3];
        for (int k = 0; k < 3; ++k) {
            mv[k] = dt * (1.0f / 6.0f) * (k1[k] + 2.0f * (k2[k] + k3[k]) + k4[k]);
            x1[k] = x0[k] + mv[k];
        }
        if (wall_hit(f, x1, 0)) { /* :134-173 */
            float len = sqrtf(mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2]) + 1e-10f;
            float dir[3] = {mv[0] / len, mv[1] / len, mv[2] / len};
            float maxstep = len;
            for (int k = 0; k < 3; ++k) {
                float pc = fractf(x0[k]);
                maxstep = fminf(maxstep, (dir[k] > 0.0f ? pc : 1.0f - pc) / fabsf(dir[k]) - 0.001f);
            }
            for (int k = 0; k < 3; ++k) mv[k] = dir[k] * maxstep;
            if ((int)x0[0] == (int)x1[0] && (int)x0[1] == (int)x1[1] && (int)x0[2] == (int)x1[2]) {
                /* stuck: push along -grad(V.w), smooth sample at the (pre-correction) new position +- one texel */
                float push[3];
                for (int k = 0; k < 3; ++k) {
                    float a[3] = {x1[0], x1[1], x1[2]}, b[3] = {x1[0], x1[1], x1[2]};
                    a[k] -= 1.0f;
                    b[k] += 1.0f;
                    push[k] = trilinear_clamp(f, f->voxel, 4, 3, a[0], a[1], a[2]) - trilinear_clamp(f, f->voxel, 4, 3, b[0], b[1], b[2]);
                }
                for (int k = 0; k < 3; ++k) mv[k] += push[k] * (dt * 50.0f);
            }
            float hi[3] = {(float)f->nx - 1.001f, (float)f->ny - 1.001f, (float)f->nz - 1.001f};
            for (int k = 0; k < 3; ++k) {
                x1[k] = clampf(x0[k] + mv[k], 1.001f, hi[k]);
                nv[k] = (dir[k] * maxstep) / dt;
            }
        }
        float *P = &f->pos[4 * (size_t)i];
        P[0] = x1[0]; P[1] = x1[1]; P[2] = x1[2];
        float *rx = &f->row[0][4 * (size_t)i], *ry = &f->row[1][4 * (size_t)i], *rz = &f->row[2][4 * (size_t)i];
        rx[0] = cx[0]; rx[1] = cx[1]; rx[2] = cx[2]; rx[3] = nv[0]; /* :184-188 (B4: Jacobian columns stored as rows) */
        ry[0] = cy[0]; ry[1] = cy[1]; ry[2] = cy[2]; ry[3] = nv[1];
        rz[0] = cz[0]; rz[1] = cz[1]; rz[2] = cz[2]; rz[3] = nv[2];
    }
    for (uint32_t i = 0; i < f->num_particles; ++i) { /* :175-181 marker + linked list for the density pass, in particle order */
        const float *x1 = &f->pos[4 * (size_t)i];
        int x = (int)x1[0], y = (int)x1[1], z = (int)x1[2];
        if (inb(f, x, y, z)) f->marker[lin(f, x, y, z)] = CELL_FLUID;
        int dx = (int)(x1[0] - 0.5f), dy = (int)(x1[1] - 0.5f), dz = (int)(x1[2] - 0.5f);
        uint32_t prev = 0;
        if (inb(f, dx, dy, dz)) {
            size_t d = lin(f, dx, dy, dz);
            prev = f->ll[d];
            f->ll[d] = i + 1;
        }
        *pnext(f, i) = prev - 1u;
    }
}

/* ------------------------------------------------------------------ A8: rhs of solve 2
 * density_projection_gather_error.comp:41-199 */
void orc_density_gather_error(OrcFluid *f, float dt) {
    const int cap = f->cap_density;
#pragma omp parallel for collapse(2) schedule(dynamic, 4)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                if (mk(f, x, y, z) != CELL_FLUID) continue;
                float q[3] = {(float)x + 0.5f, (float)y + 0.5f, (float)z + 0.5f};
                float density = 0.0f;
                uint32_t cur[8];
                for (int k = 0; k < 8; ++k) {
                    int dx = x - GATHER_ORDER[k][0], dy = y - GATHER_ORDER[k][1], dz = z - GATHER_ORDER[k][2];
                    cur[k] = (inb(f, dx, dy, dz) ? f->ll[lin(f, dx, dy, dz)] : 0u) - 1u;
                }
                for (int round = 0; cap == 0 || round < cap; ++round) {
                    int any = 0;
                    for (int k = 0; k < 8; ++k) {
                        uint32_t i = cur[k];
                        if (i == INVALID_PTR) continue;
                        any = 1;
                        const float *p = &f->pos[4 * (size_t)i];
                        cur[k] = *(const uint32_t *)&p[3];
                        float tx = q[0] - p[0], ty = q[1] - p[1], tz = q[2] - p[2];
                        density += satf(1.0f - fabsf(tx)) * satf(1.0f - fabsf(ty)) * satf(1.0f - fabsf(tz));
                    }
                    if (!any) break;
                }
                int m[6] = {mk(f, x + 1, y, z), mk(f, x, y + 1, z), mk(f, x, y, z + 1), mk(f, x - 1, y, z), mk(f, x, y - 1, z), mk(f, x, y, z - 1)};
                int any_air = 0;
                for (int k = 0; k < 6; ++k) {
                    if (m[k] == CELL_SOLID) density += 0.5625f;
                    if (m[k] == CELL_AIR) any_air = 1;
                }
                if (any_air) density = fmaxf(8.0f, density);
                density = 1.0f - density / 8.0f;
                density = clampf(density, -0.5f, 0.5f);
                density /= dt;
                f->residual[lin(f, x, y, z)] = density;
            }
}

/* ------------------------------------------------------------------ A10: displacement field + particle correction
 * density_projection_position_change.comp:18-51 (overwrites the velocity volumes!) */
void orc_density_position_change(OrcFluid *f, float dt) {
    const float *p = f->pressure[1];
#pragma omp parallel for collapse(2)
    for (int z = 0; z < f->nz; ++z)
        for (int y = 0; y < f->ny; ++y)
            for (int x = 0; x < f->nx; ++x) {
                size_t g = lin(f, x, y, z);
                int mc = f->marker[g];
                float pc = mc == CELL_FLUID ? p[g] : 0.0f;
                for (int c = 0; c < 3; ++c) {
                    int n[3] = {x, y, z};
                    n[c] += 1;
                    int mn = mk(f, n[0], n[1], n[2]);
                    float pn = mn == CELL_FLUID ? ldf(f, p, n[0], n[1], n[2]) : 0.0f;
                    float d = (pn - pc) * dt;
                    if (mc == CELL_SOLID || mn == CELL_SOLID) d = 0.0f;
                    f->u[c][g] = d;
                }
            }
}

/* density_projection_correct_particles.comp:25-73 (fp32 software trilinear; the GPU's 8-bit filter weights are B5) */
void orc_density_correct_particles(OrcFluid *f) {
#pragma omp parallel for
    for (uint32_t i = 0; i < f->num_particles; ++i) {
        float *P = &f->pos[4 * (size_t)i];
        float x0[3] = {P[0], P[1], P[2]};
        float ch[3];
        for (int c = 0; c < 3; ++c) {
            float o[3] = {0.0f, 0.0f, 0.0f};
            o[c] = 0.5f;
            ch[c] = trilinear_clamp(f, f->u[c], 1, 0, fmaxf(0.0f, x0[0] - o[0]), fmaxf(0.0f, x0[1] - o[1]), fmaxf(0.0f, x0[2] - o[2]));
        }
        float x1[3] = {x0[0] + ch[0], x0[1] + ch[1], x0[2] + ch[2]};
        if (wall_hit(f, x1, 1)) {
            float len = sqrtf(ch[0] * ch[0] + ch[1] * ch[1] + ch[2] * ch[2]) + 1e-10f;
            float dir[3] = {ch[0] / len, ch[1] / len, ch[2] / len};
            float maxstep = len;
            for (int k = 0; k < 3; ++k) {
                float pc = fractf(x0[k]);
                maxstep = fminf(maxstep, (dir[k] > 0.0f ? pc : 1.0f - pc) / fabsf(dir[k]) - 0.001f);
            }
            float hi[3] = {(float)f->nx - 1.001f, (float)f->ny - 1.001f, (float)f->nz - 1.001f};
            for (int k = 0; k < 3; ++k) x1[k] = clampf(x0[k] + dir[k] * maxstep, 1.001f, hi[k]);
        }
        P[0] = x1[0]; P[1] = x1[1]; P[2] = x1[2];
    }
}

/* ------------------------------------------------------------------ the step: HybridFluid::step, hybrid_fluid.rs:770-977 */
void orc_step(OrcFluid *f, float dt) {
    orc_stage_p2g(f, dt);                /* :798-833 */
    orc_divergence_compute(f);           /* :835-840 */
    orc_solve(f, 0, dt);                 /* :843-852 */
    if (f->rebin_frequency != 0 && f->step_counter % f->rebin_frequency == 0) orc_binning(f); /* :854-894 */
    orc_divergence_remove(f);            /* :901-904 */
    orc_extrapolate_velocity(f);         /* :906-909 */
    orc_transfer_clear(f, 0);            /* :911-916 */
    orc_advect_particles(f, dt);         /* :917-921 */
    orc_set_boundary_marker(f);          /* :923-927 */
    orc_density_gather_error(f, dt);     /* :928-932 */
    orc_solve(f, 1, dt);                 /* :940-949 */
    orc_density_position_change(f, dt);  /* :959-962 */
    orc_extrapolate_velocity(f);         /* :963-966 */
    orc_density_correct_particles(f);    /* :968-972 */
    f->step_counter += 1;
}

/* stage-wise stepping for per-stage parity taps: runs stages [from, to) of the list above (0..13) */
void orc_step_stages(OrcFluid *f, float dt, int from, int to) {
    for (int s = from; s < to; ++s) {
        switch (s) {
        case 0: orc_stage_p2g(f, dt); break;
        case 1: orc_divergence_compute(f); break;
        case 2: orc_solve(f, 0, dt); break;
        case 3: if (f->rebin_frequency != 0 && f->step_counter % f->rebin_frequency == 0) orc_binning(f); break;
        case 4: orc_divergence_remove(f); break;
        case 5: orc_extrapolate_velocity(f); break;
        case 6: orc_transfer_clear(f, 0); break;
        case 7: orc_advect_particles(f, dt); break;
        case 8: orc_set_boundary_marker(f); break;
        case 9: orc_density_gather_error(f, dt); break;
        case 10: orc_solve(f, 1, dt); break;
        case 11: orc_density_position_change(f, dt); break;
        case 12: orc_extrapolate_velocity(f); break;
        case 13: orc_density_correct_particles(f); f->step_counter += 1; break;
        }
    }
}
