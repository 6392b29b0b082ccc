// fluid_kernels.hpp -- launchers of the non-PCG kernels (fluid_kernels.cu, transfer_kernels.cu).  All enqueue-only on `st`.
#pragma once
#include "../../include/blub_fluid.h"
#include "common.cuh"

namespace blub {

// np_upper: host-side upper bound of the particle count used to size the launch; the kernels guard with
// StepParams::num_particles (device), mirroring NumParticles in the reference's uniform buffer (hybrid_fluid.glsl:7-10).

// 1 bit per cell: "the cell is FLUID", x fastest, `wpr` 32-bit words per row of nx cells (rows start on a word).  Rebuilt by every
// pass that finishes a marker volume; the extrapolation works on it.
struct FluidBits {
    uint32_t *words; // wpr * ny * nz
    int wpr;
};

// Cells that hold more than 32 particles (see cell_canonicalize_kernel): list, per-cell table slot, and the table of their 18 face sums
// (one component at a time).
struct CrowdedCells {
    uint32_t *count;        // number of crowded cells of the current lists
    uint32_t *cells;        // their cell indices, max_num_particles / 33 + 1 entries
    uint32_t *slot_of_cell; // n entries, only valid for crowded cells
    float2 *sums;           // 18 per crowded cell
};

// Per-step cell lists (counting sort of particle indices by primal cell, canonical order inside a cell): the particles of cell c are
// order[cell_start[c] .. cell_start[c + 1]).
struct CellLists {
    uint32_t *cell_start; // n + 1 entries
    uint32_t *order;      // max_num_particles entries
    uint32_t *arrival;    // scratch: the lists in arrival order of the count atomics, before canonicalisation
    uint2 *cell_slot;     // scratch: (cell, arrival slot) per particle
    uint32_t *block_sums; // scratch of the scan
    CrowdedCells crowd;
};

// Brick schedule of the density and P2G scatters (transfer_kernels.cu, DESIGN.md §3.2): built from the cell lists at every re-sort; work
// items of aligned particle warps grouped by the cell brick they were sorted into.  It never changes a result, only how many faces go through a
// block's tile.  Kept on the device, so that a captured step graph follows a rebuild or an invalidation.
struct ScatterSchedule {
    uint32_t *valid;       // device word, non-zero: the schedule describes the particle order (cleared by anything else that re-indexes)
    uint32_t *brick_warps; // nbricks + 1: warps per brick, then their exclusive scan (entry nbricks: the warps it covers)
    uint32_t *brick_items; // nbricks + 1: work items per brick, then their exclusive scan (entry nbricks: the number of items)
    uint32_t *item_start;  // per item: its first entry of `warps`
    uint32_t *item_brick;  // per item: its brick
    int4 *item_box;        // per item: (lo, -), (hi, -) -- the primal cells its particles were in at the last density scatter (lo > hi: none)
    uint32_t *warps;       // warp ids (warp w = particles 32w .. 32w + 31), by brick, ascending within a brick
    int nbricks;
};
bool scatter_schedule_enabled(); // false under BLUB_SCATTER_SCHEDULE=off
int scatter_schedule_bricks(const GridDim &g);
uint32_t scatter_schedule_max_items(const GridDim &g, uint32_t max_warps);
// after launch_binning: builds the schedule from the cell_start of that binning and sets `valid`
void launch_scatter_schedule(cudaStream_t st, const GridDim &g, const CellLists &l, const ScatterSchedule &s);

void configure_transfer_kernels(); // once per device, before the first launch (dynamic shared memory opt-in)
// clamp_lo: 1.0 velocity transfer, 0.5 density transfer, 0.0 binning (see transfer_position)
void launch_cell_lists(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, float clamp_lo, const CellLists &l);
// particle_words (nullable): 1 bit per cell "a particle is in this cell", before the boundary rule
void launch_marker_from_lists(cudaStream_t st, const GridDim &g, const CellLists &l, int8_t *marker, const uint2 *vox, const FluidBits &bits,
                              uint32_t *particle_words);
void launch_p2g_gather(cudaStream_t st, const GridDim &g, const StepParams *params, const CellLists &l, const float4 *pos, float4 *const row[3],
                       const int8_t *marker, float *const u[3]);
// scatter form of P2G / density in two halves, for callers that exchange halos in between (z-slab sharding).  sched: the brick schedule, or
// one with valid == nullptr (z-slab ranks, BLUB_SCATTER_SCHEDULE=off): 256-particle chunks only.
void launch_p2g_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, float4 *const row[3],
                        longlong2 *const nw[3], int8_t *marker, bool clear_accumulators, const ScatterSchedule &sched);
// particle_words: wpr * ny * nz words, 1 bit per cell "a particle marked this cell" (before the boundary rule); the finish pass visits and
// re-zeroes the accumulators of the one-cell dilation of those cells only
void launch_p2g_finish(cudaStream_t st, const GridDim &g, const StepParams *params, float *const u[3], longlong2 *const nw[3], int8_t *marker,
                       const uint2 *vox, const FluidBits &bits, uint32_t *particle_words);
// density: 64-bit fixed-point accumulator volume (FIXED_WEIGHT_BITS, common.cuh).  sched: the brick schedule, or one with valid == nullptr
// (z-slab ranks, BLUB_SCATTER_SCHEDULE=off): 256-particle chunks only.
void launch_density_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, long long *density,
                            const ScatterSchedule &sched);
void launch_density_finish(cudaStream_t st, const GridDim &g, const StepParams *params, const int8_t *marker, const long long *density, float *rhs);
void launch_density_rhs(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos,
                        const int8_t *marker, long long *density, float *rhs, const ScatterSchedule &sched);
// Stage 7 with the density scatter fused in (one GPU): launch_advect, and the scatter of the new positions into `density`, which must be all
// zero.  launch_density_finish_sparse then writes the right-hand side of the FLUID cells and puts the density words back to zero, visiting
// the one-cell dilation of particle_words only: the words of a marker pass over the marker this advection left (launch_boundary_marker).
void launch_advect_density(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                           float *const u[3], const uint2 *vox, int8_t *marker, long long *density, const ScatterSchedule &sched);
void launch_density_finish_sparse(cudaStream_t st, const GridDim &g, const StepParams *params, const int8_t *marker, const FluidBits &bits,
                                  const uint32_t *particle_words, long long *density, float *rhs);
void launch_boundary_marker(cudaStream_t st, const GridDim &g, int8_t *marker, const uint2 *vox, const FluidBits &bits, uint32_t *particle_words = nullptr);
void launch_fluid_bits(cudaStream_t st, const GridDim &g, const int8_t *marker, const FluidBits &bits);
int binning_scan_blocks(const GridDim &g);
void launch_binning(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *src, float4 *dst, const CellLists &l);

// grid passes: they visit the cells within one cell of the fluid (FluidBits) and, with a solid volume, divergence_remove / position_change also
// those within two / one cells of a SOLID cell that holds a particle (DESIGN section 3.3); every other cell keeps its previous value
void launch_divergence_compute(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, float *const u[3], const uint2 *vox, float *rhs);
// particle_words (with a solid volume; nullptr without one): the words of the last marker pass -- the projection also visits the cells within
// two cells, the position change those within one cell of a SOLID cell that holds a particle (the faces such a particle reads)
// beta (nullptr: every face 1, the constant-density projection): the variable-density face coefficients of launch_tag_density, u -= beta (p_i - p_j)
void launch_divergence_remove(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const float *p, const uint2 *vox,
                              const uint32_t *particle_words, float *const u[3], const float *const *beta = nullptr);
void launch_extrapolate(cudaStream_t st, const GridDim &g, const FluidBits &bits, float *const u[3]);
void launch_clear_marker(cudaStream_t st, const GridDim &g, int8_t *marker);
void launch_advect(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                   float *const u[3], const uint2 *vox, int8_t *marker);
void launch_advect_migrate(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos, float4 *const row[3],
                           float *const u[3], const uint2 *vox, int8_t *marker, const MigrateOut &mig);
void launch_position_change(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker, const float *p,
                            const uint32_t *particle_words, float *const u[3]);
void launch_correct_particles(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, float4 *pos,
                              const int8_t *marker, float *const u[3]);

// exclusive scan of n 32-bit integers in place (the 3-kernel scan of the cell lists); block_sums: exclusive_scan_blocks(n) entries
int exclusive_scan_blocks(int64_t n);
void launch_exclusive_scan(cudaStream_t st, uint32_t *data, int64_t n, uint32_t *block_sums);

// ---- sources and drains (flow_kernels.cu, DESIGN.md §8 "Sources and drains") ----
constexpr int FLOW_MAX_BOXES = 16;
constexpr uint32_t FLOW_CHUNK = 1024; // particles per block-chunk of the drain compaction
struct FlowBox {
    int lo[3], hi[3]; // cells [lo, hi), clamped to [1, dim - 1]
};
// Passed by value: a change of the set drops the cached step graphs.
struct FlowSet {
    int num_sources, num_drains;
    FlowBox source[FLOW_MAX_BOXES], drain[FLOW_MAX_BOXES];
    float velocity[FLOW_MAX_BOXES][3];    // cells/s
    uint32_t tag[FLOW_MAX_BOXES];         // the particle tag every emitted particle of a source carries
    uint32_t source_base[FLOW_MAX_BOXES + 1]; // exclusive prefix of the source box volumes: index of a box's first cell in the source cell list
};
struct FlowScratch {
    uint32_t *chunk_drained;      // drained particles per FLOW_CHUNK chunk, then their exclusive scan
    uint32_t *source_count;       // particles per source cell (source_base order, x fastest within a box)
    uint32_t *emit_offsets;       // particles to emit per source cell, then their exclusive scan (one more entry: the total)
    uint32_t *scan_sums;          // block sums of both scans
    uint32_t *scalars;            // [0] first drained index (~0u: none), [1] drained this step, [2] count before the prologue
    unsigned long long *counters; // cumulative emitted, drained, refused for capacity
    uint32_t num_chunks, source_cells;
};
// Drain, count, emit and set the source velocity (in that order, see DESIGN.md); the particle count lives in params->num_particles.
// pos_spare / row_spare: arrays of the same capacity the drain compaction writes into before it copies the suffix back.
// schedule_valid: the scatter schedule's flag (or nullptr), cleared when the drains remove particles
void launch_flow_prologue(cudaStream_t st, const GridDim &g, StepParams *params, uint32_t capacity, const FlowSet &fs, const FlowScratch &s, float4 *pos,
                          float4 *pos_spare, float4 *const row[3], float4 *const row_spare[3], const uint2 *vox, uint32_t *schedule_valid);

// ---- particle tags (flow_kernels.cu, DESIGN.md §8 "Particle tags"): the raw bits of the fourth word of every position ----
constexpr uint32_t TAG_CENSUS_MAX = 256; // tags per census: the block-private table
// The particle count: params->num_particles when `params` is not null (device-count mode), else `n_host`.  np_upper sizes the launch.
void launch_paint_tags(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t n_host, uint32_t np_upper, const FlowBox &box, uint32_t tag,
                       float4 *pos);
// out: num_tags device records, count / sums zero and bounds at INT32_MAX / INT32_MIN on entry
void launch_tag_census(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t n_host, uint32_t np_upper, uint32_t first, uint32_t num_tags,
                       const float4 *pos, float4 *const row[3], BlubTagCensus *out);

// ---- solid load probes (load_kernels.cu, DESIGN.md §8 "Solid load probes") ----
constexpr int LOAD_PROBES_MAX = BLUB_LOAD_PROBES_MAX;
constexpr uint32_t LOAD_HISTORY_LENGTH = BLUB_LOAD_HISTORY_LENGTH;
struct LoadProbeBox {
    int lo[3], hi[3]; // cells [lo, hi), clamped to [0, dim]
    float pivot[3];   // grid cells
};
// One record per probe into ring[probe * LOAD_HISTORY_LENGTH + params->step_count % LOAD_HISTORY_LENGTH]: the slot is zeroed, then every
// wetted face of the probe's box adds its fixed-point force and torque.  probes: num_probes device boxes; max_cells: cells of the largest box
// (sizes the launch).  marker / p_vel: the volumes the velocity solve used.
void launch_solid_loads(cudaStream_t st, const GridDim &g, const StepParams *params, int num_probes, uint32_t max_cells, const LoadProbeBox *probes,
                        const int8_t *marker, const float *p_vel, BlubSolidLoad *ring);

// ---- floating bodies (body_kernels.cu, DESIGN.md §8 "Floating bodies") ----
constexpr int BODIES_MAX = BLUB_BODIES_MAX;
constexpr uint32_t BODY_HISTORY_LENGTH = BLUB_BODY_HISTORY_LENGTH;
// The cells a launch walks around each body: a cube of `cube` cells per side from floor(c - e), sized at set time from the largest bounding
// sphere, so that a captured graph stays valid while the bodies move and turn.
uint32_t body_cube_side(const BlubBody &b);
// Mesh bodies (shape 2, DESIGN.md §8 "Mesh bodies"): what the device needs of body slot i beyond its BlubBody.
struct MeshBodyDev {
    float mass, inertia[3]; // per unit fluid density: the integrator's m and I_b
    float mid[3];           // (lo + hi) / 2 of the body-frame bounds; the BlubBody's half_extent is (hi - lo) / 2
    uint32_t first_vertex, num_vertices, first_triangle, num_triangles; // into the set's arrays; num_triangles == 0: a box or sphere
};
// What the body kernels read of the mesh bodies: info == nullptr when the set has none.  bits: num_bodies x cube x cube rows of `words`
// 32-bit words over each body's launch cube, bit x of row (z, y) = the cell's centre lies inside the mesh.
struct MeshBodies {
    const MeshBodyDev *info = nullptr;
    const uint32_t *bits = nullptr;
    uint32_t words = 0;
    const int *origin = nullptr; // 3 per body: the first cell of its launch cube at the step's pose, written with the bits
};
// The device arrays of a set with mesh bodies (allocated by HybridFluid::restore_bodies).
struct MeshBodySet {
    MeshBodyDev *info = nullptr;    // BODIES_MAX slots
    float *body_vertices = nullptr; // xyz per vertex, body frame
    float *grid_vertices = nullptr; // xyz per vertex at the current pose: stage 0 scratch
    uint32_t *indices = nullptr;    // 3 per triangle, into the vertex arrays
    uint32_t *bits = nullptr;
    int *origin = nullptr;          // BODIES_MAX x 3
    uint32_t words = 0, max_vertices = 0, max_triangles = 0; // the largest body's counts size the launches
    MeshBodies view() const { return {info, bits, words, origin}; }
};
// Stage 0, before the composite kernel: zero the bits, move every mesh body's vertices to the grid, flip the crossing bit of every covered
// cell-centre row, then turn each row into its crossing parity.
void launch_mesh_body_fill(cudaStream_t st, const GridDim &g, int num_bodies, uint32_t cube, const BlubBody *bodies, const MeshBodySet &mesh);
// Stage 0: the composite solid volume (n cells of RGBA16F) = the borrowed volume (or zero when vox == nullptr), then every body written over it.
void launch_body_composite(cudaStream_t st, const GridDim &g, const uint2 *vox, uint2 *composite, int num_bodies, uint32_t cube, const BlubBody *bodies,
                           const MeshBodies &mesh);
// End of stage 2: every body's wetted-face sums into sums[8 * body] (zero on entry), then the integrator: it reads and re-zeroes the sums,
// moves every body and writes its record into ring[body * BODY_HISTORY_LENGTH + params->step_count % BODY_HISTORY_LENGTH].
void launch_body_step(cudaStream_t st, const GridDim &g, const StepParams *params, int num_bodies, uint32_t cube, BlubBody *bodies, const int8_t *marker,
                      const float *p_vel, unsigned long long *sums, BlubBodyRecord *ring, const MeshBodies &mesh);
// Host twins of the device rules the setter checks a body against: the half extents of its grid-axis bounding box at its pose.
void body_bounding_extents(const BlubBody &b, float e[3]);

// ---- viscous liquids (viscosity_kernels.cu, DESIGN.md §8 "Viscous liquids") ----
// What the last viscosity solve left on the device.
struct ViscositySolveInfo {
    int iterations;
    float max_error[3]; // max |r| per component, cells/s
};
// Working memory of the viscosity stage, allocated with the first viscosity above zero: 28 bytes per cell.
struct ViscosityWork {
    uint32_t *codes = nullptr;                   // n: three 10-bit face codes per cell
    float *r[3] = {nullptr, nullptr, nullptr};   // n each: the right-hand side, then the residual
    float *s[3] = {nullptr, nullptr, nullptr};   // n each: the search direction
    uint32_t *word_flags = nullptr;              // words + 1: "the word holds a live face", then their exclusive scan (last entry: the number of active words)
    uint32_t *words = nullptr;                   // the active 32-cell words, ascending
    uint32_t *scan_sums = nullptr;               // block sums of the scan
    float *partials = nullptr;                   // 2 x 6 x blocks: the blocks' partial sums and maxima, alternating between rounds
    unsigned *barrier = nullptr;                 // arrival counter of the solve's grid-wide rounds
    BlubViscosity *block = nullptr;              // what the kernels read of the setting: a change does not invalidate a captured graph
    ViscositySolveInfo *info = nullptr;
    int blocks = 0;                              // the solve's resident grid
    int pair_blocks = 0;                         // the same for the per-pair solve (a tag viscosity table; partials are sized for the larger)
};
// SMs x resident blocks per SM of the constant (pairs = false) or the per-pair solve; throws CudaError without cooperative launch
int viscosity_solve_blocks(bool pairs = false);

// ---- liquids of different viscosities (viscosity_kernels.cu, DESIGN.md §8 "Liquids of different viscosities") ----
constexpr int TAG_VISCOSITIES_MAX = BLUB_TAG_VISCOSITIES_MAX;
constexpr int TAG_VISCOSITY_FRAC_BITS = 32; // a particle adds rint(nu_tag / nu_scale * 2^32) to its cell's sum
// What the kernels read of the table and of the fluid's nu: a change does not invalidate a captured graph.
struct TagViscosityBlock {
    uint32_t count;
    uint32_t tag[TAG_VISCOSITIES_MAX];
    unsigned long long q[TAG_VISCOSITIES_MAX]; // rint(nu_tag / nu_scale * 2^32), at most 2^32
    unsigned long long q_default;              // the same for the tags not in the table (the fluid's nu)
    float nu_scale;                            // the largest of the table's values and the fluid's nu (> 0 while the stage runs)
    float nu_fluid;                            // the fluid's nu: a FLUID cell without a particle
};
// Working memory, allocated with the first non-empty table: 64 bytes per cell.  k[c][i] = (k_{+x}, k_{+y}, k_{+z}, 1 + sum of the face's
// k_fn) of face i of component c, k_{+d} the pair coefficient k_fn with its +d neighbour face; the -d one is component d of k[c][i - e_d].
// Written on live faces only.  k[c] = k[0] + c n: the solve addresses them from one pointer.
struct TagViscosityWork {
    float4 *k[3] = {};                 // n each
    unsigned long long *sum = nullptr; // n: sum of the cell's particles' q; zero between stages 0
    uint32_t *count = nullptr;         // n: the cell's particles; zero between stages 0
    float *nu = nullptr;               // n: nu_i of the last stage 0 on FLUID cells, 0 elsewhere
    TagViscosityBlock *block = nullptr;
};

// Stage 0 of a tag viscosity table, after P2G: the cell viscosities w.nu of the live particles (params->num_particles when device_count, else
// n_host; np_upper sizes the launch) and the marker.  Leaves sum and count zero.  The scatter is the tag density one (tag_density_kernels.cu).
void launch_tag_viscosity_cells(cudaStream_t st, const GridDim &g, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper,
                                const float4 *pos, const int8_t *marker, const TagViscosityWork &w);
// The whole stage: classify the faces and list the active words from the FLUID bits and the marker, then solve all three components in one
// cooperative launch; k = block->kinematic_viscosity * params->dt is formed on the device.  Writes live faces of u only.  With `tag` (a
// non-empty table), first the cell viscosities of the live particles (params->num_particles when device_count, else n_host; np_upper sizes
// the launch), then the system with per-pair coefficients k_fn = nu_fn * params->dt.
void launch_viscosity(cudaStream_t st, const GridDim &g, const StepParams *params, const FluidBits &bits, const int8_t *marker, const uint2 *vox,
                      float *const u[3], const ViscosityWork &w, const TagViscosityWork *tag = nullptr, bool device_count = false,
                      uint32_t n_host = 0, uint32_t np_upper = 0, const float4 *pos = nullptr);

// ---- CFL-limited substeps (cfl_kernels.cu, DESIGN.md §8 "CFL-limited substeps") ----
// out[c] = the bits of max |v_c| over the particles (params->num_particles when `params` is not null, else n_host; np_upper sizes the launch).
// Zeroes the three words first.
void launch_max_particle_velocity(cudaStream_t st, const StepParams *params, uint32_t n_host, uint32_t np_upper, float4 *const row[3], uint32_t *out);

// ---- moving tanks (tank_kernels.cu, DESIGN.md §8 "Moving tanks") ----
// Stage 0 of a rotating frame, before P2G: every live particle's rows rotated by params->tank_q, plus the force params->tank_k (x - tank_pivot).
// The count: params->num_particles when device_count, else n_host; np_upper sizes the launch.
void launch_tank_frame(cudaStream_t st, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper, const float4 *pos,
                       float4 *const row[3]);

// ---- surface tension (surface_tension_kernels.cu, DESIGN.md §8 "Surface tension") ----
// Working memory, allocated with the first surface tension above zero: 12 bytes per cell.
struct SurfaceTensionWork {
    long long *psi = nullptr; // n: the wall-ruled splat (2^-32 particle weights), valid within 3 cells of FLUID
    float *kappa = nullptr;   // n: the curvature of the last stage 1 in the band (cells^-1), 0 elsewhere
    float *sigma = nullptr;   // the kinematic surface tension the kernels read (cells^3/s^2): a change does not invalidate a captured graph
};
// Stage 1: the wall rule on the splat in `density`, the smoothed field phi written back into `density` (within 2 cells of FLUID), the
// curvature into w.kappa.  `density` must hold the splat of the current positions (launch_density_scatter).
void launch_surface_curvature(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, long long *density,
                              const SurfaceTensionWork &w);
// Stage 1, after the divergence: rhs += the ghost values of every FLUID cell's AIR faces.  Writes FLUID cells only.
void launch_surface_rhs(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                        const SurfaceTensionWork &w, float *rhs);
// Stage 4, after the projection: the FLUID-AIR faces get the ghost value the solve assumed.
void launch_surface_faces(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                          const SurfaceTensionWork &w, float *const u[3]);

// ---- interfacial tension (surface_tension_kernels.cu, DESIGN.md §8 "Interfacial tension") ----
constexpr int INTERFACE_TAGS_MAX = BLUB_INTERFACE_TAGS_MAX;
// What the kernels read of the setting: a change between two values above zero does not invalidate a captured graph.
struct InterfacialTensionBlock {
    float s;        // the kinematic interfacial tension (cells^3/s^2)
    uint32_t count; // phase B: the particles whose tag is one of tag[0, count); the unused entries are 0
    uint32_t tag[INTERFACE_TAGS_MAX];
};
// Working memory, allocated with the first interfacial tension above zero: 20 bytes per cell.
struct InterfacialTensionWork {
    long long *phi = nullptr;   // n: the phase-B splat (2^-40), then the smoothed phase field phi (2^-32), valid within 2 cells of FLUID
    long long *psi = nullptr;   // n: the wall-ruled phase field, valid within 3 cells of FLUID
    float *kappa = nullptr;     // n: the interface's curvature of the last stage 1 in the band (cells^-1), 0 elsewhere
    InterfacialTensionBlock *block = nullptr;
};
// The phase-B splat: launch_density_scatter of the particles whose tag the block lists into `density` (zeroed first).
void launch_phase_scatter(cudaStream_t st, const GridDim &g, const StepParams *params, uint32_t np_upper, const float4 *pos, long long *density,
                          const ScatterSchedule &sched, const InterfacialTensionBlock *blk);
// Stage 1: the phase field of the splat of every particle in `splat_all` and of the phase-B particles in w.phi (launch_phase_scatter), in
// two parts so that the free surface can reuse `splat_all` in between: launch_interface_psi reads both splats into w.psi, then
// launch_interface_curvature smooths w.psi into w.phi and measures the curvature into w.kappa.
void launch_interface_psi(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const long long *splat_all,
                          const InterfacialTensionWork &w);
void launch_interface_curvature(cudaStream_t st, const GridDim &g, const FluidBits &bits, const int8_t *marker, const InterfacialTensionWork &w);
// Stage 1, after the divergence (and the free surface's terms): rhs += +-beta_f g_f over every band cell's interface faces.  `beta`: the
// density table's face arrays, nullptr without a table (beta_f = 1).
void launch_interface_rhs(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                          const InterfacialTensionWork &w, const float *const *beta, float *rhs);
// Stage 4, after the projection: the interface faces get the beta_f g_f the solve assumed.
void launch_interface_faces(cudaStream_t st, const GridDim &g, const FluidBits &bits, const StepParams *params, const int8_t *marker,
                            const InterfacialTensionWork &w, const float *const *beta, float *const u[3]);

// ---- liquids of different densities (tag_density_kernels.cu, DESIGN.md §8 "Liquids of different densities") ----
constexpr int TAG_DENSITIES_MAX = BLUB_TAG_DENSITIES_MAX;
constexpr int TAG_DENSITY_FRAC_BITS = 20; // a particle adds rint(rho * 2^20) to its cell's sum
// What the kernels read of the table: a change does not invalidate a captured graph.
struct TagDensityBlock {
    uint32_t count;
    uint32_t tag[TAG_DENSITIES_MAX];
    uint32_t q[TAG_DENSITIES_MAX]; // rint(relative_density * 2^20)
};
// Working memory, allocated with the first non-empty table: 36 bytes per cell.  The face arrays follow divergence_remove's layout: beta[c][i]
// is the face between cell i and its +c neighbour.
struct TagDensityWork {
    unsigned long long *sum = nullptr; // n: sum of rint(rho * 2^20) over the cell's particles; zero between stages 0
    uint32_t *count = nullptr;         // n: the cell's particles; zero between stages 0
    float *rho = nullptr;              // padded: rho_i of the last stage 0 on FLUID cells, 0 elsewhere
    float *beta[3] = {nullptr, nullptr, nullptr}; // padded: the face coefficients, 0 on faces with a SOLID side or no FLUID side
    float *diag = nullptr;             // padded: D_i, the sum of a FLUID cell's face coefficients (0 elsewhere)
    float *inv_diag2 = nullptr;        // padded: 1 / D_i^2 (1 where D_i = 0 and on every cell that is not FLUID)
    TagDensityBlock *block = nullptr;
    void *volumes = nullptr;           // the one allocation of the six padded float volumes above
};
// Stage 0, after P2G: the cell densities of the live particles (params->num_particles when device_count, else n_host; np_upper sizes the
// launch), then the face coefficients, the diagonal and the preconditioner from them and the marker.  Leaves sum and count zero.
void launch_tag_density(cudaStream_t st, const GridDim &g, const StepParams *params, bool device_count, uint32_t n_host, uint32_t np_upper,
                        const float4 *pos, const int8_t *marker, const TagDensityWork &w);

// ---- whitewater (whitewater_kernels.cu, DESIGN.md §8 "Whitewater") ----
// Xored into the (step << 32 | cell) seed of a cell's emission draws.  The low half has bit 31 set and a cell index is below 2^31, so no
// whitewater seed equals a seed of the flow prologue's emission.
constexpr uint64_t WHITEWATER_SEED_KEY = 0xD1B54A32D192ED03ull;
// The device counters: cumulative emitted, removed and refused for capacity; the live count; the survivors of the running update.
struct WhitewaterCounters {
    unsigned long long emitted, removed, refused;
    uint32_t count, survivors;
};
// Storage, allocated by the setter with a capacity above zero: 64 bytes per particle and 4 per cell.  pos[0] / vel[0] hold the live particles
// between steps (position xyz and lifetime in s; velocity xyz in cells/s and the kind's bits), pos[1] / vel[1] what the update made of them.
struct WhitewaterWork {
    float4 *pos[2] = {nullptr, nullptr}, *vel[2] = {nullptr, nullptr};
    uint32_t *flags = nullptr;       // capacity + 1: "the particle survives", then their exclusive scan
    uint32_t *cell_counts = nullptr; // n + 1: the particles each cell emits, then their exclusive scan
    uint32_t *scan_sums = nullptr;   // block sums of both scans
    WhitewaterCounters *counters = nullptr;
    uint32_t capacity = 0;
};
// The pass at the end of stage 5 (update, stable compaction, emission from the surface band), reading the projected and extrapolated u, the
// marker of this step's P2G and its FLUID bits, and the solid volume `vox` (may be nullptr).  Writes only w.
void launch_whitewater(cudaStream_t st, const GridDim &g, const StepParams *params, const FluidBits &bits, const int8_t *marker, float *const u[3],
                       const uint2 *vox, const BlubWhitewater &s, const WhitewaterWork &w);

} // namespace blub
