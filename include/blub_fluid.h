/*
 * blub_fluid.h -- C ABI of libblubcore.so, the H100-native APIC/FLIP fluid-step core.
 *
 * Drop-in boundary for Wumpf/blub's `HybridFluid` (src/simulation/hybrid_fluid.rs) and its
 * `PressureSolver`/`PressureField` (src/simulation/pressure_solver.rs).  The reference has no
 * FFI/plugin layer: its narrowest seam is the Rust method set of `HybridFluid`, whose arguments are
 * wgpu objects.  Every entry point below names the reference method it replaces (file:line relative
 * to the reference checkout); wgpu handles become plain device pointers, a CUDA stream and POD structs.
 * INTEGRATION.md shows the Rust `extern "C"` block a maintainer would add.
 *
 * Conventions kept from the reference:
 *   - positions in grid cells, velocities in cells/s, pressure pre-multiplied by dt/rho
 *     (shader/simulation/divergence_compute.comp:4-5);
 *   - the fluid owns all of its device memory; the solid-voxel volume is BORROWED and must outlive
 *     the steps that use it (hybrid_fluid.rs:99,266);
 *   - single host thread, one stream in submission order; `blub_fluid_step` only ENQUEUES work and
 *     never blocks on the GPU (README.md:94-103); the only device->host traffic is the 8-byte solver
 *     statistics read-back, which is asynchronous and may lag (pressure_solver.rs:148-209);
 *   - the reference panics on set-up failure and only logs at run time; here every fallible call
 *     returns an int code and nothing throws across the boundary.
 * There is NO CPU fallback: every call fails with BLUB_ERR_CUDA if no usable sm_90 (H100) device exists.
 */
#ifndef BLUB_FLUID_H
#define BLUB_FLUID_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BLUB_OK 0
#define BLUB_ERR_INVALID_ARGUMENT 1
#define BLUB_ERR_CUDA 2
#define BLUB_ERR_OUT_OF_MEMORY 3
#define BLUB_ERR_IO 4
#define BLUB_ERR_PARSE 5
#define BLUB_WARN_TRUNCATED 100 /* add_cube hit max_num_particles: hybrid_fluid.rs:627-633 logs + truncates */

/* HybridFluid::PARTICLES_PER_GRID_CELL, hybrid_fluid.rs:90 (read by the renderer for the particle radius) */
#define BLUB_PARTICLES_PER_GRID_CELL 8

/* marker values, shader/simulation/hybrid_fluid.glsl:20-23 (stored as int8 instead of R8Snorm) */
#define BLUB_CELL_SOLID 0
#define BLUB_CELL_FLUID 1
#define BLUB_CELL_AIR (-1)

typedef struct BlubFluid BlubFluid; /* opaque; owns its buffers like HybridFluid (hybrid_fluid.rs:24-72) */

/* SolverConfig, pressure_solver.rs:57-62; defaults 0.1 / 32 / 4 (hybrid_fluid.rs:253-257) */
typedef struct {
    float error_tolerance;        /* on max|r| * dt */
    int32_t max_num_iterations;
    int32_t error_check_frequency;
} BlubSolverConfig;

/* SolverStatisticSample, pressure_solver.rs:63-68; error = max|r| * dt (pressure_solver.rs:162) */
typedef struct {
    float error;
    int32_t iteration_count;
} BlubSolverSample;

/* Behaviour switches for the reference's driver-defined / buggy spots (SURVEY.md Appendix B). */
typedef struct {
    int32_t precond_mode;   /* 0 = z = r/diag^2 (LOD-1 fetch returns 0, default), 1 = as written with clamped LOD */
    int32_t reserved[7];
} BlubQuirks;

/* The ten read-only resources of HybridFluid::bind_group_renderer (hybrid_fluid.rs:351-369,700-713). */
typedef struct {
    const void *particles_position_ll;            /* num_particles x {float3 pos, uint32 tag} (see "particle tags") */
    const void *particles_velocity_x;             /* num_particles x float4 (C column xyz, v_x)   */
    const void *particles_velocity_y;
    const void *particles_velocity_z;
    const float *grid_velocity_x;                 /* nx*ny*nz, x fastest, value on the +x face     */
    const float *grid_velocity_y;
    const float *grid_velocity_z;
    const int8_t *marker;                         /* BLUB_CELL_*                                   */
    const float *pressure_from_velocity;
    const float *pressure_from_density;
} BlubFluidView;

/* HybridFluid::new, hybrid_fluid.rs:92-100.  Grid dimensions must be multiples of 8 (the reference dispatches
 * 8^3 groups without guards) and nx*ny*nz > 16384 (pressure_solver.rs:551).  `cuda_stream` is a cudaStream_t
 * (NULL = a private non-blocking stream owned by the fluid). */
int blub_fluid_create(BlubFluid **out, uint32_t nx, uint32_t ny, uint32_t nz, uint32_t max_num_particles, int device,
                      void *cuda_stream);
void blub_fluid_destroy(BlubFluid *fluid);

/* HybridFluid::add_fluid_cube, hybrid_fluid.rs:620-678: cell-aligned cube, corners clamped to [1, dim-1], 8
 * stratified-jittered particles per cell (xoshiro256++ seeded with the new particle count, :637).
 * Returns BLUB_WARN_TRUNCATED when max_num_particles was hit. */
int blub_fluid_add_cube(BlubFluid *fluid, const float min_grid[3], const float max_grid[3]);
/* HybridFluid::set_gravity_grid, :692 (world gravity / grid_to_world_scale, src/scene/mod.rs:139) */
int blub_fluid_set_gravity_grid(BlubFluid *fluid, const float gravity_grid[3]);
/* HybridFluid::num_particles / num_active_particles, :696,:731 */
uint32_t blub_fluid_num_particles(const BlubFluid *fluid);
/* HybridFluid::grid_dimension, :727 */
void blub_fluid_grid_dimension(const BlubFluid *fluid, uint32_t out[3]);

/* HybridFluid::pressure_solver_config_{velocity,density}, :743-749: mutable reference semantics.
 * which: 0 = velocity (divergence) solve, 1 = density solve. */
BlubSolverConfig *blub_fluid_solver_config(BlubFluid *fluid, int which);
/* HybridFluid::dynamic_settings().particle_rebinning_step_frequency, :19-22,:751; 0 disables (:854) */
uint32_t *blub_fluid_rebinning_frequency(BlubFluid *fluid);
/* HybridFluid::pressure_solver_stats_{velocity,density}, :753-761: newest <= 100 samples, oldest first */
size_t blub_fluid_solver_stats(const BlubFluid *fluid, int which, BlubSolverSample *out, size_t cap);
/* HybridFluid::update_statistics, :765: collect finished asynchronous read-backs (never blocks) */
void blub_fluid_update_statistics(BlubFluid *fluid);

/* The SceneVoxelization view bound at set 1 / binding 1 (hybrid_fluid.rs:266, src/scene/voxelization.rs:17):
 * nx*ny*nz RGBA16F texels in device memory, xyz = solid velocity in cells/s, w != 0 => solid.
 * NULL = no solids.  Borrowed. */
int blub_fluid_set_solid_voxels(BlubFluid *fluid, const void *rgba16f_device_ptr);

/* HybridFluid::step, hybrid_fluid.rs:770-977.  Enqueues one simulation step on the fluid's stream. */
int blub_fluid_step(BlubFluid *fluid, double simulation_delta_seconds);

/* bind_group_renderer, :351-369,:723 */
int blub_fluid_view(const BlubFluid *fluid, BlubFluidView *out);

int blub_fluid_set_quirks(BlubFluid *fluid, const BlubQuirks *quirks);
/* Wait for everything enqueued so far (the reference's device.poll(Maintain::Wait), simulation_controller.rs:140). */
int blub_fluid_synchronize(BlubFluid *fluid);
const char *blub_last_error(void);
const char *blub_version(void);

/* ---- checkpoint / restart (not part of the reference surface; file format: DESIGN.md section 8) ------------------------------ */
/* Everything a later step depends on (particles in their array order, grid velocities, marker, both pressure warm starts, step
 * counter, solver configs / paths, transfer path, graph replay, gravity, rebinning settings, quirks, solver statistics), written after
 * everything enqueued so far has finished (synchronises).  The file is written as `path`.tmp, flushed to disk and renamed over `path`.
 * Only between whole steps: a fluid whose last blub_fluid_step_stages call did not end at stage 14, and z-slab ranks, are refused with
 * BLUB_ERR_INVALID_ARGUMENT.  BLUB_ERR_IO: the file cannot be written. */
int blub_fluid_save_state(BlubFluid *fluid, const char *path);
/* A new fluid on `device` whose next step is bit for bit the step the saved fluid would have taken next (same library build, same
 * GPU model).  The file's settings win over the BLUB_* environment variables.  The solid-voxel volume is not part of the state:
 * attach it again with blub_fluid_set_solid_voxels.  BLUB_ERR_IO: the file cannot be opened or read; BLUB_ERR_PARSE: bad magic, format
 * version or checksum, truncated file, or a size that disagrees with the header (all sizes are checked before anything is allocated). */
int blub_fluid_load_state(BlubFluid **out, const char *path, int device, void *cuda_stream);
/* Host only, no device needed: validates the whole file (magic, version, sizes, checksums) and reports what it holds. */
typedef struct {
    uint32_t grid_dimension[3];
    uint32_t max_num_particles, num_particles, step_count, format_version;
} BlubStateInfo;
int blub_state_info(const char *path, BlubStateInfo *out);
/* number of whole steps this fluid has taken (restored by blub_fluid_load_state) */
uint32_t blub_fluid_step_count(const BlubFluid *fluid);

/* ---- sources and drains (not part of the reference surface; rules: DESIGN.md section 8) ---------------------------------------- */
/* Boxes in grid cells, corners clamped to [1, dim - 1] as blub_fluid_add_cube clamps them (the max corner is exclusive).  At the start of
 * every step the fluid removes the particles whose cell lies in a drain box (survivors keep their order), tops every source cell that holds
 * fewer than 4 particles and is neither solid nor a border cell up to 8 (appended after the survivors, up to max_num_particles), and gives
 * every particle in a source cell the source velocity (cells/s) with C = 0. */
typedef struct {
    float min_grid[3], max_grid[3], velocity_grid[3];
} BlubFluidSource;
typedef struct {
    float min_grid[3], max_grid[3];
} BlubFluidDrain;
/* Replaces the whole flow set; 0 / 0 clears it.  At most 16 boxes of each kind.  BLUB_ERR_INVALID_ARGUMENT, changing nothing: a non-finite
 * value, a box empty after clamping, two overlapping sources, a source overlapping a drain, too many boxes, a z-slab rank, or a fluid left
 * inside a step by blub_fluid_step_stages.  While the set is not empty the particle count lives on the device: blub_fluid_num_particles
 * then synchronises. */
int blub_fluid_set_flow(BlubFluid *fluid, const BlubFluidSource *sources, uint32_t num_sources, const BlubFluidDrain *drains, uint32_t num_drains);
/* Cumulative counts since the fluid was created (or saved): out[0] emitted, out[1] drained, out[2] refused for capacity.  Synchronises. */
int blub_fluid_flow_counters(BlubFluid *fluid, uint64_t out[3]);
/* 1 when the fluid has a non-empty flow set, 0 when not or when fluid is NULL */
int blub_fluid_has_flow(const BlubFluid *fluid);

/* ---- particle tags (not part of the reference surface; rules: DESIGN.md section 8) ---------------------------------------------
 * The fourth word of every particle position is its tag: a uint32 stored as raw bits, which no step reads and every path copies (binning,
 * re-sort, drain compaction, z-slab migration, checkpoints).  A fluid whose tags are all 0 computes exactly what it computed before tags
 * existed.  Tags are set by blub_fluid_add_cube_tagged (the new particles), by the sources of blub_fluid_set_flow_tagged (every particle they
 * emit), by blub_fluid_paint_tags, and directly through the fourth word of blub_fluid_set_particles / blub_fluid_upload(BLUB_TAP_PARTICLE_POS).
 * Non-zero bits written there are kept by the binning (before tags existed it zeroed the word). */
/* blub_fluid_add_cube with every new particle tagged `tag` (blub_fluid_add_cube is tag 0) */
int blub_fluid_add_cube_tagged(BlubFluid *fluid, const float min_grid[3], const float max_grid[3], uint32_t tag);
/* blub_fluid_set_flow with a tag per source (NULL = all 0; blub_fluid_set_flow passes NULL): the particles a source emits carry its tag,
 * particles already in a source cell keep theirs */
int blub_fluid_set_flow_tagged(BlubFluid *fluid, const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources,
                               const BlubFluidDrain *drains, uint32_t num_drains);
/* Tags every particle whose cell (the drains' cell rule) lies in the box, corners clamped as blub_fluid_add_cube clamps them (max exclusive).
 * Stream-ordered, never synchronises; works on the device-resident count while a flow set is active.  BLUB_ERR_INVALID_ARGUMENT, changing
 * nothing: a non-finite corner, a box empty after clamping, a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_paint_tags(BlubFluid *fluid, const float min_grid[3], const float max_grid[3], uint32_t tag);
/* What the particles of one tag add up to.  Sums are 2^16 fixed point: every particle contributes rint(value * 65536) (round to nearest
 * even; the product is exact), added as int64, so they are exact and independent of the particle order.  They stay exact for positions below
 * 2^10 cells, |v| <= 2^20 cells/s and at most 2^26 particles per tag.  Cells by the drains' rule; count == 0: cell_min = INT32_MAX,
 * cell_max = INT32_MIN. */
#define BLUB_TAG_CENSUS_FRAC_BITS 16
typedef struct {
    uint64_t count;
    int64_t position_sum_fx[3], velocity_sum_fx[3]; /* velocity component c = .w of velocity row c */
    int32_t cell_min[3], cell_max[3];
} BlubTagCensus;
/* out[k] = census of tag first_tag + k for k < num_tags; particles with other tags are skipped.  On a z-slab rank: this rank's particles.
 * Synchronises.  BLUB_ERR_INVALID_ARGUMENT: num_tags of 0 or above 256, or first_tag + num_tags above 2^32. */
int blub_fluid_tag_census(BlubFluid *fluid, uint32_t first_tag, uint32_t num_tags, BlubTagCensus *out);

/* ---- solid load probes (not part of the reference surface; rules: DESIGN.md section 8) -----------------------------------------
 * A probe is a box of cells plus a pivot, in grid cells.  The corners are converted as blub_fluid_add_cube converts them but clamped to
 * [0, dim] (the border cells, the tank walls, can be held); the max corner is exclusive.  While a fluid has probes, every step adds up on the
 * GPU, right after the velocity solve, the projection pressure on every wetted face of each probe: a face between a SOLID cell inside the box
 * and a FLUID neighbour (which may lie outside it).  q = -p_vel[fluid cell] * inv_dt (float32) is pressure / density (the velocity solve's
 * volume, BLUB_TAP_PRESSURE_VELOCITY, holds -p dt / density); the face force is q
 * along the face axis, from the fluid cell into the solid one, and the torque is (face centre - pivot) x force.  Every face contributes
 * rint(q * 2^16) to the force sums and rint((r_b * q) * 2^8) to the torque sums, added as int64: the records are exact and independent of the
 * launch order.  They are exact while |q| < 2^22, |r| < 2^11 and a probe has at most 2^21 wetted faces.
 * Units: force per unit fluid density in cells^4/s^2 (newtons = value * density * s^4, s = grid_to_world_scale in m per cell); torque
 * in cells^5/s^2 (times density * s^5).  Only the pressure of the velocity projection is measured: no density-correction pressure, no shear.
 * Probes are not part of the saved state: a loaded fluid has none. */
#define BLUB_LOAD_PROBES_MAX 16
#define BLUB_LOAD_HISTORY_LENGTH 1024 /* records per probe in the device ring: slot = step % 1024 */
#define BLUB_LOAD_FORCE_FRAC_BITS 16
#define BLUB_LOAD_TORQUE_FRAC_BITS 8
typedef struct {
    float min_grid[3], max_grid[3], pivot_grid[3];
} BlubLoadProbe;
typedef struct {
    uint32_t step;         /* blub_fluid_step_count before the step that wrote the record */
    uint32_t wetted_faces;
    int64_t force_fx[3];   /* force * 2^16 */
    int64_t torque_fx[3];  /* torque * 2^8 */
} BlubSolidLoad;
/* Replaces the whole probe set (0 clears it), resets the history and drops the cached step graphs.  Every step then records one
 * BlubSolidLoad per probe on the device without synchronising.  BLUB_ERR_INVALID_ARGUMENT, changing nothing: more than 16 probes, a
 * non-finite corner or pivot, a box empty after clamping, a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_load_probes(BlubFluid *fluid, const BlubLoadProbe *probes, uint32_t num_probes);
/* The newest min(capacity, recorded, 1024) records of probe `probe`, oldest first; *count receives their number.  Synchronises; works
 * inside a step as well (after stage 2 the record of the current step is there).  BLUB_ERR_INVALID_ARGUMENT: a probe index outside the set. */
int blub_fluid_load_history(BlubFluid *fluid, uint32_t probe, BlubSolidLoad *out, uint32_t capacity, uint32_t *count);
/* Host only: the cells [lo, hi) a probe holds on a grid of `dim` cells.  BLUB_ERR_INVALID_ARGUMENT: a non-finite value or an empty box. */
int blub_load_probe_cells(const uint32_t dim[3], const BlubLoadProbe *probe, uint32_t lo[3], uint32_t hi[3]);

/* ---- floating bodies (not part of the reference surface; rules: DESIGN.md section 8) -------------------------------------------
 * A body is an oriented box (half extents) or a sphere (radius = half_extent[0]) in grid cells whose pose lives on the device and which the
 * fluid's pressure moves.  While a fluid has bodies it owns a composite solid volume: every step first copies the borrowed volume into it
 * (or zeroes it), then writes every body over it in index order (a later body wins where they overlap): a cell whose centre lies inside a
 * body gets w = 1 and xyz = v + w x (cell centre - c), the rigid velocity.  Every later stage reads that volume; the borrowed one is never
 * written.  After the velocity solve each body's pressure force and torque about its centre are summed exactly with the face rule of the
 * load probes (wetted faces of the SOLID cells it covers; a solid overlapping a body is not told apart from it), and one thread per body
 * integrates semi-implicit Euler in float32: v += dt (g + F / m), w += dt R (I_b^-1 (R^T tau)) (no gyroscopic term), c += dt v,
 * q = normalize(q + dt/2 (0, w) q), with m = relative_density * V (V the analytic volume) per unit fluid density.  The tank walls clamp the
 * pose: a bounding box leaving [1, dim - 1] is shifted back and the outward velocity component zeroed (a clamp, not a collision model);
 * bodies do not collide with each other.  The new pose is what the next step writes.  The coupling is explicit: it was measured stable for
 * relative densities 0.5 and 0.75 (a floating box) and 2 (a sinking one); lighter bodies were not measured.  Bodies are state: a fluid with
 * bodies saves format version 8, with a mesh body version 16. */
#define BLUB_BODIES_MAX 16
#define BLUB_BODY_HISTORY_LENGTH 1024 /* records per body in the device ring: slot = step % 1024 */
typedef struct {
    int32_t shape;            /* 0 = box, 1 = sphere */
    float half_extent[3];     /* cells; a sphere's radius is half_extent[0] (the others are ignored) */
    float relative_density;   /* body density / fluid density, finite and > 0 */
    float centre[3];          /* grid cells */
    float rotation[4];        /* unit quaternion (w, x, y, z), body -> grid */
    float velocity[3];        /* cells/s */
    float angular_velocity[3];/* rad/s, grid axes */
} BlubBody;
typedef struct {
    uint32_t step;            /* blub_fluid_step_count before the step that wrote the record */
    uint32_t wetted_faces;
    int64_t force_fx[3];      /* force * 2^16, per unit fluid density (BlubSolidLoad's fixed point) */
    int64_t torque_fx[3];     /* torque about the centre * 2^8 */
    float centre[3], rotation[4], velocity[3], angular_velocity[3]; /* the pose after the step's integration */
    uint32_t reserved;
} BlubBodyRecord;
#ifdef __cplusplus
static_assert(sizeof(BlubBody) == 72 && sizeof(BlubBodyRecord) == 112, "BlubBody / BlubBodyRecord layout");
#else
_Static_assert(sizeof(BlubBody) == 72 && sizeof(BlubBodyRecord) == 112, "BlubBody / BlubBodyRecord layout");
#endif
/* Replaces the whole body set (0 clears it), resets the history and drops the cached step graphs; the quaternions are stored normalised.
 * BLUB_ERR_INVALID_ARGUMENT, changing nothing: more than 16 bodies, a non-finite value, a shape other than 0 / 1, a half extent or radius
 * below 1 cell, relative_density <= 0, a quaternion whose norm is not within 1e-3 of 1, a bounding box outside [1, dim - 1], a z-slab rank,
 * or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_bodies(BlubFluid *fluid, const BlubBody *bodies, uint32_t num_bodies);
/* The newest min(capacity, recorded, 1024) records of body `body`, oldest first; *count receives their number.  Synchronises.
 * BLUB_ERR_INVALID_ARGUMENT: a body index outside the set. */
int blub_fluid_body_history(BlubFluid *fluid, uint32_t body, BlubBodyRecord *out, uint32_t capacity, uint32_t *count);
/* The current bodies (the pose the next step writes); writes at most `capacity` and sets *count to the number in the set.  Synchronises. */
int blub_fluid_bodies(BlubFluid *fluid, BlubBody *out, uint32_t capacity, uint32_t *count);
/* The scene's optional fluid.bodies in grid cells and cells/s ((p - world_position) / grid_to_world_scale, Euler angles as for
 * static_objects).  Writes at most `capacity` bodies and sets *count to the number the scene holds.  blub_scene_load sets them. */
int blub_scene_bodies(const char *scene_json_path, BlubBody *out, uint32_t capacity, uint32_t *count);

/* ---- triangle-mesh bodies (shape 2; rules: DESIGN.md section 8 "Mesh bodies") ------------------------------------------------
 * A mesh body is a closed, consistently oriented triangle mesh (either winding) scaled by `scale` cells per model unit.  The library moves
 * it to its body frame: origin at the centre of mass, axes along the principal axes of inertia.  The stored BlubBody has centre = the centre
 * of mass in the grid, rotation = model rotation * principal rotation and half_extent = (hi - lo) / 2 of the body-frame bounds; mass and
 * principal moments come from the mesh (float64 on the host, rounded to float32 once).  A mesh body covers the cells whose centre lies
 * inside the mesh at the body's current pose, filled on the GPU every step by crossing parity along +x.  Self-intersecting meshes are not
 * detected.  A fluid with a mesh body saves state format version 16 (version 8 plus section 16, the mesh bodies as stored).  The scene key
 * fluid.bodies takes {shape: "mesh", model: OBJ path relative to the scene file, scale: world units per model unit, position,
 * rotation_angles_deg?, relative_density, velocity?, angular_velocity?}; position and rotation place the model origin and axes. */
#define BLUB_MESH_BODY_MAX_VERTICES 262144   /* over all mesh bodies of a set */
#define BLUB_MESH_BODY_MAX_TRIANGLES 524288  /* over all mesh bodies of a set */
typedef struct {
    double volume;                 /* cells^3, > 0 for either winding */
    double centroid[3];            /* the centre of mass in model units (model frame) */
    double inertia[9];             /* about the centre of mass per unit body density, cells^5, model axes, row major */
    double principal_moments[3];   /* per unit body density: the diagonal of the inertia in the principal frame */
    double principal_rotation[4];  /* unit quaternion (w, x, y, z): principal frame -> model frame, R_p */
    float bounds_lo[3], bounds_hi[3]; /* body-frame bounding box of the float32 body-frame vertices, cells */
    float mass;                    /* float32(relative_density * volume) per unit fluid density (relative_density = 1 for blub_mesh_body_properties) */
    float moments[3];              /* float32(relative_density * principal_moments) */
    float scale;                   /* cells per model unit */
    uint32_t num_vertices, num_triangles;
} BlubMeshBodyProperties;
typedef struct {
    const struct BlubMesh *mesh;   /* NULL: the body is a box or sphere (BlubBody.shape 0 / 1) */
    float scale;                   /* cells per model unit, finite and > 0 */
} BlubMeshBodyShape;
/* Host only, no device needed: checks a mesh and computes its mass properties and principal frame.  BLUB_ERR_INVALID_ARGUMENT: no
 * triangles, num_indices not a multiple of 3, an index out of range, a triangle repeating a vertex, a directed edge occurring other than
 * exactly once or without its reverse (not closed and consistently oriented), a non-finite position, zero volume, a scale that is not finite
 * and > 0, a body-frame bounding box thinner than 1 cell on some axis, or more than BLUB_MESH_BODY_MAX_VERTICES / _TRIANGLES. */
int blub_mesh_body_properties(const float *positions_xyz, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale,
                              BlubMeshBodyProperties *out);
/* Host only: the float32 body-frame vertices (xyz, num_vertices of them) a mesh body of this mesh and scale stores: R_p^T (scale p - com).
 * Refuses what blub_mesh_body_properties refuses. */
int blub_mesh_body_vertices(const float *positions_xyz, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale,
                            float *out_xyz);
/* blub_fluid_set_bodies with triangle-mesh bodies: shapes[i].mesh != NULL makes body i a mesh body (bodies[i].shape and half_extent are
 * ignored; centre and rotation place the mesh's model origin and axes in the grid).  The geometry is copied, so the meshes may be destroyed
 * afterwards.  Refuses everything blub_fluid_set_bodies refuses (but shape 2 with a mesh), what blub_mesh_body_properties refuses, a mesh on
 * another device and more than the vertex / triangle limits over the set, changing nothing.  shapes == NULL: blub_fluid_set_bodies. */
int blub_fluid_set_bodies_meshes(BlubFluid *fluid, const BlubBody *bodies, const BlubMeshBodyShape *shapes, uint32_t num_bodies);
/* The mass properties of mesh body `body` as stored (mass and moments with its relative density).  A renderer recovers the model pose
 * from the body's pose: R_model = R_body R_p^T, origin = c - R_model (scale * centroid).  BLUB_ERR_INVALID_ARGUMENT: not a mesh body. */
int blub_fluid_body_mass_properties(BlubFluid *fluid, uint32_t body, BlubMeshBodyProperties *out);
/* The resolved OBJ path (NUL-terminated, truncated to capacity - 1) and the scale in cells per model unit of the scene's mesh body `body`.
 * BLUB_ERR_INVALID_ARGUMENT: not a mesh body of the scene; the scene's own errors as blub_scene_info. */
int blub_scene_body_model(const char *scene_json_path, uint32_t body, char *model_path_out, size_t capacity, float *scale_out);

/* ---- viscous liquids (not part of the reference surface; rules: DESIGN.md section 8) ------------------------------------------------
 * With a kinematic viscosity above zero every step ends its stage 0 with an implicit diffusion of the grid velocity,
 * (I - nu dt Laplace) u_c = u_c* per component, solved by Jacobi-preconditioned CG in one persistent kernel: solids (the tank walls, the
 * solid volume, floating bodies) are no-slip with their own velocity, the free surface carries du_c/dn = 0, gravity's increment is left out
 * of the diffusion (a tank at rest stays bit for bit what it is without viscosity).  kinematic_viscosity is in cells^2/s (m^2/s divided by
 * grid_to_world_scale^2); error_tolerance is the absolute bound on max |residual| in cells/s at which the solve stops, max_num_iterations
 * its cap.  Viscosity is part of the saved state (format version 32). */
typedef struct {
    float kinematic_viscosity;
    float error_tolerance;
    int32_t max_num_iterations;
    uint32_t reserved; /* 0 */
} BlubViscosity;
/* NULL or kinematic_viscosity == 0 turns the stage off while there is no tag viscosity table (blub_fluid_set_tag_viscosities): the step is
 * then the step of a fluid that never had viscosity.  With a table, 0 makes the tags not in it inviscid.  error_tolerance and
 * max_num_iterations are kept also with kinematic_viscosity == 0, for a table that turns the stage on.  Stream-ordered;
 * turning it on or off drops the cached step graphs, a change between two positive settings does not.  BLUB_ERR_INVALID_ARGUMENT, changing
 * nothing: a negative or non-finite viscosity, a tolerance that is not finite or not above 0, max_num_iterations outside [1, 10000],
 * reserved != 0, a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_viscosity(BlubFluid *fluid, const BlubViscosity *viscosity);
/* the current setting (kinematic_viscosity 0: off) */
int blub_fluid_viscosity(const BlubFluid *fluid, BlubViscosity *out);
/* the last viscosity solve, synchronously: its iterations and max |residual| per component (cells/s); zeros before the first solve */
int blub_fluid_last_viscosity_solve(BlubFluid *fluid, int32_t *iterations, float max_error[3]);
/* The scene's optional fluid.viscosity (m^2/s) in cells^2/s: value / grid_to_world_scale^2, 0 without the key.  blub_scene_load sets it on
 * the fluid it creates.  A value that is not a number, negative or not finite makes every scene call fail with BLUB_ERR_PARSE. */
int blub_scene_viscosity(const char *scene_json_path, float *cells2_per_s);

/* ---- CFL-limited substeps (not part of the reference surface, whose clock is a fixed 120 Hz; rules: DESIGN.md section 8) -----------
 * The library can choose the length of the next step from the particles' largest velocity.  An adaptive run is an ordinary sequence of
 * blub_fluid_step calls: plan a substep of the time still to cover, step it as blub_fluid_step(fluid, blub_duration_as_secs_f32(dt_ns))
 * (the conversion blub_run uses for its fixed step), repeat until the interval is covered.  The step itself, its graphs and the state file are
 * unchanged, and a fluid that never plans launches and allocates nothing for it.
 * The rule (float64, integer nanoseconds): u = max_c |max_velocity[c]|; s = u + sqrt(5 |g|) with |g| the Euclidean norm of the gravity in
 * cells/s^2 (Bridson's margin for the speed one step of gravity adds, dx = 1 cell); d = cfl_number / s seconds (+infinity when s = 0);
 * d_ns = min(max_dt_ns, floor(d * 1e9)), saturating.  d_ns < min_dt_ns is refused with BLUB_ERR_UNSTABLE.  Otherwise, with R the time
 * still to cover: dt = R when R <= d_ns, R - R / 2 (integer division) when R < 2 d_ns (the interval does not end in a sliver), else d_ns.
 * Each particle then moves at most cfl_number cells along each axis at its current velocity (a per-axis bound, not a Euclidean one), and the
 * substeps of an interval add up to it exactly. */
#define BLUB_ERR_UNSTABLE 6 /* a non-finite particle velocity, or a CFL step below min_dt_ns: nothing was stepped */
typedef struct {
    float cfl_number;   /* C: finite, in (0, 16] */
    uint32_t reserved;  /* 0 */
    uint64_t max_dt_ns; /* the longest substep */
    uint64_t min_dt_ns; /* 1 <= min_dt_ns <= max_dt_ns: a CFL step below it is refused */
} BlubTimeStepping;
/* out[c] = max |v_c| over the live particles (v_c = the .w word of velocity row c; the device-resident count while a flow set is active),
 * exact: +0 without particles, infinity and NaN as themselves.  Runs one kernel, then synchronises.  BLUB_ERR_INVALID_ARGUMENT: a z-slab rank
 * or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_max_particle_velocity(BlubFluid *fluid, float out[3]);
/* Host only, no device needed: the rule above applied to a measured max_velocity (cells/s per axis) and gravity (cells/s^2).
 * BLUB_ERR_INVALID_ARGUMENT: a bad config (cfl_number not finite or outside (0, 16], reserved != 0, not 1 <= min_dt_ns <= max_dt_ns),
 * remaining_ns == 0 or a non-finite gravity.  BLUB_ERR_UNSTABLE: a non-finite velocity or d_ns < min_dt_ns; blub_last_error names the case
 * and the velocity. */
int blub_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTimeStepping *config, uint64_t *dt_ns);
/* blub_fluid_max_particle_velocity, then blub_cfl_substep_ns with the fluid's gravity and, while the fluid has surface tension s > 0, with
 * max_dt_ns lowered to the capillary limit floor(1e9 sqrt(1 / (4 pi s))) (a limit below min_dt_ns: BLUB_ERR_UNSTABLE).  max_velocity_out (may be
 * NULL) receives the measurement, also when the rule refuses it.  Refuses what both refuse, checking the config and remaining_ns before anything is launched. */
int blub_fluid_plan_substep(BlubFluid *fluid, uint64_t remaining_ns, const BlubTimeStepping *config, uint64_t *dt_ns, float max_velocity_out[3]);

/* ---- surface tension (not part of the reference surface; rules: DESIGN.md section 8 "Surface tension") --------------------------------
 * With a kinematic surface tension s = sigma / density above zero (cells^3/s^2: m^3/s^2 divided by grid_to_world_scale^3; water is
 * 7.28e-5 m^3/s^2) the free surface carries the pressure jump P_liquid - P_air = sigma kappa.  Stage 1 of every step measures the curvature
 * kappa of a smoothed particle density (integer arithmetic, bit-reproducible) in the band of cells on both sides of the surface and moves the
 * velocity solve's Dirichlet value on AIR from 0 to the ghost value g = -dt s (kappa_i + kappa_j) / 2 of each FLUID-AIR face; stage 4 adds g
 * to those faces.  Walls are neutrally wetting (contact angle 90 degrees).  While s > 0 blub_fluid_plan_substep also holds every substep
 * to the capillary limit floor(1e9 sqrt(1 / (4 pi s))) ns.  Surface tension is part of the saved state (format version 64). */
/* 0 turns it off: the step is then the step of a fluid that never had surface tension.  Stream-ordered; turning it on or off drops the cached
 * step graphs, a change between two positive values does not.  BLUB_ERR_INVALID_ARGUMENT, changing nothing: a negative or non-finite value,
 * a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_surface_tension(BlubFluid *fluid, float cells3_per_s2);
/* the current setting (0: off) */
int blub_fluid_surface_tension(const BlubFluid *fluid, float *cells3_per_s2);
/* The scene's optional fluid.surface_tension (m^3/s^2) in cells^3/s^2: value / grid_to_world_scale^3, 0 without the key.  blub_scene_load
 * sets it on the fluid it creates.  A value that is not a number, negative or not finite makes every scene call fail with BLUB_ERR_PARSE. */
int blub_scene_surface_tension(const char *scene_json_path, float *cells3_per_s2);

/* ---- interfacial tension (not part of the reference surface; rules: DESIGN.md section 8 "Interfacial tension") ---------------------
 * A kinematic interfacial tension s_AB = sigma_AB / rho_ref (cells^3/s^2: m^3/s^2 divided by grid_to_world_scale^3; oil on water is about
 * 3e-5 m^3/s^2) between two phases of the liquid: phase B, the particles whose tag is in a set of at most 16 tags, and phase A, every other
 * particle.  The interface carries P_B - P_A = sigma_AB kappa, kappa = div n with n pointing from B into A (+2/R for a drop of B).  Stage 1
 * of every step splats all particles and the phase-B particles, smooths 2 splat_B - splat_all in integer arithmetic (bit-reproducible) into a
 * phase field phi (> 0: phase B), measures the curvature on the FLUID cells next to a FLUID cell of the other phase and moves the velocity
 * solve's right-hand side by the ghost values g = -dt s_AB (kappa_i + kappa_j) / 2 of those faces, times the face coefficient of a tag
 * density table; stage 4 adds them to the faces.  The matrix is unchanged.  It is independent of the free surface's tension and works with
 * and without a tag density table.  Walls are neutrally wetting.  While s_AB > 0 blub_fluid_plan_substep holds every substep to the
 * capillary limit of max(surface tension, s_AB).  The tension and the tags are part of the saved state (format version 512). */
#define BLUB_INTERFACE_TAGS_MAX 16
/* Sets s_AB and phase B's tags; s_AB = 0 turns it off (the set is then ignored and may be empty), and the step is then the step of a fluid
 * that never had an interfacial tension.  Stream-ordered; turning it on or off drops the cached step graphs, a change between two settings
 * above zero does not.  BLUB_ERR_INVALID_ARGUMENT, changing nothing: a negative or non-finite value, more than 16 tags, a tag listed twice, a
 * NULL set with count > 0, a value above 0 with an empty set, a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_interfacial_tension(BlubFluid *fluid, const uint32_t *tags, uint32_t count, float cells3_per_s2);
/* the current setting: s_AB into *cells3_per_s2 (0: off), min(count, capacity) tags into tags (may be NULL with capacity 0), their number
 * into *count */
int blub_fluid_interfacial_tension(const BlubFluid *fluid, uint32_t *tags, uint32_t capacity, uint32_t *count, float *cells3_per_s2);
/* The scene's optional fluid.interfacial_tension, {"tags": [n, ...], "tension": m^3/s^2}, the tension divided by grid_to_world_scale^3 (0
 * and no tags without the key).  blub_scene_load sets it on the fluid it creates.  A value the setter would refuse makes every scene call
 * fail with BLUB_ERR_PARSE. */
int blub_scene_interfacial_tension(const char *scene_json_path, uint32_t *tags, uint32_t capacity, uint32_t *count, float *cells3_per_s2);

/* ---- whitewater (not part of the reference surface; rules: DESIGN.md section 8 "Whitewater") --------------------------------------
 * Spray, foam and bubble particles (Ihmsen et al. 2012), stepped at the end of stage 5 of every step from the projected grid velocity and
 * this step's marker.  They never act on the liquid: every liquid tap, dump and saved liquid section is what it is without them.  A live
 * particle is classified by the FLUID cells among the 27 around its cell (fewer than spray_below: spray; its own cell FLUID and at least
 * bubble_from: bubble; else foam), then spray falls ballistically, a bubble rises by buoyancy * -g and is pulled towards u by `drag` per
 * step, foam moves with u and ages; particles leaving [1, dim - 1), entering a SOLID cell or the solid volume, or out of lifetime are removed.
 * FLUID cells with an AIR neighbour emit dt (trapped_air_rate I_ta + wave_crest_rate I_wc) I_k particles, at most max_per_cell, with the
 * potentials I ramps of the curl's magnitude (1/s), of the AIR neighbour count on a crest moving outwards and of 0.5 |u|^2 (cells^2/s^2).
 * All in grid units.  Bit-reproducible.  Part of the saved state (format version 1024). */
#define BLUB_WHITEWATER_MAX_PARTICLES (1u << 26)
typedef struct BlubWhitewater {
    uint32_t max_num_particles;   /* capacity, at most BLUB_WHITEWATER_MAX_PARTICLES; 0: off */
    float trapped_air_rate;       /* particles per cell and second at full potential, >= 0 */
    float wave_crest_rate;        /* >= 0 */
    float trapped_air_range[2];   /* |curl u| in 1/s: the ramp's lo < hi */
    float wave_crest_range[2];    /* AIR neighbours of a crest cell (0 to 26): lo < hi */
    float energy_range[2];        /* 0.5 |u|^2 in cells^2/s^2: lo < hi */
    float lifetime_lo, lifetime_hi; /* seconds, a new particle's lifetime is uniform in [lo, hi): 0 <= lo < hi */
    float buoyancy;               /* a bubble accelerates by -buoyancy g */
    float drag;                   /* in [0, 1]: the share of u - v a bubble takes on per step */
    uint32_t spray_below;         /* spray_below <= bubble_from <= 27 */
    uint32_t bubble_from;
    uint32_t max_per_cell;        /* at most 16 particles a cell emits per step */
} BlubWhitewater;
/* NULL or max_num_particles 0 turns whitewater off, frees its memory and leaves an all-zero setting; a fluid that never turned it on
 * allocates and launches nothing for it.  A new capacity starts from no particles and zero counters; another change keeps them.  The new
 * storage is allocated before the old one is freed: a failed allocation returns its error and leaves the fluid as it was.  Every change drops the cached step graphs.
 * BLUB_ERR_INVALID_ARGUMENT, changing nothing: a non-finite value, a range or lifetime with lo >= hi, a negative rate or lifetime, drag outside
 * [0, 1], spray_below > bubble_from, bubble_from > 27, max_per_cell > 16, a capacity above BLUB_WHITEWATER_MAX_PARTICLES, a z-slab rank, or a
 * fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_whitewater(BlubFluid *fluid, const BlubWhitewater *settings);
/* the current setting (all zero: off) */
int blub_fluid_whitewater(const BlubFluid *fluid, BlubWhitewater *out);
/* {live, emitted, removed, refused for capacity}; the last three are cumulative since the setting that allocated the capacity.  Zeros while
 * off.  Synchronises. */
int blub_fluid_whitewater_counters(BlubFluid *fluid, uint64_t out[4]);
/* The live particles in their order: min(count, capacity) float4 positions (xyz in cells, w = remaining lifetime in s) into pos4 and
 * velocities (xyz in cells/s, w = the raw bits of the kind: 0 spray, 1 foam, 2 bubble) into vel4; the live count into *count.  pos4 / vel4
 * may be NULL with capacity 0.  Synchronises. */
#define BLUB_WHITEWATER_SPRAY 0
#define BLUB_WHITEWATER_FOAM 1
#define BLUB_WHITEWATER_BUBBLE 2
int blub_fluid_download_whitewater(BlubFluid *fluid, float *pos4, float *vel4, uint32_t capacity, uint32_t *count);
/* The scene's optional fluid.whitewater in grid units (*has = 0 and a zeroed setting without the key): the same fields in world units, the
 * energy range in m^2/s^2 divided by grid_to_world_scale^2, the curl's range in 1/s, rates in 1/s, lifetimes in s as they are.
 * blub_scene_load sets it on the fluid it creates.  A value the setter would refuse makes every scene call fail with BLUB_ERR_PARSE. */
int blub_scene_whitewater(const char *scene_json_path, BlubWhitewater *out, int32_t *has);

/* ---- liquids of different densities (not part of the reference surface; rules: DESIGN.md section 8 "Liquids of different densities") ----
 * A table gives the particles of a tag a density relative to the reference density rho_ref that the velocity solve's pressure p dt / rho_ref,
 * the bodies' relative densities, the load probes' forces, the viscosity and the surface tension are all defined against.  Tags not in the
 * table have density 1.  Stage 0 of every step averages the particles' densities per cell (exact integer sums, independent of the particle
 * order), and the velocity solve of stage 2 and the velocity update of stage 4 become variable-density: a face between the FLUID cells i and
 * j carries 2 / (rho_i + rho_j), a FLUID-AIR face 1 / rho_i.  The transfer, the divergence, the density correction of stage 10 and the
 * advection are unchanged.  The table is part of the saved state (format version 128). */
typedef struct {
    uint32_t tag;
    float relative_density; /* finite, in [1/2, 2] */
} BlubTagDensity;
#define BLUB_TAG_DENSITIES_MAX 16
/* Replaces the table; count 0 turns the feature off, and the fluid is then bit for bit a fluid that never had a table.  Stream-ordered;
 * turning it on or off drops the cached step graphs, a change between two non-empty tables does not.  BLUB_ERR_INVALID_ARGUMENT, changing
 * nothing: more than 16 entries, a tag listed twice, a density that is not finite or lies outside [1/2, 2], floating bodies (and blub_fluid_set_bodies refuses bodies while a table is
 * set), a table while the surface tension
 * is above 0, precond_mode 1 (blub_fluid_set_quirks refuses precond_mode 1 and blub_fluid_set_surface_tension a value above 0 while a table
 * is set), a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_tag_densities(BlubFluid *fluid, const BlubTagDensity *table, uint32_t count);
/* the current table in the order it was set: min(count, capacity) entries into out, their number into *count (0: off) */
int blub_fluid_tag_densities(const BlubFluid *fluid, BlubTagDensity *out, uint32_t capacity, uint32_t *count);
/* The scene's optional fluid.tag_densities, [{"tag": n, "relative_density": x}]: min(count, capacity) entries into out, their number into
 * *count (0 without the key).  blub_scene_load sets it on the fluid it creates.  A value the setter would refuse (and a table together with a
 * surface tension above 0) makes every scene call fail with BLUB_ERR_PARSE. */
int blub_scene_tag_densities(const char *scene_json_path, BlubTagDensity *out, uint32_t capacity, uint32_t *count);

/* ---- liquids of different viscosities (not part of the reference surface; rules: DESIGN.md section 8 "Liquids of different viscosities")
 * A table gives the particles of a tag their own kinematic viscosity nu_tag >= 0 in cells^2/s; tags not in it take the fluid's
 * kinematic_viscosity (blub_fluid_set_viscosity, which may be 0).  The viscosity stage runs while the fluid's value or any of the table's is
 * above 0, with the fluid's error_tolerance and max_num_iterations.  Stage 0 averages the particles' nu per FLUID cell (exact integer sums
 * of rint(nu_tag / nu_scale 2^32), nu_scale the largest value, independent of the particle order; a FLUID cell without a particle takes the
 * fluid's value), and the viscosity solve couples two velocity faces with nu_fn dt, nu_fn the mean of nu over the FLUID cells at the
 * midpoint of the two faces.  A face whose coefficients are all 0 is not solved and keeps its value.  The viscosity stays kinematic, also
 * together with a tag density table (then not momentum-conserving across a density interface).  The table is part of the saved state
 * (format version 256). */
typedef struct {
    uint32_t tag;
    float kinematic_viscosity; /* finite, >= 0, cells^2/s */
} BlubTagViscosity;
#define BLUB_TAG_VISCOSITIES_MAX 16
/* Replaces the table; count 0 clears it, and the fluid is then bit for bit a fluid that never had a table.  Stream-ordered; turning it on or
 * off drops the cached step graphs, a change between two non-empty tables does not (unless it turns the stage on or off).
 * BLUB_ERR_INVALID_ARGUMENT, changing nothing: more than 16 entries, a NULL table with count > 0, a tag listed twice, a viscosity that is
 * negative or not finite, a z-slab rank, or a fluid left inside a step by blub_fluid_step_stages. */
int blub_fluid_set_tag_viscosities(BlubFluid *fluid, const BlubTagViscosity *table, uint32_t count);
/* the current table in the order it was set: min(count, capacity) entries into out, their number into *count (0: none) */
int blub_fluid_tag_viscosities(const BlubFluid *fluid, BlubTagViscosity *out, uint32_t capacity, uint32_t *count);
/* The scene's optional fluid.tag_viscosities, [{"tag": n, "viscosity": m^2/s}], each value divided by grid_to_world_scale^2:
 * min(count, capacity) entries into out, their number into *count (0 without the key).  blub_scene_load sets it on the fluid it creates.  A
 * value the setter would refuse makes every scene call fail with BLUB_ERR_PARSE. */
int blub_scene_tag_viscosities(const char *scene_json_path, BlubTagViscosity *out, uint32_t capacity, uint32_t *count);

/* ---- moving tanks (not part of the reference surface; rules: DESIGN.md section 8 "Moving tanks") ----------------------------------
 * The liquid is simulated in the tank's own frame: the grid, the walls, the solid volume, probes, sources and drains are fixed in it, and the
 * fluid feels f = R^T (g - A) - alpha x r - omega x (omega x r) - 2 omega x v with r = x - pivot (all lengths in grid cells).  The library keeps
 * no clock: the caller sets the frame of the next steps with blub_fluid_set_tank_frame, as it rewrites the solid volume before each step.
 * The frame is not state: a saved file is the same with or without one, and a loaded fluid starts at rest. */
typedef struct {
    double rotation[9];             /* R: tank -> world, row major; orthonormal with det +1 (to 1e-6) */
    double acceleration[3];         /* A: the pivot's acceleration, world axes, cells/s^2 */
    double angular_velocity[3];     /* omega: tank axes, rad/s */
    double angular_acceleration[3]; /* alpha: tank axes, rad/s^2 */
    double pivot[3];                /* grid cells */
} BlubTankFrame;
/* One harmonic translation of the pivot: amplitude * direction * sin(2 pi frequency t + phase). */
typedef struct {
    double direction[3];            /* unit vector (to 1e-6), world axes */
    double amplitude;               /* cells */
    double frequency;               /* Hz, >= 0 */
    double phase;                   /* rad */
} BlubTankTranslation;
#define BLUB_TANK_TRANSLATIONS_MAX 4
/* A prescribed motion the library evaluates but never stores: up to 4 harmonic translations and one rotation about the fixed unit axis n
 * through the pivot by theta(t) = amplitude sin(2 pi frequency t + phase) + rate t. */
typedef struct {
    double pivot[3];                /* grid cells */
    uint32_t num_translations;      /* <= BLUB_TANK_TRANSLATIONS_MAX */
    uint32_t reserved;              /* 0 */
    BlubTankTranslation translations[BLUB_TANK_TRANSLATIONS_MAX];
    double axis[3];                 /* n: unit vector (to 1e-6) */
    double amplitude;               /* rad */
    double frequency;               /* Hz, >= 0 */
    double phase;                   /* rad */
    double rate;                    /* rad/s */
} BlubTankMotion;
/* The float32 constants one step uses, computed in float64 and rounded once (blub_tank_step_constants). */
typedef struct {
    float gravity[3];               /* g_eff = R^T (g - A) */
    float coriolis[9];              /* Q = Rot(omega / |omega|, -2 |omega| dt), row major: the exact solution of dv/dt = -2 omega x v over dt */
    float force[9];                 /* K = dt (|omega|^2 I - omega omega^T - [alpha]x), row major: the velocity increment per cell of r */
    float pivot[3];
    int32_t rotating;               /* 1 when omega or alpha is not zero: the step then runs tank_frame_kernel */
} BlubTankStepConstants;
#ifdef __cplusplus
static_assert(sizeof(BlubTankFrame) == 168 && sizeof(BlubTankMotion) == 280 && sizeof(BlubTankStepConstants) == 100, "tank layouts");
#else
_Static_assert(sizeof(BlubTankFrame) == 168 && sizeof(BlubTankMotion) == 280 && sizeof(BlubTankStepConstants) == 100, "tank layouts");
#endif
/* Host only: the frame of `motion` at t_seconds, in closed form in float64: R = Rot(n, theta), omega = theta' n, alpha = theta'' n, A = the second
 * derivative of the translations, pivot = motion->pivot.  BLUB_ERR_INVALID_ARGUMENT: a NULL pointer, a non-finite value or t, a direction or
 * axis that is not a unit vector, a negative frequency, more than 4 translations or reserved != 0. */
int blub_tank_frame_at(const BlubTankMotion *motion, double t_seconds, BlubTankFrame *out);
/* Host only: the step constants of `frame` for a fluid of float32 gravity gravity_grid and a step of dt seconds (the step's float32 delta).
 * BLUB_ERR_INVALID_ARGUMENT: a NULL pointer, a frame blub_fluid_set_tank_frame refuses, a non-finite gravity or dt <= 0. */
int blub_tank_step_constants(const BlubTankFrame *frame, const float gravity_grid[3], float dt, BlubTankStepConstants *out);
/* The frame of the following steps (NULL: at rest).  Every step then uses the constants above with the fluid's gravity: StepParams' gravity
 * becomes g_eff (a frame with omega = alpha = 0 launches nothing new and steps exactly as blub_fluid_set_gravity_grid(g_eff) would), and a
 * rotating frame runs tank_frame_kernel on every live particle in stage 0, between the sources and drains and the P2G.  Turning rotation on
 * or off drops the cached step graphs; a new frame of the same kind does not.  BLUB_ERR_INVALID_ARGUMENT, changing nothing: a frame that is not
 * finite or whose rotation is not orthonormal with det +1 to 1e-6, a rotating frame while the fluid has floating bodies, a z-slab rank, or a
 * fluid left inside a step by blub_fluid_step_stages.  While a frame is set blub_fluid_plan_substep plans with blub_tank_cfl_substep_ns. */
int blub_fluid_set_tank_frame(BlubFluid *fluid, const BlubTankFrame *frame);
/* 1 and *out = the frame when one is set, 0 when the fluid is at rest (or fluid is NULL) */
int blub_fluid_tank_frame(const BlubFluid *fluid, BlubTankFrame *out);
/* Host only: blub_cfl_substep_ns under a frame (NULL: exactly blub_cfl_substep_ns).  The gravity passed to the rule has the norm
 * |g_eff| + (|omega|^2 + |alpha|) r_max, r_max = the distance from the pivot to the farthest corner of the grid_dimension box; while omega is not
 * zero the velocity passed is the Euclidean norm of max_velocity (the Coriolis rotation moves speed between axes).  Both rounded to float32. */
int blub_tank_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTankFrame *frame,
                             const uint32_t grid_dimension[3], const BlubTimeStepping *config, uint64_t *dt_ns);
/* The scene's optional fluid.tank_motion in grid cells: {pivot, translations: [{direction, amplitude, frequency, phase?}],
 * rotation?: {axis, amplitude?, frequency?, phase?, rate?}} in world units (pivot and amplitudes / grid_to_world_scale, as the load probes'
 * pivots), Hz, rad and rad/s; directions and the axis are normalised.  *has_motion = 0 without the key.  A bad value makes every scene call fail
 * with BLUB_ERR_PARSE. */
int blub_scene_tank_motion(const char *scene_json_path, BlubTankMotion *out, int32_t *has_motion);

/* ---- scene JSON surface (src/scene/mod.rs:19-43,109-144; src/scene/models.rs:11-46) ------------------------- */
/* Scene::new + create_fluid_from_config: parses an unchanged blub scene file, creates the fluid, seeds every
 * fluid cube (world / grid_to_world_scale) and sets gravity.  static_objects are parsed (blub_scene_static_object) but their
 * meshes (git-LFS stubs in the reference checkout) are not voxelized. */
int blub_scene_load(BlubFluid **out, const char *scene_json_path, int device, void *cuda_stream);
/* Scene description without creating a fluid: fills dims, max_num_particles, scale, gravity(world), #cubes, #static objects. */
typedef struct {
    uint32_t grid_dimension[3];
    uint32_t max_num_particles;
    float grid_to_world_scale;
    float world_position[3];
    float gravity[3];
    uint32_t num_fluid_cubes;
    uint32_t num_static_objects;
} BlubSceneInfo;
int blub_scene_info(const char *scene_json_path, BlubSceneInfo *out);
/* The scene's optional fluid.load_probes in grid cells (world / grid_to_world_scale; a missing pivot is the box centre).  Writes at most
 * `capacity` probes and sets *count to the number the scene holds.  blub_scene_load sets them on the fluid it creates. */
int blub_scene_load_probes(const char *scene_json_path, BlubLoadProbe *out, uint32_t capacity, uint32_t *count);

/* ---- analytic rigid solids (stand-in for the mesh voxelizer, src/scene/voxelization.rs:118-157) ---------------------------
 * One oriented box or sphere with the reference's rigid animation (StaticObjectConfig / RigidAnimation, src/scene/models.rs:11-46,
 * 154-224) written into an RGBA16F voxel volume: xyz = solid velocity in cells/s, w = 1 inside. */
typedef struct {
    float world_position[3];
    float scale;
    float rotation_angles_deg[3];   /* static Euler angles (cgmath Euler<Deg>) */
    int32_t shape;                  /* 0 = box with half_extent (model space), 1 = sphere of radius half_extent[0], 2 = triangle mesh */
    float half_extent[3];
    int32_t has_translation;        /* TranslationAnimation: ping-pong between world_position and target */
    float translation_target[3];
    int32_t translation_curve;      /* 0 = Linear, 1 = SmoothStep */
    float translation_duration;
    int32_t has_rotation;           /* RotationAnimation */
    float rotation_axis[3];
    float rotation_deg_per_sec;
} BlubRigidObject;
typedef struct {                    /* what the animation evaluated to (for tests / logging) */
    float centre_voxel[3], velocity_voxel[3], axis_scaled[3], rotation[9];
} BlubRigidState;
/* Evaluates the animation at `total_simulated_time` (velocity = finite difference over `simulation_delta`, models.rs:186-191)
 * and enqueues the voxelization on `cuda_stream`.  clear_first != 0 zeroes the rest of the volume (first object of a step). */
int blub_solid_voxelize(void *rgba16f_device_ptr, const uint32_t grid_dimension[3], const BlubRigidObject *object, float grid_to_world_scale,
                        const float fluid_world_position[3], double total_simulated_time, double simulation_delta, int clear_first,
                        void *cuda_stream, BlubRigidState *state_out);

/* ---- simulation clock (src/timer.rs:18-36,94-126, src/simulation_controller.rs:33-35): integer nanoseconds, host only ------------- */
/* Duration::from_nanos(1e9 / steps_per_second): the simulation delta of the controller (120 Hz -> 8,333,333 ns) */
uint64_t blub_simulation_delta_ns(uint64_t steps_per_second);
/* Duration::as_secs_f32: what the shaders / the model animation receive as time */
float blub_duration_as_secs_f32(uint64_t nanoseconds);
/* One render frame of `frame_delta_ns` on the render clock (Timer::force_frame_delta as used by recording and fast forward), then
 * Timer::simulation_frame_loop until the simulation has caught up: returns how many simulation steps belong to this frame and
 * advances both clocks.  (The realtime mode's step dropping needs wall-clock frame times and is not part of a headless run.) */
uint32_t blub_timer_steps_in_frame(uint64_t *total_rendered_ns, uint64_t *total_simulated_ns, uint64_t frame_delta_ns, uint64_t simulation_delta_ns);

/* ---- small device helpers for hosts without CUDA bindings of their own (e.g. the Rust shim of INTEGRATION.md) ----------------- */
/* the stream the fluid's work is enqueued on (the one given to blub_fluid_create, or the fluid's own): enqueue the voxelization of a
 * step there and it is ordered before the step without any host synchronisation */
void *blub_fluid_stream(const BlubFluid *fluid);
int blub_device_malloc(void **out, size_t bytes, int device);  /* zero-initialised */
int blub_device_free(void *device_ptr);

/* ---- triangle meshes: the conservative hull voxelizer (src/scene/voxelization.rs:118-157, shader/voxelize/conservative_hull.*) ----
 * A BlubMesh is the geometry the voxelization pass reads: model-space positions + triangle indices (MeshVertices / MeshIndices,
 * conservative_hull.vert:16-20) resident on one device.  blub_mesh_load_obj reads a Wavefront OBJ the way the reference does
 * (tobj::load_obj with triangulate / ignore_points / ignore_lines, src/scene/models.rs:252-262; only `v` and `f` matter here). */
typedef struct BlubMesh BlubMesh;
int blub_mesh_create(BlubMesh **out, const float *positions_xyz, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices,
                     int device);
int blub_mesh_load_obj(BlubMesh **out, const char *obj_path, int device);
void blub_mesh_destroy(BlubMesh *mesh);
int blub_mesh_info(const BlubMesh *mesh, uint32_t *num_vertices, uint32_t *num_triangles);
/* Host-only OBJ reader behind blub_mesh_load_obj (no device needed).  Writes at most the given capacities and always reports the full
 * counts in counts_out = {vertices, indices}: call once with capacities 0 to size the arrays. */
int blub_obj_read(const char *obj_path, float *positions_xyz, uint32_t capacity_vertices, uint32_t *indices, uint32_t capacity_indices,
                  uint32_t counts_out[2]);
/* One draw of SceneVoxelization::update for `mesh` placed and animated by `placement` (its `shape` / `half_extent` are ignored): every
 * triangle is rasterised conservatively along its dominant axis and marks its hull voxels (+-1 in depth where the depth slope asks
 * for it) with w = 1 and xyz = ComputeVoxelSpeed.  clear_first != 0 = the clear_texture in front of the first mesh of a step; later
 * meshes overwrite earlier ones where they overlap, like consecutive draws.  Stream-ordered, deterministic. */
int blub_solid_voxelize_mesh(void *rgba16f_device_ptr, const uint32_t grid_dimension[3], BlubMesh *mesh, const BlubRigidObject *placement,
                             float grid_to_world_scale, const float fluid_world_position[3], double total_simulated_time,
                             double simulation_delta, int clear_first, void *cuda_stream, BlubRigidState *state_out);
/* static_objects[index] of a scene file: the model path as written (relative to the reference's `models/` directory) and its
 * placement + animation (shape = 2: mesh).  Returns BLUB_ERR_INVALID_ARGUMENT past the end. */
int blub_scene_static_object(const char *scene_json_path, uint32_t index, BlubRigidObject *placement_out, char *model_path_out,
                             size_t model_path_capacity);

/* ---- multi-GPU: z-slab sharding of the pressure solve (SURVEY.md section 8e; the reference is single-GPU) ---------------
 * Rank `rank` of `world` (<= 8) owns nz_owned planes of a global nx x ny x (world * nz_owned) grid; its local grid has 4
 * ghost planes on both sides (local plane 4 = first owned plane).  Each rank exposes ONE device allocation (the "window":
 * mailbox + residual + both pressure volumes).  After every rank's window has been mapped into every process
 * (blub_ipc_export / blub_ipc_open across processes, or plain pointers + blub_enable_peer_access inside one process),
 * blub_fluid_attach_slab_peers switches the solver to the sharded mode: the persistent PCG kernel then pushes its
 * boundary planes of r and p into the neighbours' ghost planes with P2P stores over NVLink and all-reduces its scalars
 * through the peers' mailboxes -- no host involvement, no NCCL call inside the solve.  All ranks must enqueue the same
 * solves in the same order. */
int blub_fluid_create_slab(BlubFluid **out, uint32_t nx, uint32_t ny, uint32_t nz_owned, uint32_t max_num_particles, int device,
                           void *cuda_stream, int rank, int world);
int blub_fluid_slab_window(BlubFluid *fluid, void **window, size_t *bytes);
int blub_fluid_attach_slab_peers(BlubFluid *fluid, void *const *windows, int world);
/* Once peers are attached, blub_fluid_step runs the WHOLE step sharded: halo sums of the P2G / density accumulators,
 * marker and velocity halos, and particle migration across the slab faces travel as stream-ordered peer copies and P2P
 * stores (blub_b200/csrc/slab.cu).  blub_fluid_add_cube then takes GLOBAL grid coordinates and every rank keeps its part
 * of the same particle stream; particle taps are in local coordinates (global z = local z - 4 + rank * nz_owned).
 * Returns 0, or 1 = a peer timed out, 2 = particle capacity exceeded, 3 = migration buffer overflow (synchronises).
 * The flag is also polled WITHOUT blocking at the start of every blub_fluid_step: once a finished step has reported a failure, the next
 * blub_fluid_step returns BLUB_ERR_CUDA instead of stepping on halos that never arrived. */
int blub_fluid_slab_error(BlubFluid *fluid);
int blub_ipc_export(const void *device_ptr, unsigned char handle[64]);
int blub_ipc_open(const unsigned char handle[64], int device, void **out);
int blub_ipc_close(void *mapped);
int blub_enable_peer_access(int device, int peer);

/* ---- test / bench taps (not part of the reference surface) ---------------------------------------------------- */
enum {
    BLUB_TAP_PARTICLE_POS = 0, BLUB_TAP_PARTICLE_VX = 1, BLUB_TAP_PARTICLE_VY = 2, BLUB_TAP_PARTICLE_VZ = 3,
    BLUB_TAP_GRID_VX = 4, BLUB_TAP_GRID_VY = 5, BLUB_TAP_GRID_VZ = 6, BLUB_TAP_MARKER = 7,
    BLUB_TAP_PRESSURE_VELOCITY = 8, BLUB_TAP_PRESSURE_DENSITY = 9, BLUB_TAP_RESIDUAL = 10,
    BLUB_TAP_SOLID_VOXELS = 11, /* the solid volume the step reads: the composite one with bodies, else the borrowed one (download only) */
    BLUB_TAP_CURVATURE = 12,    /* float per cell: the curvature (cells^-1) of the last stage 1 in the surface band, 0 elsewhere; zeros while
                                   surface tension is off (download only) */
    BLUB_TAP_DENSITY = 13,      /* DIAGNOSTIC, not a stable interface: the step's internal scratch density accumulator as the last stage that
                                   wrote it left it (int64 per cell: the stage-9 splat in 2^-40 particle weights when stage 9 ran without stage 7 in the same call
                                   -- after a whole step it is all zero --, or after a stage 1 with surface
                                   tension the smoothed field phi within 2 cells of FLUID).  Its contents and layout may change with the step's
                                   implementation; it exists so that tests can restate stage 1 bit for bit (download only) */
    BLUB_TAP_CELL_DENSITY = 14, /* float per cell: the relative density rho_i of the last stage 0 on FLUID cells, 0 elsewhere; zeros while no
                                   tag density table is set (download only) */
    BLUB_TAP_CELL_VISCOSITY = 15, /* float per cell: the kinematic viscosity nu_i (cells^2/s) of the last stage 0 on FLUID cells, 0 elsewhere;
                                    zeros while no tag viscosity table is set (download only) */
    BLUB_TAP_INTERFACE_CURVATURE = 16, /* float per cell: the interface's curvature (cells^-1) of the last stage 1 on the FLUID cells next to
                                          a FLUID cell of the other phase, 0 elsewhere; zeros while the interfacial tension is off (download
                                          only) */
    BLUB_TAP_INTERFACE_FIELD = 17      /* DIAGNOSTIC, not a stable interface: int64 per cell, the smoothed phase field phi (2^-32 particle
                                          weights, > 0 in phase B) of the last stage 1, valid within 2 cells of FLUID; elsewhere whatever an
                                          earlier step left.  Zeros while the interfacial tension is off.  Its contents and layout may change
                                          with the step's implementation; it exists so that tests can restate stage 1 bit for bit (download
                                          only) */
};
/* synchronous copies between host memory and the tapped array (bytes must not exceed the array) */
int blub_fluid_download(BlubFluid *fluid, int tap, void *host_dst, size_t bytes);
int blub_fluid_upload(BlubFluid *fluid, int tap, const void *host_src, size_t bytes);
/* replace the particle set (positions xyz + the tag bits in the fourth word, three velocity rows); rows may be NULL (zero) */
int blub_fluid_set_particles(BlubFluid *fluid, uint32_t count, const float *pos4, const float *vx4, const float *vy4,
                             const float *vz4);
/* run stages [from, to) of the 14-stage list of one step (same numbering as oracle/blub_oracle.c:orc_step_stages) */
int blub_fluid_step_stages(BlubFluid *fluid, double simulation_delta_seconds, int from, int to);
/* PCG only: solve for the rhs currently in the residual tap with the current markers; warm start from the field.  With a tag density table
 * the velocity solve (which 0) is the variable-density one, with the face coefficients of the last stage 0. */
int blub_fluid_solve_only(BlubFluid *fluid, int which, double simulation_delta_seconds);
/* viscosity only: applies the viscosity stage to the grid velocity and marker as they are (tap uploads), nothing else; with a tag viscosity
 * table it first forms the cell viscosities from the particles the fluid holds.  BLUB_ERR_INVALID_ARGUMENT while the stage is off */
int blub_fluid_viscosity_only(BlubFluid *fluid, double simulation_delta_seconds);
/* last finished solve of a field, synchronously: max|r| (not multiplied by dt) and iteration count */
int blub_fluid_last_solve(BlubFluid *fluid, int which, float *max_error, int32_t *iterations);
/* work list of the most recent solve (diagnostics for the in-step roofline; synchronises): out[0] = tiles walked by the tile body,
 * out[1] = quad columns walked by the column body, out[2] = cells per tile, out[3] = cells per column */
int blub_fluid_solver_work(BlubFluid *fluid, uint32_t out[4]);
/* scalars the last finished solve of a field left (diagnostics for tests of the solver; synchronises): out = {alpha, beta, sigma}.
 * A solve that stops after iteration K (0-based) leaves, by the kernels that actually run it (not the path that was requested: without
 * cooperative launch, or with BLUB_PCG=multikernel, paths 1, 2, 4 and 6 run the three-kernel code too)
 *   the persistent solvers (paths 1, 2, 4, 6, z-slab ranks) and the three-kernel code with precond_mode 1: (alpha_K, beta_{K-1}, sigma_K),
 *     beta_{-1} = 0;
 *   the three-kernel code with precond_mode 0, whose update kernel forms beta and sigma after it stops the solve: (alpha_K, beta_K,
 *     sigma_{K+1}).
 * Here sigma_k = z_k . r_k, alpha_k = sigma_k / (s_k . A s_k +- eps) and beta_k = sigma_{k+1} / (sigma_k +- eps). */
int blub_fluid_last_solve_scalars(BlubFluid *fluid, int which, float out[3]);
/* PCG micro-benchmark: `repetitions` times { restore the rhs that is in the residual tap now, zero the pressure field,
 * solve } with CUDA events around each solve on the fluid's stream; ms_each[repetitions] receives device milliseconds.
 * Synchronises. */
int blub_fluid_time_solve(BlubFluid *fluid, int which, double simulation_delta_seconds, int repetitions, float *ms_each);
/* device time of `steps` consecutive blub_fluid_step calls between two CUDA events on the fluid's stream (synchronises) */
int blub_fluid_time_steps(BlubFluid *fluid, double simulation_delta_seconds, int steps, float *ms_total);
/* one eagerly launched step with CUDA events between the 14 stages (same numbering as blub_fluid_step_stages); synchronises */
int blub_fluid_step_timed(BlubFluid *fluid, double simulation_delta_seconds, float ms_per_stage[14]);
/* PCG implementation: 1 (default) = one persistent cooperative kernel per solve -- tiles that are at least 3/4 FLUID by the
 * branch-free tile body, everything else as one compacted list of quad columns (z-slab ranks: tiles only);
 * 0 = three kernels per iteration; 2 = the persistent tile kernel with TMA-staged tiles (grids with nx % 128 == 0 only);
 * 4 = the persistent tile kernel without its per-thread sparsity skip; 6 = the persistent tile kernel (sparse tile bodies, no columns).
 * All paths run the same recurrence; 4 and 6 are bit-identical to each other.  A request that cannot be met returns
 * BLUB_ERR_INVALID_ARGUMENT and changes nothing. */
int blub_fluid_set_solver_path(BlubFluid *fluid, int persistent);
/* particle -> grid velocity transfer (transfer_gather_velocity.comp): 1 (default) = warp-aggregated scatter into 64-bit fixed-point
 * accumulator volumes (faster; what z-slab ranks always use), 0 = gather over per-step cell lists.  Both are bit-identical run to run;
 * they agree with each other to rounding only. */
int blub_fluid_set_transfer_path(BlubFluid *fluid, int scatter);
/* blub_fluid_step replays a captured CUDA graph of the step by default; 0 = launch every kernel eagerly instead */
int blub_fluid_set_graph_replay(BlubFluid *fluid, int enabled);
/* number of kernels launched by this library since the last reset (bench.py's gpu_launches) */
uint64_t blub_kernel_launch_count(int reset);

#ifdef __cplusplus
}
#endif
#endif /* BLUB_FLUID_H */
