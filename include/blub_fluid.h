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
    const void *particles_position_ll;            /* num_particles x {float3 pos, uint32 unused}  */
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
    BLUB_TAP_PRESSURE_VELOCITY = 8, BLUB_TAP_PRESSURE_DENSITY = 9, BLUB_TAP_RESIDUAL = 10
};
/* synchronous copies between host memory and the tapped array (bytes must not exceed the array) */
int blub_fluid_download(BlubFluid *fluid, int tap, void *host_dst, size_t bytes);
int blub_fluid_upload(BlubFluid *fluid, int tap, const void *host_src, size_t bytes);
/* replace the particle set (positions xyz_, three velocity rows); rows may be NULL (zero) */
int blub_fluid_set_particles(BlubFluid *fluid, uint32_t count, const float *pos4, const float *vx4, const float *vy4,
                             const float *vz4);
/* run stages [from, to) of the 14-stage list of one step (same numbering as oracle/blub_oracle.c:orc_step_stages) */
int blub_fluid_step_stages(BlubFluid *fluid, double simulation_delta_seconds, int from, int to);
/* PCG only: solve for the rhs currently in the residual tap with the current markers; warm start from the field */
int blub_fluid_solve_only(BlubFluid *fluid, int which, double simulation_delta_seconds);
/* last finished solve of a field, synchronously: max|r| (not multiplied by dt) and iteration count */
int blub_fluid_last_solve(BlubFluid *fluid, int which, float *max_error, int32_t *iterations);
/* work list of the most recent solve (diagnostics for the in-step roofline; synchronises): out[0] = tiles walked by the tile body,
 * out[1] = quad columns walked by the column body, out[2] = cells per tile, out[3] = cells per column */
int blub_fluid_solver_work(BlubFluid *fluid, uint32_t out[4]);
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
