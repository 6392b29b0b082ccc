// blub_core.hpp -- C++ host side of libblubcore: the H100-native counterparts of the reference's
// `HybridFluid` (src/simulation/hybrid_fluid.rs), `PressureSolver` and `PressureField`
// (src/simulation/pressure_solver.rs).  Same method names, argument meaning and defaults; wgpu objects are replaced by
// device pointers and one CUDA stream.  The C ABI in include/blub_fluid.h is a thin shim over these classes.
#pragma once
#include <deque>
#include <memory>
#include <string>
#include <vector>

#include "../../include/blub_fluid.h"
#include "common.cuh"
#include "fluid_kernels.hpp"

namespace blub {

// pressure_solver.rs:57-62
struct SolverConfig {
    float error_tolerance = 0.1f;
    int32_t max_num_iterations = 32;
    int32_t error_check_frequency = 4;
};
// pressure_solver.rs:63-68
struct SolverStatisticSample {
    float error = 0.0f;
    int32_t iteration_count = 0;
};
// hybrid_fluid.rs:19-22
struct DynamicSettings {
    uint32_t particle_rebinning_step_frequency = 60; // hybrid_fluid.rs:603-605
};

struct Quirks {
    int precond_mode = 0; // 0: z = r/diag^2 ("LOD-1 fetch returns 0"), 1: as written with clamped LOD (SURVEY B1)
};

// A mesh as the host holds it before it becomes a mesh body: present == false for a box or sphere.
struct HostMesh {
    bool present = false;
    float scale = 0.0f; // cells per model unit
    std::vector<float> positions;
    std::vector<uint32_t> indices;
};

// A body slot's host copy of a mesh body (DESIGN.md §8 "Mesh bodies"): its properties as stored, the float32 body-frame vertices and its
// indices; no vertices for a box or sphere.
struct MeshBodyHost {
    BlubMeshBodyProperties props{};
    float mid[3] = {0, 0, 0}; // (lo + hi) / 2 of the body-frame bounds
    std::vector<float> vertices;
    std::vector<uint32_t> indices;
};

// A padded device array of grid cells (see GridDim).
template <class T> struct GridArray {
    T *base = nullptr; // allocation
    T *ptr = nullptr;  // cell 0
    bool owned = true;
    static size_t bytes_for(const GridDim &g) { return (((size_t)(g.n + 2 * g.pad) * sizeof(T)) + 255) / 256 * 256; }
    void alloc(const GridDim &g) {
        size_t bytes = (size_t)(g.n + 2 * g.pad) * sizeof(T);
        BLUB_CUDA_CHECK(cudaMalloc(&base, bytes));
        BLUB_CUDA_CHECK(cudaMemset(base, 0, bytes));
        ptr = base + g.pad;
        owned = true;
    }
    // place the array in caller-owned, zero-initialised memory (the peer-visible slab window)
    void place(const GridDim &g, void *mem) {
        base = static_cast<T *>(mem);
        ptr = base + g.pad;
        owned = false;
    }
    void release() {
        if (base && owned) cudaFree(base);
        base = ptr = nullptr;
    }
};

// The setting of a fluid without viscosity, and the setter's range rules (std::invalid_argument names the field).
constexpr BlubViscosity kViscosityOff = {0.0f, 1e-4f, 200, 0u};
void check_viscosity(const BlubViscosity &v);
// A moving tank's frame (tank_kernels.cu): check_tank_frame throws std::invalid_argument on a non-finite value or a rotation that is not
// orthonormal with det +1 to 1e-6; tank_frame_rotates: omega or alpha is not zero.
void check_tank_frame(const BlubTankFrame &f);
bool tank_frame_rotates(const BlubTankFrame &f);
// Liquids of different densities (tag_density_kernels.cu): check_tag_densities throws std::invalid_argument on more than 16 entries, a tag listed
// twice or a density that is not finite or outside [1/2, 2]; make_tag_density_block is the device block of a checked table.
void check_tag_densities(const BlubTagDensity *table, uint32_t count);
TagDensityBlock make_tag_density_block(const BlubTagDensity *table, uint32_t count);
// Liquids of different viscosities (tag_density_kernels.cu): check_tag_viscosities throws std::invalid_argument on more than 16 entries, a
// NULL table with count > 0, a tag listed twice or a viscosity that is negative or not finite; tag_viscosity_scale is nu_scale, the largest
// of the table's values and the fluid's; make_tag_viscosity_block is the device block of a checked table.
void check_tag_viscosities(const BlubTagViscosity *table, uint32_t count);
float tag_viscosity_scale(const BlubTagViscosity *table, uint32_t count, float fluid_nu);
TagViscosityBlock make_tag_viscosity_block(const BlubTagViscosity *table, uint32_t count, float fluid_nu);

class PressureSolver;

// PressureField, pressure_solver.rs:84-210: one pressure volume (kept between steps = warm start), its solver
// configuration, and the asynchronous {max error, iteration count} read-back ring.
class PressureField {
  public:
    static constexpr size_t SOLVER_STATISTIC_HISTORY_LENGTH = 100; // pressure_solver.rs:101
    static constexpr int NUM_PRESSURE_ERROR_BUFFER = 32;           // pressure_solver.rs:49

    PressureField(const GridDim &grid, const SolverConfig &config, void *external_volume = nullptr);
    ~PressureField();
    PressureField(const PressureField &) = delete;

    SolverConfig config;
    std::deque<SolverStatisticSample> stats;
    float *pressure() const { return pressure_.ptr; }

    // PressureField::retrieve_new_error_samples, pressure_solver.rs:148-174 (never blocks)
    void retrieve_new_error_samples();
    // PressureField::enqueue_error_buffer_read, :176-191
    void enqueue_error_buffer_read(cudaStream_t stream, float simulation_delta);
    // blocking read of the device scalars (tests only)
    void read_last_solve(cudaStream_t stream, float *max_error, int *iterations);
    // blocking read of the scalars the last solve left: {alpha, beta, sigma} (tests only; conventions in blub_fluid.h)
    void read_last_scalars(cudaStream_t stream, float out[3]);

    PcgScalars *scalars = nullptr; // device
    bool touched = false;          // "timestamp_last_iteration == 0" of :601-603
    uint8_t *p_tiles = nullptr;    // device, per solver tile: the tile was active in this field's last solve (p may be non-zero there)

  private:
    struct Pending {
        cudaEvent_t event;
        float *host; // pinned {max_error, float(num_iterations)}
        float dt;
        bool in_flight;
    };
    GridArray<float> pressure_;
    std::vector<Pending> ring_;
    std::deque<int> pending_;
    std::vector<int> unused_;
    float *pinned_ = nullptr;
};

// PressureSolver, pressure_solver.rs:22-47,228-729: scratch volumes shared by both solves and the PCG recording.
class PressureSolver {
  public:
    PressureSolver(const GridDim &grid, void *external_residual = nullptr);
    ~PressureSolver();
    PressureSolver(const PressureSolver &) = delete;

    float *residual() const { return residual_.ptr; } // the rhs is written straight into it (hybrid_fluid.rs:836-838)

    // PressureSolver::solve, pressure_solver.rs:591-729.  Enqueue-only.  weights (liquids of different densities): the variable-density
    // operator, solved by pcg_solve_weighted_kernel whatever the path (precond_mode 0 and one GPU only); nullptr: the constant-density one.
    void solve(cudaStream_t stream, PressureField &field, int which, const int8_t *marker, const StepParams *dparams,
               const Quirks &quirks, const TagDensityWork *weights = nullptr);
    SlabComm comm; // filled by HybridFluid::attach_slab_peers; world == 1 when not sharded
    // {tiles walked by the tile body, quad columns walked by the column body, cells per tile, cells per column} of the last solve (blocking)
    void read_work(cudaStream_t stream, uint32_t out[4]);
    // The next solve of each field prepares every tile: enqueue after anything outside a step wrote a grid volume.
    void prepare_dense_next(cudaStream_t stream);

  private:
    GridDim grid_;
    GridArray<float> residual_, search_, aux_, aux_temp_;
    GridArray<uint8_t> codes_;       // per-cell code (diag | fluid << 3), rebuilt from the markers at the start of every solve
    uint8_t *tile_active_ = nullptr; // per-tile "contains FLUID" flag
    float *partials_ = nullptr;      // per-tile partial sums / maxima, 2 * tiles (+ slack for the persistent solver)
    int *tile_list_ = nullptr;       // compacted ids of the active tiles
    int *num_active_ = nullptr;
    int num_blocks_ = 0;
    int persistent_blocks_ = 0;      // co-resident blocks of the cooperative solver; 0 = not available
    // device {scratch volumes, pressure of field 0, of field 1}: non-zero = the next solve prepares every tile.  Kept on the device so
    // that a captured step graph follows them; set by prepare_dense_next and by solves on paths that may write outside the active tiles.
    int *dense_flags_ = nullptr;

  public:
    bool use_persistent = true;      // one cooperative launch per solve (diag2 preconditioner); false = three kernels per iteration
    bool use_tma = false;            // persistent solver with TMA-staged tiles (nx % 128 == 0); BLUB_PCG=tma or blub_fluid_set_solver_path(f, 2)
    bool use_dense = false;          // persistent solver without the per-thread sparsity skip (comparison only); set_solver_path(f, 4)
    bool use_columns = true;         // single GPU: dense tiles by the tile body, the rest as one list of quad columns (default); BLUB_PCG=tiles
                                     // or set_solver_path(f, 6) walks every active tile with the tile bodies instead
    bool tma_available() const { return tma_blocks_ > 0; }
    bool columns_available() const { return column_blocks_ > 0; }
    bool persistent_available() const { return persistent_blocks_ > 0; }
    // the value of blub_fluid_set_solver_path that selects the flags above (0, 1, 2, 4 or 6); set_path throws std::invalid_argument
    // on a request that cannot be met and then changes nothing
    int path() const { return !use_persistent ? 0 : use_tma ? 2 : use_dense ? 4 : use_columns ? 1 : 6; }
    void set_path(int path);

  private:
    void *tma_maps_ = nullptr;       // PcgTmaMaps (tensor maps of r, s0, s1, codes)
    int tma_blocks_ = 0, column_blocks_ = 0;
    int code_slots_ = 0;              // column solver: passes per thread whose code words stay in shared memory
    int p_slots_ = 0;                 // column solver, single GPU: passes per thread whose p stays in shared memory
    bool dense_setup_ = false;        // BLUB_PCG_SETUP=dense (test hook): the column solver prepares every tile on every solve
    int *tile_cols_ = nullptr;        // column solver: per-tile column counts | exclusive offsets | total
    int *col_list_ = nullptr;         // compacted quad columns (linear index of the quad in its tile's first plane)
    unsigned *barrier_ = nullptr;     // arrival counter of the column solver's grid-wide reductions

  public:
};

// HybridFluid, hybrid_fluid.rs:24-72,92-977
class HybridFluid {
  public:
    static constexpr uint32_t PARTICLES_PER_GRID_CELL = 8; // hybrid_fluid.rs:90

    // slab_world > 1: this fluid is rank `slab_rank` of a z-slab decomposition; `nz` is the number of OWNED planes and the
    // local grid gets SLAB_HALO ghost planes on both sides (see SlabComm).
    HybridFluid(uint32_t nx, uint32_t ny, uint32_t nz, uint32_t max_num_particles, int device, cudaStream_t stream, int slab_rank = 0,
                int slab_world = 1);
    ~HybridFluid();
    HybridFluid(const HybridFluid &) = delete;

    // returns true when the cube was truncated to max_num_particles (hybrid_fluid.rs:627-633); the new particles carry `tag`
    bool add_fluid_cube(const float min_grid[3], const float max_grid[3], uint32_t tag = 0);
    void set_gravity_grid(const float g[3]) { gravity_[0] = g[0]; gravity_[1] = g[1]; gravity_[2] = g[2]; }
    uint32_t num_particles() const;
    uint32_t num_active_particles() const { return num_particles(); }
    const GridDim &grid_dimension() const { return grid_; }
    SolverConfig &pressure_solver_config_velocity() { return field_velocity_->config; }
    SolverConfig &pressure_solver_config_density() { return field_density_->config; }
    DynamicSettings &dynamic_settings() { return dynamic_settings_; }
    const std::deque<SolverStatisticSample> &pressure_solver_stats_velocity() const { return field_velocity_->stats; }
    const std::deque<SolverStatisticSample> &pressure_solver_stats_density() const { return field_density_->stats; }
    void update_statistics();
    void set_solid_voxels(const void *rgba16f) { voxels_ = static_cast<const uint2 *>(rgba16f); }
    void step(double simulation_delta_seconds);
    void step_stages(double simulation_delta_seconds, int from, int to);
    // one eager step with CUDA events between the 14 stages; ms[14] (synchronises; diagnostics only)
    void step_timed(double simulation_delta_seconds, float ms[14]);
    bool use_graph = true; // replay the step as a CUDA graph (BLUB_NO_GRAPH=1 disables)
    void solve_only(int which, double simulation_delta_seconds);
    void synchronize();
    // peer-visible window (residual, both pressure volumes, mailbox) of a slab rank, and the peers' windows as mapped here
    void *slab_window() const { return window_; }
    size_t slab_window_bytes() const { return window_bytes_; }
    void attach_slab_peers(void *const *windows, int world);
    int slab_rank() const { return slab_rank_; }
    int slab_world() const { return slab_world_; }
    bool sharded() const { return slab_world_ > 1; }
    // 0 = fine; 1 = a peer timed out in a barrier; 2 = particle capacity exceeded; 3 = migration buffer overflow (synchronises)
    int slab_error();
    void invalidate_graphs() { destroy_graphs(); }
    void set_transfer_path(int scatter);
    void marker_written_externally() { fluid_bits_stale_ = true; }
    // a grid volume was written from outside the step: the next solves prepare every tile
    void grids_written_externally() { solver_->prepare_dense_next(stream_); }
    // number of whole steps taken (drives the rebinning cadence)
    uint32_t step_count() const { return step_counter_; }
    // Checkpoint / restart (state_file.cpp, format in DESIGN.md §8).  save_state synchronises, then writes everything a later step
    // depends on to `path` atomically; it refuses z-slab ranks and a fluid left inside a step by step_stages (std::invalid_argument).
    void save_state(const std::string &path);
    // a new fluid whose next step is bit for bit the step the saved fluid would have taken next (same library build, same GPU model)
    static std::unique_ptr<HybridFluid> load_state(const std::string &path, int device, cudaStream_t stream);

    Quirks quirks;

    // raw views (renderer bind group, hybrid_fluid.rs:351-369) and test taps
    float4 *particles_position() const { return pos_[cur_]; }
    float4 *particles_row(int c) const { return row_[c]; }
    float *grid_velocity(int c) const { return u_[c].ptr; }
    int8_t *marker() const { return marker_.ptr; }
    PressureField &field(int which) { return which == 0 ? *field_velocity_ : *field_density_; }
    PressureSolver &solver() { return *solver_; }
    cudaStream_t stream() const { return stream_; }
    int device() const { return device_; }
    uint32_t max_num_particles() const { return max_num_particles_; }
    void set_particles(uint32_t count, const float *pos4, const float *vx4, const float *vy4, const float *vz4);

    // Sources and drains (flow_kernels.cu): replaces the whole flow set; 0 / 0 clears it.  Throws std::invalid_argument and changes nothing on a
    // non-finite value, a box that is empty after clamping, overlapping sources, a source overlapping a drain, more than 16 boxes of a kind,
    // a z-slab rank or a fluid inside a step.  While the set is not empty the particle count lives on the device (num_particles()
    // synchronises).  source_tags: the tag of each source's emitted particles (nullptr = all 0).
    void set_flow(const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources, const BlubFluidDrain *drains, uint32_t num_drains);
    bool has_flow() const { return flow_active_; }
    const FlowSet &flow_set() const { return flow_; }
    // cumulative {emitted, drained, refused for capacity} (synchronises)
    void flow_counters(uint64_t out[3]);

    // Particle tags (flow_kernels.cu): the raw bits of the fourth word of every position.  paint_tags is stream-ordered and throws
    // std::invalid_argument (changing nothing) under the rules of set_flow for one box; tag_census synchronises and throws on num_tags of 0 or
    // above TAG_CENSUS_MAX or first + num_tags above 2^32.
    void paint_tags(const float min_grid[3], const float max_grid[3], uint32_t tag);
    void tag_census(uint32_t first, uint32_t num_tags, BlubTagCensus *out);

    // Solid load probes (load_kernels.cu): replaces the whole set (0 clears it), resets the history and drops the step graphs.  Throws
    // std::invalid_argument and changes nothing on more than LOAD_PROBES_MAX probes, a non-finite corner or pivot, a box empty after clamping,
    // a z-slab rank or a fluid inside a step.  While the set is not empty, stage 2 of every step records one BlubSolidLoad per probe.
    void set_load_probes(const BlubLoadProbe *probes, uint32_t num_probes);
    uint32_t num_load_probes() const { return num_load_probes_; }
    // the newest min(capacity, recorded, LOAD_HISTORY_LENGTH) records of `probe`, oldest first; returns their number (synchronises)
    uint32_t load_history(uint32_t probe, BlubSolidLoad *out, uint32_t capacity);

    // Floating bodies (body_kernels.cu): replaces the whole set (0 clears it), resets the history and drops the step graphs.  Throws
    // std::invalid_argument and changes nothing when make_body_set refuses the set, on a z-slab rank or a fluid inside a step.  While the set is
    // not empty, stage 0 builds the composite solid volume and stage 2 moves the bodies and records one BlubBodyRecord each.
    void set_bodies(const BlubBody *bodies, uint32_t num_bodies);
    uint32_t num_bodies() const { return num_bodies_; }
    // the current bodies, at most `capacity` of them (synchronises)
    uint32_t bodies(BlubBody *out, uint32_t capacity);
    // the newest min(capacity, recorded, BODY_HISTORY_LENGTH) records of `body`, oldest first; returns their number (synchronises)
    uint32_t body_history(uint32_t body, BlubBodyRecord *out, uint32_t capacity);
    // the solid volume the step reads: the composite one while there are bodies, else the borrowed one (may be nullptr)
    const uint2 *solid_volume() const { return num_bodies_ ? composite_ : voxels_; }
    // set_bodies with mesh bodies (DESIGN.md §8 "Mesh bodies"): meshes[i] != nullptr makes body i a mesh body scaled by scales[i].  Copies
    // the geometry; refuses what set_bodies and make_mesh_body refuse, a mesh on another device and sets over the vertex / triangle limits.
    void set_bodies_meshes(const BlubBody *bodies, const BlubMesh *const *meshes, const float *scales, uint32_t num_bodies);
    // the same with host meshes, one per body (meshes.size() bodies)
    void set_bodies_host(const BlubBody *bodies, const std::vector<HostMesh> &meshes);
    // the properties of mesh body `body` as stored; throws std::invalid_argument when it is not a mesh body
    BlubMeshBodyProperties body_mass_properties(uint32_t body) const;
    bool has_mesh_bodies() const { return !mesh_bodies_.empty(); }

    // Viscous liquids (viscosity_kernels.cu): nullptr or a kinematic viscosity of 0 turns the stage off while there is no tag viscosity table
    // (with one, 0 makes the tags not in it inviscid; the tolerance and the cap are kept either way).  Stream-ordered; the working volumes are
    // allocated with the first viscosity above zero, and only a change between off and on drops the step graphs.  Throws std::invalid_argument
    // and changes nothing on a value check_viscosity refuses, a z-slab rank or a fluid inside a step.
    void set_viscosity(const BlubViscosity *v);
    const BlubViscosity &viscosity() const { return viscosity_; }
    // iterations and max |r| per component of the last viscosity solve (synchronises); zeros before the first one
    void last_viscosity_solve(int32_t *iterations, float max_error[3]);
    // test hook: the viscosity stage on the grid velocity and marker as they are (with a tag viscosity table, the cell viscosities are first
    // formed from the particles the fluid holds)
    void viscosity_only(double simulation_delta_seconds);
    // Liquids of different viscosities (viscosity_kernels.cu): replaces the table, count 0 clears it.  Stream-ordered; the working volumes are
    // allocated with the first non-empty table, and only a change that turns the table or the stage on or off drops the step graphs.  Throws
    // std::invalid_argument and changes nothing on a table check_tag_viscosities refuses, a z-slab rank or a fluid inside a step.
    void set_tag_viscosities(const BlubTagViscosity *table, uint32_t count);
    const std::vector<BlubTagViscosity> &tag_viscosities() const { return tag_viscosities_; }
    float *cell_viscosity() const { return tv_.nu; } // nullptr before the first non-empty table
    // the viscosity stage runs: the fluid's nu or a value of the table is above 0
    bool viscosity_on() const;

    // CFL-limited substeps (cfl_kernels.cu): max |v_c| over the live particles per axis (one kernel, then synchronises), and the next substep
    // of `remaining_ns` by cfl_substep_ns with this fluid's gravity (max_velocity_out, may be nullptr, receives the measurement even when the
    // rule refuses it).  Both throw std::invalid_argument on a z-slab rank or a fluid inside a step; plan_substep checks its arguments before it
    // launches anything.  The 12-byte result is allocated with the first measurement.
    void max_particle_velocity(float out[3]);
    uint64_t plan_substep(uint64_t remaining_ns, const BlubTimeStepping &ts, float max_velocity_out[3]);

    // Surface tension (surface_tension_kernels.cu): a kinematic surface tension in cells^3/s^2, 0 turns it off.  Stream-ordered; the working
    // volumes are allocated with the first value above zero, and only a change between off and on drops the step graphs.  Throws
    // std::invalid_argument and changes nothing on a negative or non-finite value, a z-slab rank or a fluid inside a step.  While it is on,
    // plan_substep holds every substep to capillary_limit_ns.
    void set_surface_tension(float cells3_per_s2);
    float surface_tension() const { return surface_tension_; }
    // Moving tanks (tank_kernels.cu): the frame of the following steps (nullptr: at rest).  Not state.  Throws std::invalid_argument and changes
    // nothing on a frame check_tank_frame refuses, a rotating frame while the fluid has bodies, a z-slab rank or a fluid inside a step.  Only a
    // change between rotating and not rotating drops the step graphs.
    void set_tank_frame(const BlubTankFrame *frame);
    const BlubTankFrame *tank_frame() const { return has_tank_frame_ ? &tank_frame_ : nullptr; }
    float *curvature() const { return st_.kappa; }             // nullptr before the first surface tension above zero
    // Interfacial tension (surface_tension_kernels.cu): a kinematic tension in cells^3/s^2 between phase B (the particles whose tag is one of
    // `tags`) and the rest of the liquid, 0 turns it off.  Stream-ordered; the working volumes are allocated with the first value above zero,
    // and only a change between off and on drops the step graphs.  Throws std::invalid_argument and changes nothing on a value or set
    // check_interfacial_tension refuses, a z-slab rank or a fluid inside a step.  While it is on, plan_substep holds every substep to the
    // capillary limit of the larger tension.
    void set_interfacial_tension(const uint32_t *tags, uint32_t count, float cells3_per_s2);
    float interfacial_tension() const { return interfacial_tension_; }
    const std::vector<uint32_t> &interface_tags() const { return interface_tags_; }
    float *interface_curvature() const { return it_.kappa; } // nullptr before the first interfacial tension above zero
    long long *interface_field() const { return it_.phi; }   // likewise
    long long *density_accumulator() const { return density_.ptr; }
    // Liquids of different densities (tag_density_kernels.cu): replaces the table, count 0 turns the feature off.  Stream-ordered; the working
    // volumes are allocated with the first non-empty table, and only a change between off and on drops the step graphs.  Throws
    // std::invalid_argument and changes nothing on a table check_tag_densities refuses, a table while the surface tension is above 0 or floating bodies are set, precond_mode
    // 1, a z-slab rank or a fluid inside a step.
    void set_tag_densities(const BlubTagDensity *table, uint32_t count);
    const std::vector<BlubTagDensity> &tag_densities() const { return tag_densities_; }
    bool has_tag_densities() const { return !tag_densities_.empty(); }
    float *cell_density() const { return td_.rho; } // nullptr before the first non-empty table

    // Whitewater (whitewater_kernels.cu): nullptr or a capacity of 0 turns it off, frees its memory and stores an all-zero setting.  A new
    // capacity starts from no particles and zero counters (its storage is allocated before the old one is freed), another change keeps them;
    // every change drops the step graphs.  Throws std::invalid_argument and changes nothing on a
    // setting check_whitewater refuses, a z-slab rank or a fluid inside a step.
    void set_whitewater(const BlubWhitewater *s);
    const BlubWhitewater &whitewater() const { return whitewater_; }
    bool whitewater_on() const { return whitewater_.max_num_particles > 0; }
    // {live, emitted, removed, refused}, zeros while off (synchronises)
    void whitewater_counters(uint64_t out[4]);
    // the live particles, at most `capacity` of them (pos4 / vel4: 4 floats each); returns the live count (synchronises)
    uint32_t download_whitewater(float *pos4, float *vel4, uint32_t capacity);

  private:
    BlubWhitewater whitewater_{};
    WhitewaterWork ww_;
    // a state file's whitewater: the setting, the counters {emitted, removed, refused} and `count` particles (4 + 4 floats each, host memory)
    void restore_whitewater(const BlubWhitewater &s, const uint64_t counters[3], uint32_t count, const float *particles);
    std::vector<BlubTagDensity> tag_densities_;
    TagDensityWork td_;
    const TagDensityWork *solve_weights() const { return tag_densities_.empty() ? nullptr : &td_; }
    BlubTankFrame tank_frame_{};
    bool has_tank_frame_ = false;
    bool tank_rotating() const { return has_tank_frame_ && tank_frame_rotates(tank_frame_); }
    uint32_t *max_velocity_dev_ = nullptr;
    BlubBody *bodies_dev_ = nullptr;          // BODIES_MAX bodies, BODIES_MAX x 8 sums, BODIES_MAX x BODY_HISTORY_LENGTH records and the
    unsigned long long *body_sums_ = nullptr; // composite volume, allocated with the first non-empty set
    BlubBodyRecord *body_ring_ = nullptr;
    uint2 *composite_ = nullptr;
    uint32_t num_bodies_ = 0, body_cube_ = 0;
    std::deque<uint32_t> body_steps_; // step numbers of the records in the body ring, oldest first
    // a validated set (set_bodies, state file load); meshes: one host copy per body when the set has mesh bodies, else empty
    void restore_bodies(const std::vector<BlubBody> &bodies, std::vector<MeshBodyHost> meshes = {});
    std::vector<MeshBodyHost> mesh_bodies_; // one per body while the set has a mesh body, else empty
    MeshBodySet mesh_;                      // device arrays, reallocated by every set with mesh bodies
    void free_mesh_bodies();
    BlubViscosity viscosity_ = kViscosityOff;
    ViscosityWork visc_;
    std::vector<BlubTagViscosity> tag_viscosities_;
    TagViscosityWork tv_;
    void ensure_viscosity_work();
    float surface_tension_ = 0.0f;
    SurfaceTensionWork st_;
    float interfacial_tension_ = 0.0f;
    std::vector<uint32_t> interface_tags_;
    InterfacialTensionWork it_;
    void run_viscosity();
    LoadProbeBox *load_probes_dev_ = nullptr; // LOAD_PROBES_MAX boxes and LOAD_PROBES_MAX x LOAD_HISTORY_LENGTH records, allocated with the
    BlubSolidLoad *load_ring_ = nullptr;      // first non-empty set
    uint32_t num_load_probes_ = 0, load_max_cells_ = 0;
    std::deque<uint32_t> load_steps_; // step numbers of the records in the ring, oldest first (at most LOAD_HISTORY_LENGTH)
    void note_load_record(uint32_t step);
    BlubTagCensus *census_dev_ = nullptr; // TAG_CENSUS_MAX records, allocated with the first census
    bool device_count_mode() const { return slab_world_ > 1 || flow_active_; }
    void run_flow_prologue();
    void restore_flow(const FlowSet &set, const uint64_t counters[3]); // state file load
    FlowSet flow_{};
    bool flow_active_ = false;
    FlowScratch flow_scratch_{}; // the drain compaction writes into pos_[1 - cur_] (free at stage 0) and row_alt_ (allocated with the first drain)
    uint32_t flow_scratch_cells_ = 0; // source cells the scratch has room for
    void upload_step_params(float dt);
    void run_stage(int stage, float dt);
    void refresh_fluid_bits();
    bool binning_step() const;
    uint32_t internal_resort_every_ = 8; // see binning_step(); single GPU and z-slab ranks alike
    void destroy_graphs();
    // brick schedule of the density and P2G scatters, rebuilt at every re-sort (single GPU, unless BLUB_SCATTER_SCHEDULE=off: then valid == nullptr).  It is
    // not state: a fluid that is loaded, or whose particles are replaced or added to, runs the 256-particle chunks until its next re-sort.
    ScatterSchedule sched_{};
    void invalidate_schedule();

    // ---- z-slab sharding of the whole step (slab.cu) ----
    struct SlabHaloItem {
        void *cell0;           // cell-0 pointer of a grid volume
        size_t bytes_per_cell;
        int kind;              // 0 SUM (64-bit fixed-point data) / 1 MAX (int8) over the 4 overlap planes, 2 COPY of 2 owned planes into the ghost planes
    };
    size_t slab_extra_window_bytes() const;
    uint32_t slab_migrant_capacity() const;
    void slab_layout(void *window, char *&halo0, size_t &halo_bytes, char *&part0, size_t &part_bytes, unsigned int *&counts) const;
    void slab_barrier();
    void slab_halo_exchange(const SlabHaloItem *items, int n_items);
    MigrateOut slab_migrate_targets();
    void slab_migrate_finish();
    void set_device_particle_count(uint32_t n);
    bool add_fluid_cube_slab(const uint32_t mn[3], const uint32_t ext[3], uint32_t tag);
    uint32_t seeded_global_ = 0;
    float4 *row_alt_[3] = {nullptr, nullptr, nullptr}; // spare velocity rows: migration compacts out of place
    unsigned int *mig_counters_ = nullptr;
    int *slab_error_ = nullptr;      // device alias of slab_error_host_
    int *slab_error_host_ = nullptr; // mapped pinned flag: 0 fine, 1 peer timed out, 2 particle capacity exceeded, 3 migration buffer overflow
    void *slab_peer_window_[2] = {nullptr, nullptr};
    uint32_t slab_exchange_index_ = 0;

    // Cached executable graphs of one step, keyed by (position buffer in use, binning step?).  Everything a graph bakes
    // in besides that key is in `GraphSignature`; a change drops the cache.
    struct GraphSignature {
        uint32_t num_particles = 0xFFFFFFFFu;
        const void *voxels = nullptr;
        int precond_mode = -1;
        int max_it[2] = {-1, -1}, freq[2] = {-1, -1};
        bool operator==(const GraphSignature &o) const {
            return num_particles == o.num_particles && voxels == o.voxels && precond_mode == o.precond_mode && max_it[0] == o.max_it[0] &&
                   max_it[1] == o.max_it[1] && freq[0] == o.freq[0] && freq[1] == o.freq[1];
        }
    };
    GraphSignature graph_signature_;
    // key: [position buffer][binning step?][velocity-row buffer (slab migration)][halo receive buffer (slab exchanges)]
    cudaGraphExec_t graph_exec_[2][2][2][2] = {};
    uint64_t graph_kernel_nodes_[2][2][2][2] = {}; // kernels inside each graph (for blub_kernel_launch_count)
    int row_parity_ = 0;                           // toggled by every slab migration (row_ <-> row_alt_)
    struct GraphRolesAfter {
        int cur, row_parity;
        uint32_t exchanges;
        bool density_zero;
    };
    GraphRolesAfter graph_roles_after_[2][2][2][2] = {};
    bool capturing_ = false;
    bool mid_step_ = false; // the last step_stages call did not end at stage 14: the fluid is inside a step and cannot be saved

    GridDim grid_;
    int device_;
    cudaStream_t stream_;
    bool owns_stream_;
    uint32_t max_num_particles_, num_particles_ = 0;
    float gravity_[3] = {0, 0, 0};
    uint32_t step_counter_ = 0;
    DynamicSettings dynamic_settings_;

    float4 *pos_[2] = {nullptr, nullptr}; // ping-pong for the binning reorder
    int cur_ = 0;
    float4 *row_[3] = {nullptr, nullptr, nullptr};
    GridArray<float> u_[3];
    GridArray<long long> density_;     // density scatter accumulator, 64-bit fixed point (common.cuh: to_fixed)
    // Stage 7 scatters the density of the new positions along with the advection (launch_advect_density) on one GPU and grids of 2^21 cells
    // or more (BLUB_DENSITY_FUSE=off / on, read when the fluid is created, decides for any grid); stage 9 then only finishes it on the
    // particles' cells and leaves the volume zero.
    bool density_fuse_ = true;
    bool density_fused_ = false; // stage 7 of the running step / step_stages call scattered the density of the positions as they are now
    bool density_zero_ = true;   // the density volume is all zero once the enqueued work has run: the fused stage 7 needs no memset
    GridArray<longlong2> numw_[3];     // scatter-form P2G accumulators: (sum w*value, sum w) per face, 64-bit fixed point
    FluidBits fluid_bits_ = {nullptr, 0}; // 1 bit per cell "FLUID", rebuilt with every finished marker volume
    bool fluid_bits_stale_ = false;       // the marker volume was written through a tap since
    GridArray<int8_t> marker_;
    CellLists lists_ = {nullptr, nullptr, nullptr, nullptr, nullptr, {nullptr, nullptr, nullptr, nullptr}}; // per-step cell lists (P2G gather, binning)
    uint32_t *particle_words_ = nullptr;  // 1 bit per cell "a particle marked this cell" (scatter form: which accumulators to visit and re-zero)
    bool use_scatter_ = true;             // scatter form of P2G (default; z-slab ranks always); false = deterministic gather over cell lists
    const uint2 *voxels_ = nullptr;

    std::unique_ptr<PressureSolver> solver_;
    std::unique_ptr<PressureField> field_velocity_, field_density_;

    int slab_rank_ = 0, slab_world_ = 1;
    void *window_ = nullptr;
    size_t window_bytes_ = 0;

    StepParams *params_dev_ = nullptr;
    StepParams *params_host_ = nullptr; // pinned ring of 64
    uint32_t step_param_slot_ = 0;
    cudaEvent_t param_events_[64] = {};
};

// Errors of the state file reader / writer: IoError = the file cannot be opened, written or read (BLUB_ERR_IO); ParseError = it is not a
// valid state file of this format version (BLUB_ERR_PARSE).
struct IoError : std::runtime_error {
    explicit IoError(const std::string &what) : std::runtime_error(what) {}
};
struct ParseError : std::runtime_error {
    explicit ParseError(const std::string &what) : std::runtime_error(what) {}
};
// A CFL substep that cannot be planned: a non-finite particle velocity, or a step below min_dt_ns (BLUB_ERR_UNSTABLE).
struct UnstableError : std::runtime_error {
    explicit UnstableError(const std::string &what) : std::runtime_error(what) {}
};
// CFL-limited substeps (cfl_kernels.cu, DESIGN.md §8): the config's range rules (std::invalid_argument), and the host rule of blub_cfl_substep_ns.
void check_time_stepping(const BlubTimeStepping &ts);
// Brackbill's capillary step limit with dx = 1 cell and the mean of the liquid and air densities: floor(1e9 sqrt(1 / (4 pi s))) ns for a
// kinematic surface tension s > 0 (cells^3/s^2), saturating at UINT64_MAX.
uint64_t capillary_limit_ns(float cells3_per_s2);
// The interfacial tension setter's rules: s finite and >= 0, at most BLUB_INTERFACE_TAGS_MAX tags, none twice, not NULL with count > 0, and
// at least one tag when s > 0.  Throws std::invalid_argument naming `who`.
void check_interfacial_tension(const uint32_t *tags, uint32_t count, float s, const char *who);
uint64_t cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTimeStepping &ts);
// Moving tanks (tank_kernels.cu, DESIGN.md §8 "Moving tanks"): the host rules of blub_tank_frame_at, blub_tank_step_constants and
// blub_tank_cfl_substep_ns (frame == nullptr: cfl_substep_ns).
BlubTankFrame tank_frame_at(const BlubTankMotion &m, double t_seconds);
BlubTankStepConstants tank_step_constants(const BlubTankFrame &f, const float gravity_grid[3], float dt);
uint64_t tank_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTankFrame *frame,
                             const uint32_t dim[3], const BlubTimeStepping &ts);
struct StateInfo {
    uint32_t grid_dimension[3], max_num_particles, num_particles, step_count, format_version;
};
// A box in grid units clamped like add_fluid_cube (corners in [1, dim - 1], max exclusive); throws std::invalid_argument on a non-finite corner
// or a box that is empty after clamping (`what` names it in the message).
FlowBox clamp_box(const uint32_t dim[3], const float min_grid[3], const float max_grid[3], const char *what);
// A load probe in grid units: corners converted as clamp_box converts them but clamped to [0, dim] (max exclusive); throws
// std::invalid_argument on a non-finite corner or pivot or a box that is empty after clamping.
LoadProbeBox clamp_load_probe(const uint32_t dim[3], const BlubLoadProbe &probe);
// A body set checked against the rules of set_bodies on a grid of `dim` cells; throws std::invalid_argument when it breaks one.  set_bodies
// (loaded == false) normalises the quaternions; a state file's bodies (loaded == true) are kept bit for bit and their bounding boxes may
// leave [1, dim - 1] by the rounding of the integrator's clamp (1e-3 cells).
std::vector<BlubBody> make_body_set(const uint32_t dim[3], const BlubBody *bodies, uint32_t num_bodies, bool loaded);

// Mesh bodies (mesh_body.cpp, DESIGN.md §8 "Mesh bodies").
// Checks a mesh and computes its mass properties and principal frame (blub_mesh_body_properties); throws std::invalid_argument.
// body_vertices (if given) receives the float32 body-frame vertices.
BlubMeshBodyProperties mesh_body_properties(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale,
                                            std::vector<float> *body_vertices);
// A mesh body placed by `placement` (centre and rotation: the model origin and axes in the grid): its host copy and, in `stored`, the BlubBody
// the device keeps (centre of mass, model rotation * principal rotation, half extents of the body-frame bounds).  Checks the placement as
// set_bodies does and the bounding box against [1, dim - 1] (skipped when dim == nullptr); throws std::invalid_argument.
MeshBodyHost make_mesh_body(const uint32_t dim[3], const BlubBody &placement, const float *positions, uint32_t num_vertices, const uint32_t *indices,
                            uint32_t num_indices, float scale, BlubBody &stored);
// A body set with mesh bodies checked against the rules of set_bodies_meshes: `set` receives the stored bodies; returns one host copy per body,
// or none when no body has a mesh.  Throws std::invalid_argument.
std::vector<MeshBodyHost> make_mesh_body_set(const uint32_t dim[3], const BlubBody *bodies, const std::vector<HostMesh> &meshes, std::vector<BlubBody> &set);
// The setter's view of a mesh body's grid-axis bounding box: e = its half extents, off = R mid its centre relative to the centre of mass.
// Not bit-exact with the device: off is float64 rounded once, not the device's float32 dot3, so a pose within rounding of [1, dim - 1] may be
// accepted here and then moved by the first step's clamp.
void mesh_body_box(const BlubBody &b, const float mid[3], float e[3], float off[3]);
// The launch cube side of a mesh body: from the farthest corner of its body-frame bounds to the centre of mass.
uint32_t mesh_body_cube_side(const float h[3], const float mid[3]);
void quat_rotation_f64(const double q[4], double R[9]);
// cgmath's Quaternion::from(Euler<Deg>) as (w, x, y, z) (solids.cu)
void quat_from_euler_deg_wxyz(const float deg[3], float q[4]);
// A flow set from the public boxes (grid units), clamped like add_fluid_cube; throws std::invalid_argument when it breaks a rule of set_flow
// that does not depend on the fluid.  source_tags may be nullptr (all 0).
FlowSet make_flow_set(const uint32_t dim[3], const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources, const BlubFluidDrain *drains,
                      uint32_t num_drains);
// The whitewater setter's rules (DESIGN.md §8 "Whitewater"); throws std::invalid_argument naming `who` and the field.  A capacity of 0 is off
// and passes whatever the other fields hold.
void check_whitewater(const BlubWhitewater &s, const char *who);
// Host only: reads and validates the whole state file (header, every section length and checksum).
StateInfo read_state_info(const std::string &path);

void voxelize_rigid_solid(void *rgba16f, const uint32_t dim[3], const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3],
                          double total_time, double delta, int clear_first, cudaStream_t stream, BlubRigidState *state_out);

// shared animation evaluation (solids.cu) and the triangle-mesh hull voxelizer (mesh_voxelizer.cu)
void rigid_state_at(const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3], double total_time, double delta,
                    BlubRigidState &out);
BlubMesh *mesh_create(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, int device);
void mesh_destroy(BlubMesh *mesh);
void mesh_info(const BlubMesh &mesh, uint32_t &num_vertices, uint32_t &num_triangles);
int mesh_device(const BlubMesh &mesh);
// the mesh's positions and indices, copied to the host (synchronous)
void mesh_download(const BlubMesh &mesh, std::vector<float> &positions, std::vector<uint32_t> &indices);
void voxelize_mesh(void *rgba16f, const uint32_t dim[3], BlubMesh &mesh, const BlubRigidObject &o, float grid_to_world_scale, const float fluid_world_position[3],
                   double total_time, double delta, int clear_first, cudaStream_t stream, BlubRigidState *state_out);
void read_obj(const std::string &path, std::vector<float> &positions, std::vector<uint32_t> &indices);

// scene JSON (src/scene/mod.rs:19-43)
struct SceneStaticObject {
    std::string model;          // path below the reference's `models/` directory (models.rs:253)
    BlubRigidObject placement;  // pose + animation; shape = 2 (mesh)
};
struct SceneBox {
    float min[3], max[3];
    uint32_t tag = 0; // optional "tag" of a fluid cube (drains have none)
};
struct SceneSource {
    float min[3], max[3], velocity[3];
    uint32_t tag = 0;
};
struct SceneLoadProbe {
    float min[3], max[3], pivot[3];
    bool has_pivot = false; // without one the pivot is the box centre
};
struct SceneBody {
    int32_t shape = 0;            // "box" 0, "sphere" 1, "mesh" 2
    std::string model;            // a mesh body's OBJ file, resolved against the scene file's directory
    float model_scale = 1.0f;     // a mesh body's world units per model unit
    float position[3], half_extent[3], rotation_angles_deg[3] = {0, 0, 0}, relative_density = 1.0f;
    float velocity[3] = {0, 0, 0}, angular_velocity[3] = {0, 0, 0}; // m/s, rad/s
};
struct SceneConfig {
    float gravity[3] = {0, 0, 0};
    float world_position[3] = {0, 0, 0};
    float grid_to_world_scale = 1.0f;
    uint32_t grid_dimension[3] = {0, 0, 0};
    uint32_t max_num_particles = 0;
    std::vector<SceneBox> fluid_cubes;
    std::vector<SceneSource> sources; // optional fluid.sources / fluid.drains (world units, m/s)
    std::vector<SceneBox> drains;
    std::vector<SceneLoadProbe> load_probes; // optional fluid.load_probes (world units)
    std::vector<SceneBody> bodies;           // optional fluid.bodies (world units, m/s)
    float viscosity = 0.0f;                  // optional fluid.viscosity: kinematic, m^2/s
    float surface_tension = 0.0f;            // optional fluid.surface_tension: kinematic, m^3/s^2
    float interfacial_tension = 0.0f;        // optional fluid.interfacial_tension: kinematic, m^3/s^2, between the tags below and the rest
    std::vector<uint32_t> interface_tags;    // checked with the setter's rules
    std::vector<BlubTagDensity> tag_densities; // optional fluid.tag_densities, checked with the setter's rules
    std::vector<BlubTagViscosity> tag_viscosities; // optional fluid.tag_viscosities (m^2/s), checked in cells^2/s with the setter's rules
    bool has_whitewater = false;             // optional fluid.whitewater, in grid units (the energy range / grid_to_world_scale^2), checked
    BlubWhitewater whitewater{};
    bool has_tank_motion = false;            // optional fluid.tank_motion (world units, Hz, rad, rad/s; directions and axis normalised)
    BlubTankMotion tank_motion{};
    uint32_t num_static_objects = 0;
    std::vector<SceneStaticObject> static_objects;
};
SceneConfig parse_scene_file(const std::string &path);
// the scene's load probes in grid cells: corners and pivot / grid_to_world_scale, pivot (min + max) / 2 when the scene gives none
std::vector<BlubLoadProbe> scene_load_probes_grid(const SceneConfig &cfg);
// the scene's tank motion in grid cells: pivot and amplitudes / grid_to_world_scale (in float32, as the load probes' pivots), the rest as parsed
BlubTankMotion scene_tank_motion_grid(const SceneConfig &cfg);
// the scene's kinematic viscosity in cells^2/s: viscosity / grid_to_world_scale^2
float scene_viscosity_grid(const SceneConfig &cfg);
std::vector<BlubTagViscosity> scene_tag_viscosities_grid(const SceneConfig &cfg); // fluid.tag_viscosities in cells^2/s
// the scene's kinematic surface tension in cells^3/s^2: surface_tension / grid_to_world_scale^3
float scene_surface_tension_grid(const SceneConfig &cfg);
// the scene's kinematic interfacial tension in cells^3/s^2: interfacial_tension / grid_to_world_scale^3
float scene_interfacial_tension_grid(const SceneConfig &cfg);
// the scene's bodies in grid cells and cells/s: (position - world_position) / scale, half extents and velocity / scale, the Euler angles as a
// quaternion (quat_from_euler_deg_wxyz), the angular velocity unchanged
std::vector<BlubBody> scene_bodies_grid(const SceneConfig &cfg);
// the scene's bodies' meshes (read from their OBJ files; scale in cells per model unit = model_scale / grid_to_world_scale), one per body
std::vector<HostMesh> scene_body_meshes(const SceneConfig &cfg);
// Scene::create_fluid_from_config, src/scene/mod.rs:109-144
std::unique_ptr<HybridFluid> create_fluid_from_config(const SceneConfig &cfg, int device, cudaStream_t stream);

} // namespace blub
