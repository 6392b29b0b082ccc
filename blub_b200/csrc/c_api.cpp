// c_api.cpp -- the extern "C" boundary (include/blub_fluid.h) over blub::HybridFluid.  Nothing throws across it.
#include <algorithm>
#include <cstring>
#include <ios>
#include <new>

#include "../../include/blub_fluid.h"
#include "blub_core.hpp"

struct BlubFluid {
    std::unique_ptr<blub::HybridFluid> impl;
    BlubSolverConfig config_mirror[2]; // BlubSolverConfig and blub::SolverConfig are layout-identical; see static_asserts
    uint32_t rebin_mirror;
};

static_assert(sizeof(BlubSolverConfig) == sizeof(blub::SolverConfig), "SolverConfig layout");
static_assert(sizeof(BlubSolverSample) == sizeof(blub::SolverStatisticSample), "SolverStatisticSample layout");

namespace {
thread_local std::string g_last_error;

int fail(int code, const std::string &what) {
    g_last_error = what;
    return code;
}

template <class F> int guarded(F &&f) {
    try {
        return f();
    } catch (const blub::CudaError &e) {
        return fail(BLUB_ERR_CUDA, e.what());
    } catch (const std::bad_alloc &e) {
        return fail(BLUB_ERR_OUT_OF_MEMORY, e.what());
    } catch (const std::invalid_argument &e) {
        return fail(BLUB_ERR_INVALID_ARGUMENT, e.what());
    } catch (const std::ios_base::failure &e) {
        return fail(BLUB_ERR_IO, e.what());
    } catch (const blub::IoError &e) {
        return fail(BLUB_ERR_IO, e.what());
    } catch (const blub::ParseError &e) {
        return fail(BLUB_ERR_PARSE, e.what());
    } catch (const blub::UnstableError &e) {
        return fail(BLUB_ERR_UNSTABLE, e.what());
    } catch (const std::exception &e) {
        return fail(BLUB_ERR_PARSE, e.what());
    } catch (...) {
        return fail(BLUB_ERR_CUDA, "unknown exception");
    }
}

struct Tap {
    void *ptr;
    size_t bytes;
};
Tap tap_of(BlubFluid *f, int tap) {
    blub::HybridFluid &h = *f->impl;
    const size_t n = (size_t)h.grid_dimension().n;
    const size_t np = (size_t)h.num_particles() * sizeof(float4);
    switch (tap) {
    case BLUB_TAP_PARTICLE_POS: return {h.particles_position(), np};
    case BLUB_TAP_PARTICLE_VX: return {h.particles_row(0), np};
    case BLUB_TAP_PARTICLE_VY: return {h.particles_row(1), np};
    case BLUB_TAP_PARTICLE_VZ: return {h.particles_row(2), np};
    case BLUB_TAP_GRID_VX: return {h.grid_velocity(0), n * 4};
    case BLUB_TAP_GRID_VY: return {h.grid_velocity(1), n * 4};
    case BLUB_TAP_GRID_VZ: return {h.grid_velocity(2), n * 4};
    case BLUB_TAP_MARKER: return {h.marker(), n};
    case BLUB_TAP_PRESSURE_VELOCITY: return {h.field(0).pressure(), n * 4};
    case BLUB_TAP_PRESSURE_DENSITY: return {h.field(1).pressure(), n * 4};
    case BLUB_TAP_RESIDUAL: return {h.solver().residual(), n * 4};
    case BLUB_TAP_SOLID_VOXELS: return {const_cast<uint2 *>(h.solid_volume()), n * 8};
    case BLUB_TAP_CURVATURE: return {h.curvature(), n * 4}; // nullptr before the first surface tension above zero: zeros
    case BLUB_TAP_DENSITY: return {h.density_accumulator(), n * 8};
    case BLUB_TAP_CELL_DENSITY: return {h.cell_density(), n * 4}; // nullptr before the first table: zeros
    case BLUB_TAP_CELL_VISCOSITY: return {h.cell_viscosity(), n * 4}; // nullptr before the first table: zeros
    case BLUB_TAP_INTERFACE_CURVATURE: return {h.interface_curvature(), n * 4}; // nullptr before the first interfacial tension: zeros
    case BLUB_TAP_INTERFACE_FIELD: return {h.interface_field(), n * 8};         // likewise
    default: return {nullptr, 0};
    }
}
} // namespace

extern "C" {

const char *blub_last_error(void) { return g_last_error.c_str(); }
const char *blub_version(void) { return "blub-b200 0.1 (sm_90a)"; }

int blub_fluid_create(BlubFluid **out, uint32_t nx, uint32_t ny, uint32_t nz, uint32_t max_num_particles, int device, void *cuda_stream) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "out is NULL");
    *out = nullptr;
    return guarded([&] {
        std::unique_ptr<BlubFluid> f(new BlubFluid());
        f->impl.reset(new blub::HybridFluid(nx, ny, nz, max_num_particles, device, static_cast<cudaStream_t>(cuda_stream)));
        *out = f.release();
        return BLUB_OK;
    });
}

void blub_fluid_destroy(BlubFluid *fluid) { delete fluid; }

int blub_fluid_create_slab(BlubFluid **out, uint32_t nx, uint32_t ny, uint32_t nz_owned, uint32_t max_num_particles, int device, void *cuda_stream,
                           int rank, int world) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "out is NULL");
    *out = nullptr;
    return guarded([&] {
        std::unique_ptr<BlubFluid> f(new BlubFluid());
        f->impl.reset(new blub::HybridFluid(nx, ny, nz_owned, max_num_particles, device, static_cast<cudaStream_t>(cuda_stream), rank, world));
        *out = f.release();
        return BLUB_OK;
    });
}

int blub_fluid_slab_window(BlubFluid *fluid, void **window, size_t *bytes) {
    if (!fluid || !window || !bytes) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *window = fluid->impl->slab_window();
    *bytes = fluid->impl->slab_window_bytes();
    return *window ? BLUB_OK : fail(BLUB_ERR_INVALID_ARGUMENT, "not a slab rank");
}

int blub_fluid_attach_slab_peers(BlubFluid *fluid, void *const *windows, int world) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->attach_slab_peers(windows, world); return BLUB_OK; });
}

int blub_solid_voxelize(void *rgba16f, const uint32_t dim[3], const BlubRigidObject *object, float scale, const float fluid_world_position[3],
                        double total_time, double delta, int clear_first, void *cuda_stream, BlubRigidState *state_out) {
    if (!rgba16f || !dim || !object || !fluid_world_position) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (!(scale > 0.0f) || !(delta > 0.0)) return fail(BLUB_ERR_INVALID_ARGUMENT, "scale and delta must be positive");
    return guarded([&] {
        blub::voxelize_rigid_solid(rgba16f, dim, *object, scale, fluid_world_position, total_time, delta, clear_first, static_cast<cudaStream_t>(cuda_stream), state_out);
        return BLUB_OK;
    });
}

uint64_t blub_simulation_delta_ns(uint64_t steps_per_second) { return steps_per_second ? 1000ull * 1000ull * 1000ull / steps_per_second : 0; }

float blub_duration_as_secs_f32(uint64_t ns) { // core::time::Duration::as_secs_f32
    return (float)(ns / 1000000000ull) + (float)(uint32_t)(ns % 1000000000ull) / 1000000000.0f;
}

uint32_t blub_timer_steps_in_frame(uint64_t *total_rendered_ns, uint64_t *total_simulated_ns, uint64_t frame_delta_ns, uint64_t simulation_delta_ns) {
    if (!total_rendered_ns || !total_simulated_ns || simulation_delta_ns == 0) return 0;
    *total_rendered_ns += frame_delta_ns; // force_frame_delta on a fresh frame, timer.rs:70-74
    uint32_t steps = 0;
    // simulation_frame_loop, timer.rs:94-126: "simulation time shouldn't advance faster than render time"
    while (*total_rendered_ns >= *total_simulated_ns && *total_rendered_ns - *total_simulated_ns >= simulation_delta_ns) {
        *total_simulated_ns += simulation_delta_ns;
        ++steps;
    }
    return steps;
}

void *blub_fluid_stream(const BlubFluid *fluid) { return fluid ? static_cast<void *>(fluid->impl->stream()) : nullptr; }

int blub_device_malloc(void **out, size_t bytes, int device) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = nullptr;
    return guarded([&] {
        BLUB_CUDA_CHECK(cudaSetDevice(device));
        BLUB_CUDA_CHECK(cudaMalloc(out, bytes ? bytes : 1));
        BLUB_CUDA_CHECK(cudaMemset(*out, 0, bytes ? bytes : 1));
        return BLUB_OK;
    });
}

int blub_device_free(void *device_ptr) {
    return guarded([&] {
        BLUB_CUDA_CHECK(cudaFree(device_ptr));
        return BLUB_OK;
    });
}

int blub_mesh_create(BlubMesh **out, const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, int device) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = nullptr;
    return guarded([&] {
        *out = blub::mesh_create(positions, num_vertices, indices, num_indices, device);
        return BLUB_OK;
    });
}

int blub_mesh_load_obj(BlubMesh **out, const char *obj_path, int device) {
    if (!out || !obj_path) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = nullptr;
    return guarded([&] {
        std::vector<float> positions;
        std::vector<uint32_t> indices;
        blub::read_obj(obj_path, positions, indices);
        *out = blub::mesh_create(positions.data(), (uint32_t)(positions.size() / 3), indices.data(), (uint32_t)indices.size(), device);
        return BLUB_OK;
    });
}

void blub_mesh_destroy(BlubMesh *mesh) { blub::mesh_destroy(mesh); }

int blub_mesh_info(const BlubMesh *mesh, uint32_t *num_vertices, uint32_t *num_triangles) {
    if (!mesh || !num_vertices || !num_triangles) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    blub::mesh_info(*mesh, *num_vertices, *num_triangles);
    return BLUB_OK;
}

int blub_obj_read(const char *obj_path, float *positions, uint32_t capacity_vertices, uint32_t *indices, uint32_t capacity_indices, uint32_t counts_out[2]) {
    if (!obj_path || !counts_out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        std::vector<float> p;
        std::vector<uint32_t> idx;
        blub::read_obj(obj_path, p, idx);
        counts_out[0] = (uint32_t)(p.size() / 3);
        counts_out[1] = (uint32_t)idx.size();
        if (positions) std::memcpy(positions, p.data(), sizeof(float) * 3 * std::min<size_t>(capacity_vertices, p.size() / 3));
        if (indices) std::memcpy(indices, idx.data(), sizeof(uint32_t) * std::min<size_t>(capacity_indices, idx.size()));
        return BLUB_OK;
    });
}

int blub_solid_voxelize_mesh(void *rgba16f, const uint32_t dim[3], BlubMesh *mesh, const BlubRigidObject *placement, float scale,
                             const float fluid_world_position[3], double total_time, double delta, int clear_first, void *cuda_stream,
                             BlubRigidState *state_out) {
    if (!rgba16f || !dim || !mesh || !placement || !fluid_world_position) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (!(scale > 0.0f) || !(delta > 0.0)) return fail(BLUB_ERR_INVALID_ARGUMENT, "scale and delta must be positive");
    if (dim[0] == 0 || dim[1] == 0 || dim[2] == 0 || (uint64_t)dim[0] * dim[1] * dim[2] >= (1ull << 31)) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad grid dimension");
    return guarded([&] {
        blub::voxelize_mesh(rgba16f, dim, *mesh, *placement, scale, fluid_world_position, total_time, delta, clear_first, static_cast<cudaStream_t>(cuda_stream), state_out);
        return BLUB_OK;
    });
}

int blub_scene_static_object(const char *path, uint32_t index, BlubRigidObject *placement_out, char *model_path_out, size_t capacity) {
    if (!path || !placement_out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        blub::SceneConfig c = blub::parse_scene_file(path);
        if (index >= c.static_objects.size()) throw std::invalid_argument("static object index out of range");
        *placement_out = c.static_objects[index].placement;
        if (model_path_out && capacity) {
            std::strncpy(model_path_out, c.static_objects[index].model.c_str(), capacity - 1);
            model_path_out[capacity - 1] = 0;
        }
        return BLUB_OK;
    });
}

int blub_fluid_slab_error(BlubFluid *fluid) {
    if (!fluid) return -1;
    int e = -1;
    guarded([&] { e = fluid->impl->slab_error(); return BLUB_OK; });
    return e;
}

int blub_ipc_export(const void *device_ptr, unsigned char handle[64]) {
    if (!device_ptr || !handle) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t size");
        cudaIpcMemHandle_t h;
        BLUB_CUDA_CHECK(cudaIpcGetMemHandle(&h, const_cast<void *>(device_ptr)));
        std::memcpy(handle, &h, 64);
        return BLUB_OK;
    });
}

int blub_ipc_open(const unsigned char handle[64], int device, void **out) {
    if (!handle || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        cudaIpcMemHandle_t h;
        std::memcpy(&h, handle, 64);
        BLUB_CUDA_CHECK(cudaSetDevice(device));
        BLUB_CUDA_CHECK(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
        return BLUB_OK;
    });
}

int blub_ipc_close(void *mapped) {
    if (!mapped) return BLUB_OK;
    return guarded([&] { BLUB_CUDA_CHECK(cudaIpcCloseMemHandle(mapped)); return BLUB_OK; });
}

int blub_enable_peer_access(int device, int peer) {
    return guarded([&] {
        int can = 0;
        BLUB_CUDA_CHECK(cudaDeviceCanAccessPeer(&can, device, peer));
        if (!can) return fail(BLUB_ERR_CUDA, "devices cannot access each other's memory");
        BLUB_CUDA_CHECK(cudaSetDevice(device));
        cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) BLUB_CUDA_CHECK(e);
        cudaGetLastError();
        return BLUB_OK;
    });
}

int blub_fluid_add_cube_tagged(BlubFluid *fluid, const float min_grid[3], const float max_grid[3], uint32_t tag) {
    if (!fluid || !min_grid || !max_grid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { return fluid->impl->add_fluid_cube(min_grid, max_grid, tag) ? BLUB_WARN_TRUNCATED : BLUB_OK; });
}

int blub_fluid_add_cube(BlubFluid *fluid, const float min_grid[3], const float max_grid[3]) { return blub_fluid_add_cube_tagged(fluid, min_grid, max_grid, 0); }

int blub_fluid_set_gravity_grid(BlubFluid *fluid, const float g[3]) {
    if (!fluid || !g) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    fluid->impl->set_gravity_grid(g);
    return BLUB_OK;
}

uint32_t blub_fluid_num_particles(const BlubFluid *fluid) { return fluid ? fluid->impl->num_particles() : 0; }

void blub_fluid_grid_dimension(const BlubFluid *fluid, uint32_t out[3]) {
    if (!fluid || !out) return;
    const blub::GridDim &g = fluid->impl->grid_dimension();
    out[0] = (uint32_t)g.nx; out[1] = (uint32_t)g.ny; out[2] = (uint32_t)g.nz;
}

BlubSolverConfig *blub_fluid_solver_config(BlubFluid *fluid, int which) {
    if (!fluid || which < 0 || which > 1) return nullptr;
    blub::SolverConfig &c = which == 0 ? fluid->impl->pressure_solver_config_velocity() : fluid->impl->pressure_solver_config_density();
    return reinterpret_cast<BlubSolverConfig *>(&c);
}

uint32_t *blub_fluid_rebinning_frequency(BlubFluid *fluid) {
    return fluid ? &fluid->impl->dynamic_settings().particle_rebinning_step_frequency : nullptr;
}

size_t blub_fluid_solver_stats(const BlubFluid *fluid, int which, BlubSolverSample *out, size_t cap) {
    if (!fluid || which < 0 || which > 1) return 0;
    const auto &st = which == 0 ? fluid->impl->pressure_solver_stats_velocity() : fluid->impl->pressure_solver_stats_density();
    if (!out) return st.size();
    const size_t n = st.size() < cap ? st.size() : cap;
    const size_t first = st.size() - n; // newest n, oldest first
    for (size_t k = 0; k < n; ++k) {
        out[k].error = st[first + k].error;
        out[k].iteration_count = st[first + k].iteration_count;
    }
    return n;
}

void blub_fluid_update_statistics(BlubFluid *fluid) {
    if (!fluid) return;
    guarded([&] { fluid->impl->update_statistics(); return BLUB_OK; });
}

int blub_fluid_set_solid_voxels(BlubFluid *fluid, const void *rgba16f_device_ptr) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    fluid->impl->set_solid_voxels(rgba16f_device_ptr);
    return BLUB_OK;
}

int blub_fluid_step(BlubFluid *fluid, double dt) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->step(dt); return BLUB_OK; });
}

int blub_fluid_view(const BlubFluid *fluid, BlubFluidView *out) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    blub::HybridFluid &h = *fluid->impl;
    out->particles_position_ll = h.particles_position();
    out->particles_velocity_x = h.particles_row(0);
    out->particles_velocity_y = h.particles_row(1);
    out->particles_velocity_z = h.particles_row(2);
    out->grid_velocity_x = h.grid_velocity(0);
    out->grid_velocity_y = h.grid_velocity(1);
    out->grid_velocity_z = h.grid_velocity(2);
    out->marker = h.marker();
    out->pressure_from_velocity = h.field(0).pressure();
    out->pressure_from_density = h.field(1).pressure();
    return BLUB_OK;
}

int blub_fluid_set_quirks(BlubFluid *fluid, const BlubQuirks *q) {
    if (!fluid || !q) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (q->precond_mode < 0 || q->precond_mode > 1) return fail(BLUB_ERR_INVALID_ARGUMENT, "precond_mode must be 0 or 1");
    if (q->precond_mode != 0 && fluid->impl->has_tag_densities())
        return fail(BLUB_ERR_INVALID_ARGUMENT, "precond_mode 1 is not supported with a tag density table");
    fluid->impl->quirks.precond_mode = q->precond_mode;
    return BLUB_OK;
}

int blub_fluid_synchronize(BlubFluid *fluid) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->synchronize(); return BLUB_OK; });
}

int blub_fluid_save_state(BlubFluid *fluid, const char *path) {
    if (!fluid || !path) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->save_state(path); return BLUB_OK; });
}

int blub_fluid_load_state(BlubFluid **out, const char *path, int device, void *cuda_stream) {
    if (!out || !path) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = nullptr;
    return guarded([&] {
        std::unique_ptr<BlubFluid> f(new BlubFluid());
        f->impl = blub::HybridFluid::load_state(path, device, static_cast<cudaStream_t>(cuda_stream));
        *out = f.release();
        return BLUB_OK;
    });
}

int blub_state_info(const char *path, BlubStateInfo *out) {
    if (!path || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::StateInfo s = blub::read_state_info(path);
        for (int k = 0; k < 3; ++k) out->grid_dimension[k] = s.grid_dimension[k];
        out->max_num_particles = s.max_num_particles;
        out->num_particles = s.num_particles;
        out->step_count = s.step_count;
        out->format_version = s.format_version;
        return BLUB_OK;
    });
}

uint32_t blub_fluid_step_count(const BlubFluid *fluid) { return fluid ? fluid->impl->step_count() : 0; }

int blub_fluid_set_flow_tagged(BlubFluid *fluid, const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources,
                               const BlubFluidDrain *drains, uint32_t num_drains) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_flow(sources, source_tags, num_sources, drains, num_drains); return BLUB_OK; });
}

int blub_fluid_set_flow(BlubFluid *fluid, const BlubFluidSource *sources, uint32_t num_sources, const BlubFluidDrain *drains, uint32_t num_drains) {
    return blub_fluid_set_flow_tagged(fluid, sources, nullptr, num_sources, drains, num_drains);
}

int blub_fluid_paint_tags(BlubFluid *fluid, const float min_grid[3], const float max_grid[3], uint32_t tag) {
    if (!fluid || !min_grid || !max_grid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->paint_tags(min_grid, max_grid, tag); return BLUB_OK; });
}

int blub_fluid_tag_census(BlubFluid *fluid, uint32_t first_tag, uint32_t num_tags, BlubTagCensus *out) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->tag_census(first_tag, num_tags, out); return BLUB_OK; });
}

int blub_fluid_set_load_probes(BlubFluid *fluid, const BlubLoadProbe *probes, uint32_t num_probes) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_load_probes(probes, num_probes); return BLUB_OK; });
}

int blub_fluid_load_history(BlubFluid *fluid, uint32_t probe, BlubSolidLoad *out, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *count = 0;
    return guarded([&] { *count = fluid->impl->load_history(probe, out, capacity); return BLUB_OK; });
}

int blub_load_probe_cells(const uint32_t dim[3], const BlubLoadProbe *probe, uint32_t lo[3], uint32_t hi[3]) {
    if (!dim || !probe || !lo || !hi) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::LoadProbeBox b = blub::clamp_load_probe(dim, *probe);
        for (int k = 0; k < 3; ++k) {
            lo[k] = (uint32_t)b.lo[k];
            hi[k] = (uint32_t)b.hi[k];
        }
        return BLUB_OK;
    });
}

int blub_fluid_set_bodies(BlubFluid *fluid, const BlubBody *bodies, uint32_t num_bodies) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_bodies(bodies, num_bodies); return BLUB_OK; });
}

int blub_fluid_body_history(BlubFluid *fluid, uint32_t body, BlubBodyRecord *out, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *count = 0;
    return guarded([&] { *count = fluid->impl->body_history(body, out, capacity); return BLUB_OK; });
}

int blub_fluid_bodies(BlubFluid *fluid, BlubBody *out, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *count = 0;
    return guarded([&] { *count = fluid->impl->bodies(out, capacity); return BLUB_OK; });
}

int blub_mesh_body_properties(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale,
                              BlubMeshBodyProperties *out) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL output");
    return guarded([&] { *out = blub::mesh_body_properties(positions, num_vertices, indices, num_indices, scale, nullptr); return BLUB_OK; });
}

int blub_mesh_body_vertices(const float *positions, uint32_t num_vertices, const uint32_t *indices, uint32_t num_indices, float scale, float *out) {
    if (!out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL output");
    return guarded([&] {
        std::vector<float> vb;
        blub::mesh_body_properties(positions, num_vertices, indices, num_indices, scale, &vb);
        std::copy(vb.begin(), vb.end(), out);
        return BLUB_OK;
    });
}

int blub_fluid_set_bodies_meshes(BlubFluid *fluid, const BlubBody *bodies, const BlubMeshBodyShape *shapes, uint32_t num_bodies) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    if (!shapes) return blub_fluid_set_bodies(fluid, bodies, num_bodies);
    if (num_bodies > BLUB_BODIES_MAX) return fail(BLUB_ERR_INVALID_ARGUMENT, "set_bodies: at most 16 bodies");
    const BlubMesh *meshes[BLUB_BODIES_MAX];
    float scales[BLUB_BODIES_MAX];
    for (uint32_t i = 0; i < num_bodies; ++i) meshes[i] = shapes[i].mesh, scales[i] = shapes[i].scale;
    return guarded([&] { fluid->impl->set_bodies_meshes(bodies, meshes, scales, num_bodies); return BLUB_OK; });
}

int blub_fluid_body_mass_properties(BlubFluid *fluid, uint32_t body, BlubMeshBodyProperties *out) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *out = fluid->impl->body_mass_properties(body); return BLUB_OK; });
}

int blub_fluid_set_viscosity(BlubFluid *fluid, const BlubViscosity *viscosity) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_viscosity(viscosity); return BLUB_OK; });
}

int blub_fluid_viscosity(const BlubFluid *fluid, BlubViscosity *out) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = fluid->impl->viscosity();
    return BLUB_OK;
}

int blub_fluid_last_viscosity_solve(BlubFluid *fluid, int32_t *iterations, float max_error[3]) {
    if (!fluid || !iterations || !max_error) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->last_viscosity_solve(iterations, max_error); return BLUB_OK; });
}

int blub_scene_viscosity(const char *path, float *cells2_per_s) {
    if (!path || !cells2_per_s) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *cells2_per_s = blub::scene_viscosity_grid(blub::parse_scene_file(path)); return BLUB_OK; });
}

int blub_fluid_max_particle_velocity(BlubFluid *fluid, float out[3]) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->max_particle_velocity(out); return BLUB_OK; });
}

int blub_fluid_set_surface_tension(BlubFluid *fluid, float cells3_per_s2) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_surface_tension(cells3_per_s2); return BLUB_OK; });
}

int blub_fluid_surface_tension(const BlubFluid *fluid, float *cells3_per_s2) {
    if (!fluid || !cells3_per_s2) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *cells3_per_s2 = fluid->impl->surface_tension();
    return BLUB_OK;
}

int blub_scene_surface_tension(const char *path, float *cells3_per_s2) {
    if (!path || !cells3_per_s2) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *cells3_per_s2 = blub::scene_surface_tension_grid(blub::parse_scene_file(path)); return BLUB_OK; });
}

int blub_fluid_set_interfacial_tension(BlubFluid *fluid, const uint32_t *tags, uint32_t count, float cells3_per_s2) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_interfacial_tension(tags, count, cells3_per_s2); return BLUB_OK; });
}

int blub_fluid_interfacial_tension(const BlubFluid *fluid, uint32_t *tags, uint32_t capacity, uint32_t *count, float *cells3_per_s2) {
    if (!fluid || !count || !cells3_per_s2 || (capacity && !tags)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    const std::vector<uint32_t> &t = fluid->impl->interface_tags();
    for (uint32_t k = 0; k < capacity && k < t.size(); ++k) tags[k] = t[k];
    *count = (uint32_t)t.size();
    *cells3_per_s2 = fluid->impl->interfacial_tension();
    return BLUB_OK;
}

int blub_scene_interfacial_tension(const char *path, uint32_t *tags, uint32_t capacity, uint32_t *count, float *cells3_per_s2) {
    if (!path || !count || !cells3_per_s2 || (capacity && !tags)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig c = blub::parse_scene_file(path);
        for (uint32_t k = 0; k < capacity && k < c.interface_tags.size(); ++k) tags[k] = c.interface_tags[k];
        *count = (uint32_t)c.interface_tags.size();
        *cells3_per_s2 = blub::scene_interfacial_tension_grid(c);
        return BLUB_OK;
    });
}

int blub_fluid_set_whitewater(BlubFluid *fluid, const BlubWhitewater *settings) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_whitewater(settings); return BLUB_OK; });
}

int blub_fluid_whitewater(const BlubFluid *fluid, BlubWhitewater *out) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = fluid->impl->whitewater();
    return BLUB_OK;
}

int blub_fluid_whitewater_counters(BlubFluid *fluid, uint64_t out[4]) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->whitewater_counters(out); return BLUB_OK; });
}

int blub_fluid_download_whitewater(BlubFluid *fluid, float *pos4, float *vel4, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && (!pos4 || !vel4))) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *count = fluid->impl->download_whitewater(pos4, vel4, capacity); return BLUB_OK; });
}

int blub_scene_whitewater(const char *path, BlubWhitewater *out, int32_t *has) {
    if (!path || !out || !has) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig c = blub::parse_scene_file(path);
        *has = c.has_whitewater ? 1 : 0;
        *out = c.whitewater;
        return BLUB_OK;
    });
}

int blub_fluid_set_tag_densities(BlubFluid *fluid, const BlubTagDensity *table, uint32_t count) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_tag_densities(table, count); return BLUB_OK; });
}

int blub_fluid_tag_densities(const BlubFluid *fluid, BlubTagDensity *out, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    const std::vector<BlubTagDensity> &t = fluid->impl->tag_densities();
    for (size_t k = 0; k < t.size() && k < capacity; ++k) out[k] = t[k];
    *count = (uint32_t)t.size();
    return BLUB_OK;
}

int blub_fluid_set_tag_viscosities(BlubFluid *fluid, const BlubTagViscosity *table, uint32_t count) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_tag_viscosities(table, count); return BLUB_OK; });
}

int blub_fluid_tag_viscosities(const BlubFluid *fluid, BlubTagViscosity *out, uint32_t capacity, uint32_t *count) {
    if (!fluid || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    const std::vector<BlubTagViscosity> &t = fluid->impl->tag_viscosities();
    for (size_t k = 0; k < t.size() && k < capacity; ++k) out[k] = t[k];
    *count = (uint32_t)t.size();
    return BLUB_OK;
}

int blub_scene_tag_viscosities(const char *path, BlubTagViscosity *out, uint32_t capacity, uint32_t *count) {
    if (!path || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig c = blub::parse_scene_file(path);
        const std::vector<BlubTagViscosity> t = blub::scene_tag_viscosities_grid(c);
        for (size_t k = 0; k < t.size() && k < capacity; ++k) out[k] = t[k];
        *count = (uint32_t)t.size();
        return BLUB_OK;
    });
}

int blub_scene_tag_densities(const char *path, BlubTagDensity *out, uint32_t capacity, uint32_t *count) {
    if (!path || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig c = blub::parse_scene_file(path);
        for (size_t k = 0; k < c.tag_densities.size() && k < capacity; ++k) out[k] = c.tag_densities[k];
        *count = (uint32_t)c.tag_densities.size();
        return BLUB_OK;
    });
}

int blub_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTimeStepping *config, uint64_t *dt_ns) {
    if (!max_velocity || !gravity_grid || !config || !dt_ns) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *dt_ns = blub::cfl_substep_ns(remaining_ns, max_velocity, gravity_grid, *config); return BLUB_OK; });
}

int blub_fluid_plan_substep(BlubFluid *fluid, uint64_t remaining_ns, const BlubTimeStepping *config, uint64_t *dt_ns, float max_velocity_out[3]) {
    if (!fluid || !config || !dt_ns) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *dt_ns = fluid->impl->plan_substep(remaining_ns, *config, max_velocity_out); return BLUB_OK; });
}

int blub_tank_frame_at(const BlubTankMotion *motion, double t_seconds, BlubTankFrame *out) {
    if (!motion || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *out = blub::tank_frame_at(*motion, t_seconds); return BLUB_OK; });
}

int blub_tank_step_constants(const BlubTankFrame *frame, const float gravity_grid[3], float dt, BlubTankStepConstants *out) {
    if (!frame || !gravity_grid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *out = blub::tank_step_constants(*frame, gravity_grid, dt); return BLUB_OK; });
}

int blub_fluid_set_tank_frame(BlubFluid *fluid, const BlubTankFrame *frame) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->set_tank_frame(frame); return BLUB_OK; });
}

int blub_fluid_tank_frame(const BlubFluid *fluid, BlubTankFrame *out) {
    const BlubTankFrame *f = fluid ? fluid->impl->tank_frame() : nullptr;
    if (f && out) *out = *f;
    return f ? 1 : 0;
}

int blub_tank_cfl_substep_ns(uint64_t remaining_ns, const float max_velocity[3], const float gravity_grid[3], const BlubTankFrame *frame,
                             const uint32_t grid_dimension[3], const BlubTimeStepping *config, uint64_t *dt_ns) {
    if (!max_velocity || !gravity_grid || !grid_dimension || !config || !dt_ns) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { *dt_ns = blub::tank_cfl_substep_ns(remaining_ns, max_velocity, gravity_grid, frame, grid_dimension, *config); return BLUB_OK; });
}

int blub_scene_tank_motion(const char *path, BlubTankMotion *out, int32_t *has_motion) {
    if (!path || !out || !has_motion) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig cfg = blub::parse_scene_file(path);
        *has_motion = cfg.has_tank_motion ? 1 : 0;
        *out = cfg.has_tank_motion ? blub::scene_tank_motion_grid(cfg) : BlubTankMotion{};
        return BLUB_OK;
    });
}

int blub_fluid_has_flow(const BlubFluid *fluid) { return fluid && fluid->impl->has_flow() ? 1 : 0; }

int blub_fluid_flow_counters(BlubFluid *fluid, uint64_t out[3]) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->flow_counters(out); return BLUB_OK; });
}

int blub_scene_info(const char *path, BlubSceneInfo *out) {
    if (!path || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        blub::SceneConfig c = blub::parse_scene_file(path);
        for (int k = 0; k < 3; ++k) {
            out->grid_dimension[k] = c.grid_dimension[k];
            out->world_position[k] = c.world_position[k];
            out->gravity[k] = c.gravity[k];
        }
        out->max_num_particles = c.max_num_particles;
        out->grid_to_world_scale = c.grid_to_world_scale;
        out->num_fluid_cubes = (uint32_t)c.fluid_cubes.size();
        out->num_static_objects = c.num_static_objects;
        return BLUB_OK;
    });
}

int blub_scene_load_probes(const char *path, BlubLoadProbe *out, uint32_t capacity, uint32_t *count) {
    if (!path || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const std::vector<BlubLoadProbe> probes = blub::scene_load_probes_grid(blub::parse_scene_file(path));
        for (size_t k = 0; k < probes.size() && k < capacity; ++k) out[k] = probes[k];
        *count = (uint32_t)probes.size();
        return BLUB_OK;
    });
}

int blub_scene_bodies(const char *path, BlubBody *out, uint32_t capacity, uint32_t *count) {
    if (!path || !count || (capacity && !out)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const std::vector<BlubBody> bodies = blub::scene_bodies_grid(blub::parse_scene_file(path));
        for (size_t k = 0; k < bodies.size() && k < capacity; ++k) out[k] = bodies[k];
        *count = (uint32_t)bodies.size();
        return BLUB_OK;
    });
}

int blub_scene_body_model(const char *path, uint32_t body, char *model_path_out, size_t capacity, float *scale_out) {
    if (!path) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        const blub::SceneConfig c = blub::parse_scene_file(path);
        if (body >= c.bodies.size() || c.bodies[body].shape != 2) throw std::invalid_argument("scene body_model: not a mesh body");
        if (model_path_out && capacity) {
            std::strncpy(model_path_out, c.bodies[body].model.c_str(), capacity - 1);
            model_path_out[capacity - 1] = 0;
        }
        if (scale_out) *scale_out = c.bodies[body].model_scale / c.grid_to_world_scale;
        return BLUB_OK;
    });
}

int blub_scene_load(BlubFluid **out, const char *path, int device, void *cuda_stream) {
    if (!out || !path) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    *out = nullptr;
    return guarded([&] {
        blub::SceneConfig c = blub::parse_scene_file(path);
        std::unique_ptr<BlubFluid> f(new BlubFluid());
        f->impl = blub::create_fluid_from_config(c, device, static_cast<cudaStream_t>(cuda_stream));
        *out = f.release();
        return BLUB_OK;
    });
}

// ---- taps -----------------------------------------------------------------------------------------------------
int blub_fluid_download(BlubFluid *fluid, int tap, void *host_dst, size_t bytes) {
    if (!fluid || !host_dst) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] {
        Tap t = tap_of(fluid, tap);
        if ((tap == BLUB_TAP_CURVATURE || tap == BLUB_TAP_CELL_DENSITY || tap == BLUB_TAP_CELL_VISCOSITY || tap == BLUB_TAP_INTERFACE_CURVATURE ||
             tap == BLUB_TAP_INTERFACE_FIELD) && !t.ptr) {
            if (bytes > (size_t)fluid->impl->grid_dimension().n * (tap == BLUB_TAP_INTERFACE_FIELD ? 8 : 4)) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad tap or size");
            std::memset(host_dst, 0, bytes);
            return BLUB_OK;
        }
        if (!t.ptr || bytes > t.bytes) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad tap or size");
        BLUB_CUDA_CHECK(cudaSetDevice(fluid->impl->device()));
        BLUB_CUDA_CHECK(cudaMemcpyAsync(host_dst, t.ptr, bytes, cudaMemcpyDeviceToHost, fluid->impl->stream()));
        BLUB_CUDA_CHECK(cudaStreamSynchronize(fluid->impl->stream()));
        return BLUB_OK;
    });
}

int blub_fluid_upload(BlubFluid *fluid, int tap, const void *host_src, size_t bytes) {
    if (!fluid || !host_src) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    if (tap == BLUB_TAP_SOLID_VOXELS || tap == BLUB_TAP_CURVATURE || tap == BLUB_TAP_DENSITY || tap == BLUB_TAP_CELL_DENSITY ||
        tap == BLUB_TAP_CELL_VISCOSITY || tap == BLUB_TAP_INTERFACE_CURVATURE || tap == BLUB_TAP_INTERFACE_FIELD)
        return fail(BLUB_ERR_INVALID_ARGUMENT,
                    "the solid volume, curvature, density, cell density, cell viscosity, interface curvature and interface field taps are download only");
    return guarded([&] {
        Tap t = tap_of(fluid, tap);
        if (!t.ptr || bytes > t.bytes) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad tap or size");
        BLUB_CUDA_CHECK(cudaSetDevice(fluid->impl->device()));
        BLUB_CUDA_CHECK(cudaMemcpyAsync(t.ptr, host_src, bytes, cudaMemcpyHostToDevice, fluid->impl->stream()));
        BLUB_CUDA_CHECK(cudaStreamSynchronize(fluid->impl->stream()));
        if (tap == BLUB_TAP_MARKER) fluid->impl->marker_written_externally();
        fluid->impl->grids_written_externally();
        return BLUB_OK;
    });
}

int blub_fluid_set_particles(BlubFluid *fluid, uint32_t count, const float *pos4, const float *vx4, const float *vy4, const float *vz4) {
    if (!fluid || (!pos4 && count)) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL argument");
    return guarded([&] { fluid->impl->set_particles(count, pos4, vx4, vy4, vz4); return BLUB_OK; });
}

int blub_fluid_step_stages(BlubFluid *fluid, double dt, int from, int to) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->step_stages(dt, from, to); return BLUB_OK; });
}

int blub_fluid_solve_only(BlubFluid *fluid, int which, double dt) {
    if (!fluid || which < 0 || which > 1) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] { fluid->impl->solve_only(which, dt); return BLUB_OK; });
}

int blub_fluid_viscosity_only(BlubFluid *fluid, double dt) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] { fluid->impl->viscosity_only(dt); return BLUB_OK; });
}

int blub_fluid_last_solve(BlubFluid *fluid, int which, float *max_error, int32_t *iterations) {
    if (!fluid || which < 0 || which > 1 || !max_error || !iterations) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] {
        BLUB_CUDA_CHECK(cudaSetDevice(fluid->impl->device()));
        int it = 0;
        fluid->impl->field(which).read_last_solve(fluid->impl->stream(), max_error, &it);
        *iterations = it;
        return BLUB_OK;
    });
}

int blub_fluid_last_solve_scalars(BlubFluid *fluid, int which, float out[3]) {
    if (!fluid || which < 0 || which > 1 || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] {
        BLUB_CUDA_CHECK(cudaSetDevice(fluid->impl->device()));
        fluid->impl->field(which).read_last_scalars(fluid->impl->stream(), out);
        return BLUB_OK;
    });
}

int blub_fluid_solver_work(BlubFluid *fluid, uint32_t out[4]) {
    if (!fluid || !out) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] {
        BLUB_CUDA_CHECK(cudaSetDevice(fluid->impl->device()));
        fluid->impl->solver().read_work(fluid->impl->stream(), out);
        return BLUB_OK;
    });
}

int blub_fluid_time_solve(BlubFluid *fluid, int which, double dt, int repetitions, float *ms_each) {
    if (!fluid || which < 0 || which > 1 || repetitions <= 0 || !ms_each) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] {
        blub::HybridFluid &h = *fluid->impl;
        BLUB_CUDA_CHECK(cudaSetDevice(h.device()));
        cudaStream_t st = h.stream();
        const size_t bytes = (size_t)h.grid_dimension().n * sizeof(float);
        float *backup = nullptr;
        BLUB_CUDA_CHECK(cudaMalloc(&backup, bytes));
        cudaEvent_t e0, e1;
        BLUB_CUDA_CHECK(cudaEventCreate(&e0));
        BLUB_CUDA_CHECK(cudaEventCreate(&e1));
        BLUB_CUDA_CHECK(cudaMemcpyAsync(backup, h.solver().residual(), bytes, cudaMemcpyDeviceToDevice, st));
        int rc = BLUB_OK;
        try {
            for (int k = 0; k < repetitions; ++k) {
                BLUB_CUDA_CHECK(cudaMemcpyAsync(h.solver().residual(), backup, bytes, cudaMemcpyDeviceToDevice, st));
                BLUB_CUDA_CHECK(cudaMemsetAsync(h.field(which).pressure(), 0, bytes, st));
                h.grids_written_externally();
                BLUB_CUDA_CHECK(cudaEventRecord(e0, st));
                h.solve_only(which, dt);
                BLUB_CUDA_CHECK(cudaEventRecord(e1, st));
                BLUB_CUDA_CHECK(cudaEventSynchronize(e1));
                BLUB_CUDA_CHECK(cudaEventElapsedTime(&ms_each[k], e0, e1));
            }
        } catch (...) {
            cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(backup);
            throw;
        }
        cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(backup);
        return rc;
    });
}

int blub_fluid_time_steps(BlubFluid *fluid, double dt, int steps, float *ms_total) {
    if (!fluid || steps <= 0 || !ms_total) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] {
        blub::HybridFluid &h = *fluid->impl;
        BLUB_CUDA_CHECK(cudaSetDevice(h.device()));
        cudaEvent_t e0, e1;
        BLUB_CUDA_CHECK(cudaEventCreate(&e0));
        BLUB_CUDA_CHECK(cudaEventCreate(&e1));
        BLUB_CUDA_CHECK(cudaStreamSynchronize(h.stream()));
        BLUB_CUDA_CHECK(cudaEventRecord(e0, h.stream()));
        for (int k = 0; k < steps; ++k) h.step(dt);
        BLUB_CUDA_CHECK(cudaEventRecord(e1, h.stream()));
        BLUB_CUDA_CHECK(cudaEventSynchronize(e1));
        BLUB_CUDA_CHECK(cudaEventElapsedTime(ms_total, e0, e1));
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        return BLUB_OK;
    });
}

int blub_fluid_step_timed(BlubFluid *fluid, double dt, float ms_per_stage[14]) {
    if (!fluid || !ms_per_stage) return fail(BLUB_ERR_INVALID_ARGUMENT, "bad argument");
    return guarded([&] { fluid->impl->step_timed(dt, ms_per_stage); return BLUB_OK; });
}

int blub_fluid_set_solver_path(BlubFluid *fluid, int persistent) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    return guarded([&] {
        fluid->impl->solver().set_path(persistent); // a refused request leaves the solver and the cached step graphs as they were
        fluid->impl->invalidate_graphs();
        return BLUB_OK;
    });
}

int blub_fluid_set_transfer_path(BlubFluid *fluid, int scatter) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    if (scatter != 0 && scatter != 1) return fail(BLUB_ERR_INVALID_ARGUMENT, "transfer path must be 0 (gather) or 1 (scatter)");
    if (fluid->impl->sharded() && scatter == 0) return fail(BLUB_ERR_INVALID_ARGUMENT, "a z-slab rank always uses the scatter form (halo sums of the accumulators)");
    return guarded([&] { fluid->impl->set_transfer_path(scatter); return BLUB_OK; });
}

int blub_fluid_set_graph_replay(BlubFluid *fluid, int enabled) {
    if (!fluid) return fail(BLUB_ERR_INVALID_ARGUMENT, "NULL fluid");
    fluid->impl->use_graph = enabled != 0;
    return BLUB_OK;
}

uint64_t blub_kernel_launch_count(int reset) {
    uint64_t v = blub::g_kernel_launches.load();
    if (reset) blub::g_kernel_launches.store(0);
    return v;
}

} // extern "C"
