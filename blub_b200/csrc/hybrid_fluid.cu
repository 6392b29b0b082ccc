// hybrid_fluid.cu -- host side of the fluid: allocation, particle seeding and the recording of one step.
// Counterpart of src/simulation/hybrid_fluid.rs (HybridFluid::{new, add_fluid_cube, step, ...}).
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <algorithm>

#include <nvtx3/nvToolsExt.h>

#include "blub_core.hpp"
#include "fluid_kernels.hpp"
#include "xoshiro.hpp"

namespace blub {

namespace {
// NVTX ranges with the reference's profiler scope labels (hybrid_fluid.rs:780-973, SURVEY.md Appendix E): a timeline of a run under
// Nsight shows the same tree the reference's "Write Chrometrace" shows.  Header-only NVTX: no cost without a profiler attached.
const char *const kScopeLabels[14] = {
    "transfer particle velocity to grid", "compute divergence", "primary pressure solver (divergence)", "Particle Binning",
    "make velocity grid divergence free", "extrapolate velocity grid", "clear marker & linked list grids",
    "advect particles & write new linked list grid", "density projection: set boundary marker",
    "density projection: compute density error via gather", "secondary pressure solver (density)", "compute position change",
    "extrapolate velocity grid", "correct particle density error"};
struct NvtxScope {
    explicit NvtxScope(const char *name) { nvtxRangePushA(name); }
    ~NvtxScope() { nvtxRangePop(); }
};
// The step numbers of the records in a device ring of `length` slots (slot = step % length), oldest first: the probes' and the bodies' rings.
void note_record(std::deque<uint32_t> &steps, uint32_t step, uint32_t length) {
    if (!steps.empty() && steps.back() == step) return; // the same step again (a repeated step_stages): the same slot
    steps.push_back(step);
    // a slot holds the newest of the steps that map to it
    while (steps.size() > length || (uint64_t)steps.front() + length <= step) steps.pop_front();
}
// Frees what an allocation of the working memory got to (cudaFree(nullptr) is a no-op): the destructor, and a first allocation that failed halfway.
void free_work(ViscosityWork &w) {
    cudaFree(w.codes);
    for (int c = 0; c < 3; ++c) {
        cudaFree(w.r[c]);
        cudaFree(w.s[c]);
    }
    cudaFree(w.word_flags);
    cudaFree(w.words);
    cudaFree(w.scan_sums);
    cudaFree(w.partials);
    cudaFree(w.barrier);
    cudaFree(w.block);
    cudaFree(w.info);
    w = ViscosityWork{};
}
void free_work(TagViscosityWork &w) {
    cudaFree(w.k[0]); // the one allocation of every volume
    cudaFree(w.block);
    w = TagViscosityWork{};
}
void free_work(SurfaceTensionWork &w) {
    cudaFree(w.psi);
    cudaFree(w.kappa);
    cudaFree(w.sigma);
    w = SurfaceTensionWork{};
}
void free_work(InterfacialTensionWork &w) {
    cudaFree(w.phi);
    cudaFree(w.psi);
    cudaFree(w.kappa);
    cudaFree(w.block);
    w = InterfacialTensionWork{};
}
void free_work(WhitewaterWork &w) {
    for (int k = 0; k < 2; ++k) {
        cudaFree(w.pos[k]);
        cudaFree(w.vel[k]);
    }
    cudaFree(w.flags);
    cudaFree(w.cell_counts);
    cudaFree(w.scan_sums);
    cudaFree(w.counters);
    w = WhitewaterWork{};
}
void free_work(TagDensityWork &w) {
    cudaFree(w.sum);
    cudaFree(w.count);
    cudaFree(w.volumes);
    cudaFree(w.block);
    w = TagDensityWork{};
}
} // namespace

HybridFluid::HybridFluid(uint32_t nx, uint32_t ny, uint32_t nz, uint32_t max_num_particles, int device, cudaStream_t stream, int slab_rank,
                         int slab_world)
    : device_(device), stream_(stream), owns_stream_(false), max_num_particles_(max_num_particles), slab_rank_(slab_rank), slab_world_(slab_world) {
    if (slab_world < 1 || slab_world > SLAB_MAX_WORLD || slab_rank < 0 || slab_rank >= slab_world) throw std::invalid_argument("bad slab rank / world");
    const uint32_t owned_nz = nz;
    if (slab_world > 1) nz += 2 * SLAB_HALO; // ghost planes on both sides
    // the reference dispatches 8^3 groups without guards (hybrid_fluid.rs:735-741) and asserts N > 16384 (pressure_solver.rs:551)
    if (nx == 0 || ny == 0 || nz == 0 || nx % 8 || ny % 8 || nz % 8) throw std::invalid_argument("grid dimensions must be positive multiples of 8");
    if ((uint64_t)nx * ny * nz <= 16384) throw std::invalid_argument("grid must have more than 16384 cells");
    if ((uint64_t)nx * ny * nz >= (1ull << 31)) throw std::invalid_argument("grid too large");
    int count = 0;
    BLUB_CUDA_CHECK(cudaGetDeviceCount(&count));
    if (device < 0 || device >= count) throw CudaError("no such CUDA device");
    BLUB_CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop;
    BLUB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) throw CudaError(std::string("libblubcore is built for sm_90a only, found ") + prop.name);
    if (stream_ == nullptr) {
        BLUB_CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
        owns_stream_ = true;
    }
    grid_ = make_grid((int)nx, (int)ny, (int)nz);
    if (slab_world_ > 1) { // only the first / last rank has a z wall; local plane SLAB_HALO is global plane rank * owned_nz
        grid_.z_wall_lo = slab_rank_ == 0 ? SLAB_HALO : -(1 << 20);
        grid_.z_wall_hi = slab_rank_ == slab_world_ - 1 ? SLAB_HALO + (int)owned_nz - 1 : (1 << 20);
        if (slab_rank_ > 0) grid_.z_keep_lo = (float)SLAB_HALO - 0.5f;
        if (slab_rank_ < slab_world_ - 1) grid_.z_keep_hi = (float)(SLAB_HALO + owned_nz) + 0.499f;
    }
    const size_t pbytes = ((size_t)max_num_particles + 64) * sizeof(float4);
    for (int k = 0; k < 2; ++k) {
        BLUB_CUDA_CHECK(cudaMalloc(&pos_[k], pbytes));
        BLUB_CUDA_CHECK(cudaMemset(pos_[k], 0, pbytes));
    }
    for (int c = 0; c < 3; ++c) {
        BLUB_CUDA_CHECK(cudaMalloc(&row_[c], pbytes));
        BLUB_CUDA_CHECK(cudaMemset(row_[c], 0, pbytes));
        u_[c].alloc(grid_);
        // accumulators of the scatter form: allocated by set_transfer_path / always on a z-slab rank
    }
    density_.alloc(grid_);
    marker_.alloc(grid_);
    fluid_bits_.wpr = ((int)nx + 31) / 32;
    BLUB_CUDA_CHECK(cudaMalloc(&fluid_bits_.words, (size_t)fluid_bits_.wpr * ny * nz * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMemset(fluid_bits_.words, 0, (size_t)fluid_bits_.wpr * ny * nz * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMalloc(&particle_words_, (size_t)fluid_bits_.wpr * ny * nz * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMemset(particle_words_, 0, (size_t)fluid_bits_.wpr * ny * nz * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMalloc(&lists_.cell_start, (size_t)(grid_.n + 1 + 8) * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMemset(lists_.cell_start, 0, (size_t)(grid_.n + 1 + 8) * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMalloc(&lists_.order, ((size_t)max_num_particles + 64) * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMalloc(&lists_.arrival, ((size_t)max_num_particles + 64) * sizeof(uint32_t)));
    BLUB_CUDA_CHECK(cudaMalloc(&lists_.cell_slot, ((size_t)max_num_particles + 64) * sizeof(uint2)));
    BLUB_CUDA_CHECK(cudaMalloc(&lists_.block_sums, (size_t)(binning_scan_blocks(grid_) + 1024) * sizeof(uint32_t)));
    {
        const size_t max_crowded = (size_t)max_num_particles / 33 + 1;
        BLUB_CUDA_CHECK(cudaMalloc(&lists_.crowd.count, sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMemset(lists_.crowd.count, 0, sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&lists_.crowd.cells, max_crowded * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&lists_.crowd.slot_of_cell, (size_t)grid_.n * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&lists_.crowd.sums, max_crowded * 18 * sizeof(float2)));
    }
    configure_transfer_kernels();
    if (slab_world_ == 1 && scatter_schedule_enabled()) { // z-slab ranks re-index their particles in every step's migration
        const uint32_t max_warps = max_num_particles / 32 + 1, max_items = scatter_schedule_max_items(grid_, max_warps);
        sched_.nbricks = scatter_schedule_bricks(grid_);
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.valid, sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMemset(sched_.valid, 0, sizeof(uint32_t))); // no schedule before the first re-sort
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.brick_warps, ((size_t)sched_.nbricks + 1) * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.brick_items, ((size_t)sched_.nbricks + 1) * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.item_start, (size_t)max_items * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.item_brick, (size_t)max_items * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.item_box, 2 * (size_t)max_items * sizeof(int4)));
        BLUB_CUDA_CHECK(cudaMalloc(&sched_.warps, (size_t)max_warps * sizeof(uint32_t)));
    }
    {
        // Default: the scatter form, faster than the gather on the 256^3 dam break; both are bit-reproducible.  BLUB_P2G=gather or
        // blub_fluid_set_transfer_path(f, 0) selects the gather.
        const char *tp = std::getenv("BLUB_P2G");
        set_transfer_path(tp && std::string(tp) == "gather" ? 0 : 1);
    }
    SolverConfig cfg; // defaults .1 / 32 / 4, hybrid_fluid.rs:253-257
    if (slab_world_ > 1) {
        // peer-visible window: [mailbox 4 KiB | residual | pressure (velocity) | pressure (density)], one cudaMalloc so that
        // a single IPC handle (or peer pointer) exposes everything a neighbour writes into
        const size_t vol = GridArray<float>::bytes_for(grid_);
        window_bytes_ = 4096 + 3 * vol + slab_extra_window_bytes();
        BLUB_CUDA_CHECK(cudaMalloc(&window_, window_bytes_));
        BLUB_CUDA_CHECK(cudaMemset(window_, 0, window_bytes_));
        char *w = static_cast<char *>(window_);
        solver_.reset(new PressureSolver(grid_, w + 4096));
        field_velocity_.reset(new PressureField(grid_, cfg, w + 4096 + vol));
        field_density_.reset(new PressureField(grid_, cfg, w + 4096 + 2 * vol));
        SlabComm &c = solver_->comm;
        c.rank = slab_rank_;
        c.world = 1; // becomes slab_world_ in attach_slab_peers
        c.halo = SLAB_HALO;
        c.owned_nz = (int)owned_nz;
        BLUB_CUDA_CHECK(cudaMalloc(&c.seq, sizeof(unsigned int)));
        BLUB_CUDA_CHECK(cudaMemset(c.seq, 0, sizeof(unsigned int)));
        for (int k = 0; k < 3; ++k) {
            BLUB_CUDA_CHECK(cudaMalloc(&row_alt_[k], pbytes));
            BLUB_CUDA_CHECK(cudaMemset(row_alt_[k], 0, pbytes));
        }
        BLUB_CUDA_CHECK(cudaMalloc(&mig_counters_, 4 * sizeof(unsigned int)));
        BLUB_CUDA_CHECK(cudaMemset(mig_counters_, 0, 4 * sizeof(unsigned int)));
        // the error flag lives in mapped pinned host memory: the kernels store to it through the device alias, blub_fluid_step polls the host
        // side without blocking (a dead peer must not let the caller go on stepping on halos that never arrived)
        BLUB_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void **>(&slab_error_host_), sizeof(int), cudaHostAllocMapped));
        *slab_error_host_ = 0;
        BLUB_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void **>(&slab_error_), slab_error_host_, 0));
    } else {
        solver_.reset(new PressureSolver(grid_));
        field_velocity_.reset(new PressureField(grid_, cfg));
        field_density_.reset(new PressureField(grid_, cfg));
    }
    BLUB_CUDA_CHECK(cudaMalloc(&params_dev_, sizeof(StepParams)));
    BLUB_CUDA_CHECK(cudaMemset(params_dev_, 0, sizeof(StepParams))); // a device count of 0 until particles arrive
    BLUB_CUDA_CHECK(cudaMallocHost(&params_host_, sizeof(StepParams) * 64));
    for (int k = 0; k < 64; ++k) BLUB_CUDA_CHECK(cudaEventCreateWithFlags(&param_events_[k], cudaEventDisableTiming));
    BLUB_CUDA_CHECK(cudaDeviceSynchronize());
    if (const char *rs = std::getenv("BLUB_RESORT_EVERY")) internal_resort_every_ = (uint32_t)std::atoi(rs);
    const char *ng = std::getenv("BLUB_NO_GRAPH");
    if (ng && ng[0] == '1') use_graph = false;
    // The fused stage 7 pays where its blocks' tile atomics can hide under other blocks' advection traffic: on grids of 2^21 cells and more.
    // On the 128 x 64 x 64 scenes it measured 1.3-1.5 % slower than the separate kernels.  BLUB_DENSITY_FUSE=off / on (a test hook) decides
    // for every grid.
    const char *df = std::getenv("BLUB_DENSITY_FUSE");
    density_fuse_ = df && std::string(df) == "off" ? false : (df && std::string(df) == "on") || grid_.n >= (int64_t(1) << 21);
}

void HybridFluid::destroy_graphs() {
    cudaGraphExec_t *e = &graph_exec_[0][0][0][0];
    for (int k = 0; k < 16; ++k) {
        if (e[k]) cudaGraphExecDestroy(e[k]);
        e[k] = nullptr;
    }
}

HybridFluid::~HybridFluid() {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_);
    destroy_graphs();
    for (int k = 0; k < 2; ++k) cudaFree(pos_[k]);
    for (int c = 0; c < 3; ++c) {
        cudaFree(row_[c]);
        u_[c].release();
        numw_[c].release();
    }
    density_.release();
    marker_.release();
    cudaFree(fluid_bits_.words);
    cudaFree(particle_words_);
    cudaFree(lists_.cell_start);
    cudaFree(lists_.order);
    cudaFree(lists_.arrival);
    cudaFree(lists_.cell_slot);
    cudaFree(lists_.block_sums);
    cudaFree(lists_.crowd.count);
    cudaFree(lists_.crowd.cells);
    cudaFree(lists_.crowd.slot_of_cell);
    cudaFree(lists_.crowd.sums);
    cudaFree(sched_.valid);
    cudaFree(sched_.brick_warps);
    cudaFree(sched_.brick_items);
    cudaFree(sched_.item_start);
    cudaFree(sched_.item_brick);
    cudaFree(sched_.item_box);
    cudaFree(sched_.warps);
    if (solver_ && solver_->comm.seq) cudaFree(solver_->comm.seq);
    solver_.reset();
    field_velocity_.reset();
    field_density_.reset();
    if (window_) cudaFree(window_);
    for (int k = 0; k < 3; ++k) cudaFree(row_alt_[k]);
    cudaFree(flow_scratch_.chunk_drained);
    cudaFree(flow_scratch_.source_count);
    cudaFree(flow_scratch_.emit_offsets);
    cudaFree(flow_scratch_.scan_sums);
    cudaFree(flow_scratch_.scalars);
    cudaFree(flow_scratch_.counters);
    free_work(visc_);
    free_work(tv_);
    free_work(st_);
    free_work(it_);
    free_work(td_);
    free_work(ww_);
    cudaFree(census_dev_);
    cudaFree(max_velocity_dev_);
    cudaFree(load_probes_dev_);
    cudaFree(load_ring_);
    cudaFree(bodies_dev_);
    cudaFree(body_sums_);
    cudaFree(body_ring_);
    cudaFree(composite_);
    free_mesh_bodies();
    cudaFree(mig_counters_);
    if (slab_error_host_) cudaFreeHost(slab_error_host_);
    cudaFree(params_dev_);
    cudaFreeHost(params_host_);
    for (int k = 0; k < 64; ++k) cudaEventDestroy(param_events_[k]);
    if (owns_stream_) cudaStreamDestroy(stream_);
}

// ---------------------------------------------------------------------------------------------------------------
// Particle seeding, hybrid_fluid.rs:609-678.  The jitter stream is cgmath::Vector3<f32> drawn as x, y, z from Xoshiro256pp
// (xoshiro.hpp, shared with the source emission on the device).
static uint32_t clamp_to_grid(uint32_t dim, float v) { // hybrid_fluid.rs:609-617; Rust `as u32` saturates, NaN -> 0
    uint32_t u = !(v > 0.0f) ? 0u : (v >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)v);
    uint32_t m = dim - 1 < u ? dim - 1 : u;
    return m < 1 ? 1 : m;
}

static float tag_bits(uint32_t tag) { // the tag as the raw bits of the fourth position word
    float w;
    std::memcpy(&w, &tag, sizeof(w));
    return w;
}

bool HybridFluid::add_fluid_cube(const float min_grid[3], const float max_grid[3], uint32_t tag) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (flow_active_) num_particles_ = num_particles(); // sources and drains change the count on the device
    // a slab rank takes GLOBAL grid coordinates: the cube is clamped against the global grid and every rank keeps its part
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny,
                             slab_world_ > 1 ? (uint32_t)(solver_->comm.owned_nz * slab_world_) : (uint32_t)grid_.nz};
    uint32_t mn[3], ext[3];
    for (int k = 0; k < 3; ++k) {
        mn[k] = clamp_to_grid(dim[k], min_grid[k]);
        ext[k] = clamp_to_grid(dim[k], max_grid[k]) - mn[k]; // exclusive max corner; wraps like the reference if max < min
    }
    uint32_t num_new = ext[0] * ext[1] * ext[2] * PARTICLES_PER_GRID_CELL;
    bool truncated = false;
    if (max_num_particles_ < num_new + num_particles_) { // :627-633
        num_new = max_num_particles_ - num_particles_;
        truncated = true;
    }
    if (slab_world_ > 1) return add_fluid_cube_slab(mn, ext, tag);
    if (num_new == 0) return truncated;
    Xoshiro256pp rng((uint64_t)(num_particles_ + num_new)); // :637
    std::vector<float4> fresh(num_new);
    for (uint32_t i = 0; i < num_new; ++i) {
        const float cell[3] = {(float)(mn[0] + i / 8u % ext[0]), (float)(mn[1] + i / 8u / ext[0] % ext[1]), (float)(mn[2] + i / 8u / ext[0] / ext[1])};
        const uint32_t s = i % 8u;
        const float strat[3] = {(float)(s % 2u), (float)(s / 2u % 2u), (float)(s / 4u % 2u)};
        float p[3];
        for (int k = 0; k < 3; ++k) {
            const float r = rng.next_f32();
            p[k] = cell[k] + (strat[k] * 0.5f + r * 0.5f); // stratified jitter, :664-665
        }
        fresh[i] = make_float4(p[0], p[1], p[2], tag_bits(tag));
    }
    BLUB_CUDA_CHECK(cudaMemcpyAsync(pos_[cur_] + num_particles_, fresh.data(), (size_t)num_new * sizeof(float4), cudaMemcpyHostToDevice, stream_));
    invalidate_schedule();
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // `fresh` is pageable: finish before it dies (queue.write_buffer semantics)
    num_particles_ += num_new;
    if (flow_active_) set_device_particle_count(num_particles_);
    return truncated;
}

// Slab rank: the same particle stream as the single-GPU seeding (same RNG draws in the same order -- the seed is the GLOBAL
// particle count, hybrid_fluid.rs:637), of which this rank keeps the particles whose cell lies in its planes, re-based to
// local z.  `seeded_global_` mirrors the reference's running num_particles for the seed of the next cube.
bool HybridFluid::add_fluid_cube_slab(const uint32_t mn[3], const uint32_t ext[3], uint32_t tag) {
    const uint32_t num_new = ext[0] * ext[1] * ext[2] * PARTICLES_PER_GRID_CELL;
    if (num_new == 0) return false;
    const int zs = solver_->comm.owned_nz;
    const uint32_t z0 = (uint32_t)(slab_rank_ * zs), z1 = z0 + (uint32_t)zs;
    Xoshiro256pp rng((uint64_t)(seeded_global_ + num_new));
    std::vector<float4> fresh;
    fresh.reserve((size_t)num_new / slab_world_ + 1024);
    for (uint32_t i = 0; i < num_new; ++i) {
        const uint32_t cz = mn[2] + i / 8u / ext[0] / ext[1];
        const float cell[3] = {(float)(mn[0] + i / 8u % ext[0]), (float)(mn[1] + i / 8u / ext[0] % ext[1]), (float)cz};
        const uint32_t s = i % 8u;
        const float strat[3] = {(float)(s % 2u), (float)(s / 2u % 2u), (float)(s / 4u % 2u)};
        float p[3];
        for (int k = 0; k < 3; ++k) {
            const float r = rng.next_f32();
            p[k] = cell[k] + (strat[k] * 0.5f + r * 0.5f);
        }
        if (cz >= z0 && cz < z1) fresh.push_back(make_float4(p[0], p[1], p[2] - (float)z0 + (float)SLAB_HALO, tag_bits(tag)));
    }
    seeded_global_ += num_new;
    bool truncated = false;
    size_t keep = fresh.size();
    if (num_particles_ + keep > max_num_particles_) {
        keep = max_num_particles_ - num_particles_;
        truncated = true;
    }
    if (keep) {
        BLUB_CUDA_CHECK(cudaMemcpyAsync(pos_[cur_] + num_particles_, fresh.data(), keep * sizeof(float4), cudaMemcpyHostToDevice, stream_));
        BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    num_particles_ += (uint32_t)keep;
    set_device_particle_count(num_particles_);
    return truncated;
}

void HybridFluid::invalidate_schedule() {
    if (sched_.valid) BLUB_CUDA_CHECK(cudaMemsetAsync(sched_.valid, 0, sizeof(uint32_t), stream_));
}

void HybridFluid::set_device_particle_count(uint32_t n) {
    BLUB_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<char *>(params_dev_) + offsetof(StepParams, num_particles), &n, sizeof(uint32_t),
                                    cudaMemcpyHostToDevice, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

uint32_t HybridFluid::num_particles() const {
    if (!device_count_mode()) return num_particles_;
    uint32_t n = 0; // authoritative count lives on the device (migration, sources and drains)
    cudaSetDevice(device_);
    cudaMemcpyAsync(&n, reinterpret_cast<const char *>(params_dev_) + offsetof(StepParams, num_particles), sizeof(uint32_t), cudaMemcpyDeviceToHost, stream_);
    cudaStreamSynchronize(stream_);
    return n;
}

int HybridFluid::slab_error() {
    if (!slab_error_host_) return 0;
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    return *static_cast<volatile int *>(slab_error_host_);
}

void HybridFluid::set_particles(uint32_t count, const float *pos4, const float *vx4, const float *vy4, const float *vz4) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (count > max_num_particles_) throw std::invalid_argument("count exceeds max_num_particles");
    const size_t bytes = (size_t)count * sizeof(float4);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(pos_[cur_], pos4, bytes, cudaMemcpyHostToDevice, stream_));
    const float *rows[3] = {vx4, vy4, vz4};
    for (int c = 0; c < 3; ++c) {
        if (rows[c]) BLUB_CUDA_CHECK(cudaMemcpyAsync(row_[c], rows[c], bytes, cudaMemcpyHostToDevice, stream_));
        else BLUB_CUDA_CHECK(cudaMemsetAsync(row_[c], 0, bytes, stream_));
    }
    invalidate_schedule();
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    num_particles_ = count;
    if (device_count_mode()) set_device_particle_count(count);
}

// windows[k] = rank k's slab window as mapped in THIS process (cudaIpcOpenMemHandle, or a plain peer pointer when all
// ranks live in one process); windows[rank] must be this fluid's own window.
void HybridFluid::attach_slab_peers(void *const *windows, int world) {
    if (slab_world_ <= 1 || world != slab_world_ || !windows) throw std::invalid_argument("attach_slab_peers: not a slab rank / wrong world size");
    if (windows[slab_rank_] != window_) throw std::invalid_argument("attach_slab_peers: windows[rank] is not this fluid's window");
    destroy_graphs();
    SlabComm &c = solver_->comm;
    const size_t vol = GridArray<float>::bytes_for(grid_);
    auto cell0 = [&](void *win, int volume) { return reinterpret_cast<float *>(static_cast<char *>(win) + 4096 + (size_t)volume * vol) + grid_.pad; };
    for (int k = 0; k < world; ++k) {
        if (!windows[k]) throw std::invalid_argument("attach_slab_peers: NULL window");
        c.mailbox[k] = static_cast<unsigned long long *>(windows[k]);
    }
    for (int side = 0; side < 2; ++side) {
        const int nb = slab_rank_ + (side == 0 ? -1 : 1);
        const bool has = nb >= 0 && nb < world;
        c.peer_r[side] = has ? cell0(windows[nb], 0) : nullptr;
        c.peer_p[0][side] = has ? cell0(windows[nb], 1) : nullptr;
        c.peer_p[1][side] = has ? cell0(windows[nb], 2) : nullptr;
        slab_peer_window_[side] = has ? windows[nb] : nullptr;
    }
    c.world = world;
}

void HybridFluid::update_statistics() {
    // HybridFluid::update_statistics, :765-768 kicks map_async; retrieval happens at the next solve (:614).  Here both are
    // the same non-blocking poll of the read-back ring.
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    field_density_->retrieve_new_error_samples();
    field_velocity_->retrieve_new_error_samples();
}

void HybridFluid::synchronize() {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// "update uniforms", hybrid_fluid.rs:780-784: one small H2D copy from a pinned ring in front of every step.
void HybridFluid::upload_step_params(float dt) {
    static_assert(sizeof(StepParams) % 4 == 0, "");
    const uint32_t slot = step_param_slot_++ % 64;
    StepParams *h = params_host_ + slot;
    // the copy reads the pinned slot when it EXECUTES: only block if the host is a full ring (64 steps) ahead of the GPU
    BLUB_CUDA_CHECK(cudaEventSynchronize(param_events_[slot]));
    h->dt = dt;
    h->inv_dt = 1.0f / dt;
    // a moving tank's frame: g_eff replaces the gravity of this step only (gravity_ keeps the configured value), Q and K reach tank_frame_kernel
    BlubTankStepConstants tank{};
    if (has_tank_frame_) tank = tank_step_constants(tank_frame_, gravity_, dt);
    for (int c = 0; c < 3; ++c) {
        const float g = has_tank_frame_ ? tank.gravity[c] : gravity_[c];
        h->gravity_dt[c] = g * dt;
        h->gravity[c] = g;
    }
    for (int i = 0; i < 9; ++i) {
        h->tank_q[i] = has_tank_frame_ ? tank.coriolis[i] : (i % 4 == 0 ? 1.0f : 0.0f);
        h->tank_k[i] = tank.force[i];
    }
    for (int c = 0; c < 3; ++c) h->tank_pivot[c] = tank.pivot[c];
    h->tolerance[0] = field_velocity_->config.error_tolerance / dt; // pressure_solver.rs:193-201
    h->tolerance[1] = field_density_->config.error_tolerance / dt;
    h->step_count = step_counter_;
    h->num_particles = num_particles_;
    // sharded or with sources / drains: the particle count changes on the device (migration, flow prologue) and is the last field: leave
    // it alone
    const size_t bytes = device_count_mode() ? offsetof(StepParams, num_particles) : sizeof(StepParams);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(params_dev_, h, bytes, cudaMemcpyHostToDevice, stream_));
    BLUB_CUDA_CHECK(cudaEventRecord(param_events_[slot], stream_));
}

// Particle binning (hybrid_fluid.rs:854-894): every `particle_rebinning_step_frequency`-th step including step 0, 0 = never -- and, because
// a re-sort (positions only, deterministic) costs about what a decayed particle order costs the scatters and the G2P kernels in
// EVERY step, additionally every `internal_resort_every_`-th step (8; BLUB_RESORT_EVERY=0 turns that off).
// Binning only permutes the particle arrays: with it or without it a step computes the same sums in a different order.
bool HybridFluid::binning_step() const {
    const uint32_t rebin = dynamic_settings_.particle_rebinning_step_frequency;
    if (rebin == 0) return false;
    if (step_counter_ % rebin == 0) return true;
    return internal_resort_every_ != 0 && internal_resort_every_ < rebin && step_counter_ % internal_resort_every_ == 0;
}

// The extrapolation works on the FLUID bit mask, which every marker-finishing pass of a step rebuilds.  A marker volume written
// from outside (test taps) makes it stale: rebuild it from the marker volume as it is.
void HybridFluid::refresh_fluid_bits() {
    if (!fluid_bits_stale_) return;
    launch_fluid_bits(stream_, grid_, marker_.ptr, fluid_bits_);
    fluid_bits_stale_ = false;
}

// 1: scatter form of P2G (default; fixed-point integer reductions into accumulator volumes; what the sharded step uses), 0: gather form over
// per-step cell lists.  Both are bit-reproducible run to run; they agree with each other to rounding only.
void HybridFluid::set_transfer_path(int scatter) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if ((scatter || slab_world_ > 1) && !numw_[0].ptr)
        for (int c = 0; c < 3; ++c) numw_[c].alloc(grid_); // zero-filled; the finish pass keeps them zero between steps
    use_scatter_ = scatter != 0 || slab_world_ > 1;
    destroy_graphs();
}

// Stage numbering shared with oracle/blub_oracle.c:orc_step_stages (the order of hybrid_fluid.rs:798-974).
void HybridFluid::run_stage(int stage, float dt) {
    float *u[3] = {u_[0].ptr, u_[1].ptr, u_[2].ptr};
    longlong2 *nw[3] = {numw_[0].ptr, numw_[1].ptr, numw_[2].ptr};
    const FluidBits &bits = fluid_bits_;
    const bool shard = slab_world_ > 1 && solver_->comm.world > 1;
    // sharded or with sources / drains: the device-side count guards the kernels, launches are sized by the capacity
    const uint32_t np = device_count_mode() ? max_num_particles_ : num_particles_;
    const NvtxScope scope(stage >= 0 && stage < 14 ? kScopeLabels[stage] : "stage");
    const uint2 *vox = solid_volume();
    switch (stage) {
    case 0: // transfer particle velocity to grid (:806-833)
        if (num_bodies_ > 0) { // before the flow prologue: sources do not emit into bodies
            const NvtxScope body_scope("floating bodies: composite solid volume");
            if (!mesh_bodies_.empty()) launch_mesh_body_fill(stream_, grid_, (int)num_bodies_, body_cube_, bodies_dev_, mesh_);
            launch_body_composite(stream_, grid_, voxels_, composite_, (int)num_bodies_, body_cube_, bodies_dev_, mesh_.view());
        }
        if (flow_active_) {
            const NvtxScope flow_scope("fluid sources & drains");
            run_flow_prologue();
        }
        if (tank_rotating()) { // after the prologue: emitted particles start with the source velocity in the tank frame, then feel the frame
            const NvtxScope tank_scope("moving tank: frame forces");
            launch_tank_frame(stream_, params_dev_, device_count_mode(), num_particles_, np, pos_[cur_], row_);
        }
        if (!shard && !use_scatter_) {
            // cell lists -> marker (+ FLUID bits) -> one gather per component; deterministic, no accumulator volumes
            launch_cell_lists(stream_, grid_, params_dev_, np, pos_[cur_], 1.0f, lists_);
            launch_marker_from_lists(stream_, grid_, lists_, marker_.ptr, vox, bits, vox ? particle_words_ : nullptr);
            fluid_bits_stale_ = false;
            if (np > 0) launch_p2g_gather(stream_, grid_, params_dev_, lists_, pos_[cur_], row_, marker_.ptr, u);
            else for (int c = 0; c < 3; ++c) BLUB_CUDA_CHECK(cudaMemsetAsync(u[c], 0, (size_t)grid_.n * sizeof(float), stream_));
        } else if (!shard) {
            launch_p2g_scatter(stream_, grid_, params_dev_, np, pos_[cur_], row_, nw, marker_.ptr, false, sched_);
            launch_p2g_finish(stream_, grid_, params_dev_, u, nw, marker_.ptr, vox, bits, particle_words_);
            fluid_bits_stale_ = false;
        } else {
            launch_p2g_scatter(stream_, grid_, params_dev_, np, pos_[cur_], row_, nw, marker_.ptr, true, sched_);
            const SlabHaloItem items[4] = {{nw[0], sizeof(longlong2), 0}, {nw[1], sizeof(longlong2), 0}, {nw[2], sizeof(longlong2), 0}, {marker_.ptr, 1, 1}};
            slab_halo_exchange(items, 4); // X1
            launch_p2g_finish(stream_, grid_, params_dev_, u, nw, marker_.ptr, vox, bits, particle_words_);
            fluid_bits_stale_ = false;
        }
        if (!tag_densities_.empty()) { // the marker P2G finished: the cell densities and the coefficients of stages 2 and 4
            const NvtxScope td_scope("liquids of different densities: cell density");
            launch_tag_density(stream_, grid_, params_dev_, device_count_mode(), num_particles_, np, pos_[cur_], marker_.ptr, td_);
        }
        if (viscosity_on()) run_viscosity();
        break;
    case 1: // compute divergence -> PCG residual (:835-840)
        refresh_fluid_bits();
        launch_divergence_compute(stream_, grid_, bits, marker_.ptr, u, vox, solver_->residual());
        if (surface_tension_ > 0.0f || interfacial_tension_ > 0.0f) {
            const NvtxScope st_scope("surface tension: curvature");
            // The density accumulator is free until stage 7 or 9 clears it.  On the scheduled path the splats rewrite sched_.item_box, the
            // boxes the next P2G reads: harmless, because stage 7 or 9 of this step rewrites them before that P2G.  One splat of every particle
            // serves both tensions: the interface reads it before the free surface overwrites it with its phi.
            launch_density_scatter(stream_, grid_, params_dev_, np, pos_[cur_], density_.ptr, sched_);
            density_zero_ = false;
            if (interfacial_tension_ > 0.0f) {
                launch_phase_scatter(stream_, grid_, params_dev_, np, pos_[cur_], it_.phi, sched_, it_.block);
                launch_interface_psi(stream_, grid_, bits, marker_.ptr, density_.ptr, it_);
            }
            if (surface_tension_ > 0.0f) {
                launch_surface_curvature(stream_, grid_, bits, marker_.ptr, density_.ptr, st_);
                launch_surface_rhs(stream_, grid_, bits, params_dev_, marker_.ptr, st_, solver_->residual());
            }
            if (interfacial_tension_ > 0.0f) {
                const NvtxScope it_scope("interfacial tension: curvature");
                launch_interface_curvature(stream_, grid_, bits, marker_.ptr, it_);
                launch_interface_rhs(stream_, grid_, bits, params_dev_, marker_.ptr, it_, tag_densities_.empty() ? nullptr : td_.beta, solver_->residual());
            }
        }
        break;
    case 2: // primary pressure solver (:843-852)
        solver_->solve(stream_, *field_velocity_, 0, marker_.ptr, params_dev_, quirks, solve_weights());
        if (!capturing_) field_velocity_->enqueue_error_buffer_read(stream_, dt); // the scalars live until this field's next solve
        if (num_load_probes_ > 0) { // the marker and pressure this solve used: stage 6 rewrites the marker
            launch_solid_loads(stream_, grid_, params_dev_, (int)num_load_probes_, load_max_cells_, load_probes_dev_, marker_.ptr, field_velocity_->pressure(),
                               load_ring_);
            if (!capturing_) note_load_record(step_counter_);
        }
        if (num_bodies_ > 0) { // after the probes: the integrator moves the bodies the probes saw
            launch_body_step(stream_, grid_, params_dev_, (int)num_bodies_, body_cube_, bodies_dev_, marker_.ptr, field_velocity_->pressure(), body_sums_,
                             body_ring_, mesh_.view());
            if (!capturing_) note_record(body_steps_, step_counter_, BODY_HISTORY_LENGTH);
        }
        break;
    case 3: // particle binning every n-th step, including step 0 (:854-894)
        if (binning_step()) {
            launch_binning(stream_, grid_, params_dev_, np, pos_[cur_], pos_[1 - cur_], lists_);
            if (np > 0) {
                cur_ = 1 - cur_; // ping-pong instead of the reference's full-buffer copy-back (:884-892)
                if (sched_.valid) launch_scatter_schedule(stream_, grid_, lists_, sched_);
            }
        }
        break;
    case 4: // make velocity grid divergence free (:901-904)
        refresh_fluid_bits();
        launch_divergence_remove(stream_, grid_, bits, marker_.ptr, field_velocity_->pressure(), vox, vox ? particle_words_ : nullptr, u,
                                 tag_densities_.empty() ? nullptr : td_.beta);
        if (surface_tension_ > 0.0f) {
            const NvtxScope st_scope("surface tension: pressure jump");
            launch_surface_faces(stream_, grid_, bits, params_dev_, marker_.ptr, st_, u);
        }
        if (interfacial_tension_ > 0.0f) {
            const NvtxScope it_scope("interfacial tension: pressure jump");
            launch_interface_faces(stream_, grid_, bits, params_dev_, marker_.ptr, it_, tag_densities_.empty() ? nullptr : td_.beta, u);
        }
        break;
    case 5: // extrapolate velocity grid (:906-909)
        refresh_fluid_bits();
        launch_extrapolate(stream_, grid_, bits, u);
        if (shard) {
            const SlabHaloItem items[3] = {{u[0], sizeof(float), 2}, {u[1], sizeof(float), 2}, {u[2], sizeof(float), 2}};
            slab_halo_exchange(items, 3); // X2
        }
        if (whitewater_on()) { // u is projected and extrapolated, the marker is this step's P2G marker: stage 6 clears it
            const NvtxScope ww_scope("whitewater");
            launch_whitewater(stream_, grid_, params_dev_, bits, marker_.ptr, u, vox, whitewater_, ww_);
        }
        break;
    case 6: // clear marker (& linked list) grids (:911-916)
        launch_clear_marker(stream_, grid_, marker_.ptr);
        break;
    case 7: // advect particles (:917-921)
        if (!shard && density_fuse_) { // + the density scatter of stage 9
            if (!density_zero_) BLUB_CUDA_CHECK(cudaMemsetAsync(density_.ptr, 0, (size_t)grid_.n * sizeof(long long), stream_));
            launch_advect_density(stream_, grid_, params_dev_, np, pos_[cur_], row_, u, vox, marker_.ptr, density_.ptr, sched_);
            density_fused_ = true;
            density_zero_ = false;
        } else if (!shard) {
            launch_advect(stream_, grid_, params_dev_, np, pos_[cur_], row_, u, vox, marker_.ptr);
        } else {
            launch_advect_migrate(stream_, grid_, params_dev_, np, pos_[cur_], row_, u, vox, marker_.ptr, slab_migrate_targets());
            slab_migrate_finish();
            const SlabHaloItem items[1] = {{marker_.ptr, 1, 1}};
            slab_halo_exchange(items, 1); // X3
        }
        break;
    case 8: // density projection: set boundary marker (:923-927)
        // the particle words: with a solid volume the cells stage 11 visits around, after a fused stage 7 the cells stage 9 finishes around
        launch_boundary_marker(stream_, grid_, marker_.ptr, vox, bits, vox || density_fused_ ? particle_words_ : nullptr);
        fluid_bits_stale_ = false;
        break;
    case 9: // density projection: compute density error (:928-932)
        if (density_fused_) {
            launch_density_finish_sparse(stream_, grid_, params_dev_, marker_.ptr, bits, particle_words_, density_.ptr, solver_->residual());
            density_fused_ = false;
            density_zero_ = true;
        } else if (!shard) { // the positions may have changed since a fused stage 7 (a step_stages window, an upload): scatter them afresh
            launch_density_rhs(stream_, grid_, params_dev_, np, pos_[cur_], marker_.ptr, density_.ptr, solver_->residual(), sched_);
            density_zero_ = false;
        } else {
            launch_density_scatter(stream_, grid_, params_dev_, np, pos_[cur_], density_.ptr, sched_);
            const SlabHaloItem items[1] = {{density_.ptr, sizeof(long long), 0}};
            slab_halo_exchange(items, 1); // X4
            launch_density_finish(stream_, grid_, params_dev_, marker_.ptr, density_.ptr, solver_->residual());
            density_zero_ = false;
        }
        break;
    case 10: // secondary pressure solver (:940-949)
        solver_->solve(stream_, *field_density_, 1, marker_.ptr, params_dev_, quirks);
        if (!capturing_) field_density_->enqueue_error_buffer_read(stream_, dt);
        break;
    case 11: // compute position change (:959-962)
        refresh_fluid_bits();
        launch_position_change(stream_, grid_, bits, params_dev_, marker_.ptr, field_density_->pressure(), vox ? particle_words_ : nullptr, u);
        break;
    case 12: // extrapolate (:963-966)
        refresh_fluid_bits();
        launch_extrapolate(stream_, grid_, bits, u);
        if (shard) {
            const SlabHaloItem items[3] = {{u[0], sizeof(float), 2}, {u[1], sizeof(float), 2}, {u[2], sizeof(float), 2}};
            slab_halo_exchange(items, 3); // X5
        }
        break;
    case 13: // correct particle density error (:968-972)
        launch_correct_particles(stream_, grid_, params_dev_, np, pos_[cur_], marker_.ptr, u);
        step_counter_ += 1;
        break;
    default: break;
    }
}

// HybridFluid::step, hybrid_fluid.rs:770-977.  The reference re-records ~650 dispatches into a command encoder every
// step; here the 14 stages are captured ONCE into a CUDA graph (per position-buffer parity and binning/non-binning step)
// and replayed with one launch -- dt, gravity*dt and the tolerances reach the kernels through the device StepParams block.
void HybridFluid::step(double simulation_delta_seconds) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const NvtxScope scope("HybridFluid step");
    if (slab_error_host_ && *static_cast<volatile int *>(slab_error_host_) != 0) // non-blocking: whatever the finished steps have reported so far
        throw CudaError("z-slab exchange failed in an earlier step (1 = a peer timed out, 2 = particle capacity exceeded, 3 = migration buffer overflow): code " +
                        std::to_string(*static_cast<volatile int *>(slab_error_host_)));
    const float dt = (float)simulation_delta_seconds; // Duration::as_secs_f32 (SURVEY B14)
    if (!(dt > 0.0f)) throw std::invalid_argument("simulation delta must be positive");
    field_velocity_->retrieve_new_error_samples(); // pressure_solver.rs:614
    field_density_->retrieve_new_error_samples();
    upload_step_params(dt);
    density_fused_ = false;
    if (!use_graph) {
        for (int s = 0; s < 14; ++s) run_stage(s, dt);
        return;
    }
    // a graph is recorded from an all-zero density volume, so that its stage 7 needs no memset when it fuses
    if (density_fuse_ && !density_zero_) {
        BLUB_CUDA_CHECK(cudaMemsetAsync(density_.ptr, 0, (size_t)grid_.n * sizeof(long long), stream_));
        density_zero_ = true;
    }
    GraphSignature sig;
    sig.num_particles = flow_active_ ? 0xFFFFFFFEu : num_particles_; // with sources / drains the launches do not depend on the count
    sig.voxels = voxels_;
    sig.precond_mode = quirks.precond_mode;
    sig.max_it[0] = field_velocity_->config.max_num_iterations; sig.freq[0] = field_velocity_->config.error_check_frequency;
    sig.max_it[1] = field_density_->config.max_num_iterations; sig.freq[1] = field_density_->config.error_check_frequency;
    if (!(sig == graph_signature_)) {
        destroy_graphs();
        graph_signature_ = sig;
    }
    const bool binning = binning_step() && (flow_active_ || num_particles_ > 0);
    // Host-side buffer roles that a captured step bakes in (and changes): the graph is keyed by them.
    struct Roles {
        int cur, row_parity;
        uint32_t exchange_index, step_counter;
        float4 *row[3], *row_alt[3];
        bool density_zero;
    };
    auto save_roles = [&]() {
        Roles r{cur_, row_parity_, slab_exchange_index_, step_counter_, {row_[0], row_[1], row_[2]}, {row_alt_[0], row_alt_[1], row_alt_[2]}, density_zero_};
        return r;
    };
    auto restore_roles = [&](const Roles &r) {
        cur_ = r.cur; row_parity_ = r.row_parity; slab_exchange_index_ = r.exchange_index; step_counter_ = r.step_counter; density_zero_ = r.density_zero;
        for (int k = 0; k < 3; ++k) { row_[k] = r.row[k]; row_alt_[k] = r.row_alt[k]; }
    };
    const Roles before = save_roles();
    const int kb = binning ? 1 : 0, kx = (int)(before.exchange_index & 1u);
    cudaGraphExec_t &exec = graph_exec_[before.cur][kb][before.row_parity][kx];
    uint64_t &nodes_in_graph = graph_kernel_nodes_[before.cur][kb][before.row_parity][kx];
    if (!exec) {
        const uint64_t launches0 = g_kernel_launches.load();
        cudaGraph_t graph = nullptr;
        capturing_ = true;
        BLUB_CUDA_CHECK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
        try {
            for (int s = 0; s < 14; ++s) run_stage(s, dt);
        } catch (...) {
            cudaStreamEndCapture(stream_, &graph);
            if (graph) cudaGraphDestroy(graph);
            capturing_ = false;
            restore_roles(before);
            throw;
        }
        capturing_ = false;
        graph_roles_after_[before.cur][kb][before.row_parity][kx] = {cur_, row_parity_, slab_exchange_index_ - before.exchange_index, density_zero_};
        restore_roles(before); // capture only recorded; the replay below performs the step
        nodes_in_graph = g_kernel_launches.load() - launches0; // recorded, not launched
        g_kernel_launches.fetch_sub(nodes_in_graph);
        BLUB_CUDA_CHECK(cudaStreamEndCapture(stream_, &graph));
        cudaError_t err = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        BLUB_CUDA_CHECK(err);
    }
    BLUB_CUDA_CHECK(cudaGraphLaunch(exec, stream_));
    g_kernel_launches.fetch_add(nodes_in_graph, std::memory_order_relaxed);
    // what the recorded stages did to the buffer roles
    const GraphRolesAfter &after = graph_roles_after_[before.cur][kb][before.row_parity][kx];
    cur_ = after.cur;
    if (after.row_parity != before.row_parity) {
        for (int k = 0; k < 3; ++k) std::swap(row_[k], row_alt_[k]);
        row_parity_ = after.row_parity;
    }
    slab_exchange_index_ = before.exchange_index + after.exchanges;
    density_zero_ = after.density_zero;
    step_counter_ = before.step_counter + 1;
    if (num_load_probes_ > 0) note_load_record(before.step_counter);
    if (num_bodies_ > 0) note_record(body_steps_, before.step_counter, BODY_HISTORY_LENGTH);
    field_velocity_->enqueue_error_buffer_read(stream_, dt);
    field_density_->enqueue_error_buffer_read(stream_, dt);
}

void HybridFluid::step_stages(double simulation_delta_seconds, int from, int to) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    if (!(dt > 0.0f)) throw std::invalid_argument("simulation delta must be positive");
    upload_step_params(dt);
    density_fused_ = false; // what happened to the particles between two calls is unknown
    for (int s = from; s < to && s < 14; ++s) run_stage(s, dt);
    mid_step_ = to < 14;
}

void HybridFluid::step_timed(double simulation_delta_seconds, float ms[14]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    upload_step_params(dt);
    density_fused_ = false;
    cudaEvent_t ev[15];
    for (auto &e : ev) BLUB_CUDA_CHECK(cudaEventCreate(&e));
    BLUB_CUDA_CHECK(cudaEventRecord(ev[0], stream_));
    for (int s = 0; s < 14; ++s) {
        run_stage(s, dt);
        BLUB_CUDA_CHECK(cudaEventRecord(ev[s + 1], stream_));
    }
    BLUB_CUDA_CHECK(cudaEventSynchronize(ev[14]));
    for (int s = 0; s < 14; ++s) BLUB_CUDA_CHECK(cudaEventElapsedTime(&ms[s], ev[s], ev[s + 1]));
    for (auto &e : ev) cudaEventDestroy(e);
}

// ---------------------------------------------------------------------------------------------------------------
// Viscous liquids (viscosity_kernels.cu).  Not in the reference.
void check_viscosity(const BlubViscosity &v) {
    if (!std::isfinite(v.kinematic_viscosity) || v.kinematic_viscosity < 0.0f) throw std::invalid_argument("viscosity: kinematic_viscosity must be finite and not negative");
    if (!std::isfinite(v.error_tolerance) || !(v.error_tolerance > 0.0f)) throw std::invalid_argument("viscosity: error_tolerance must be finite and above 0");
    if (v.max_num_iterations < 1 || v.max_num_iterations > 10000) throw std::invalid_argument("viscosity: max_num_iterations must lie in [1, 10000]");
    if (v.reserved != 0u) throw std::invalid_argument("viscosity: reserved must be 0");
}

bool HybridFluid::viscosity_on() const {
    return viscosity_.kinematic_viscosity > 0.0f || tag_viscosity_scale(tag_viscosities_.data(), (uint32_t)tag_viscosities_.size(), 0.0f) > 0.0f;
}

void HybridFluid::ensure_viscosity_work() {
    if (visc_.block) return;
    ViscosityWork w;
    w.blocks = viscosity_solve_blocks();
    w.pair_blocks = viscosity_solve_blocks(true);
    const size_t n = (size_t)grid_.n, words = (size_t)fluid_bits_.wpr * grid_.ny * grid_.nz;
    try {
        BLUB_CUDA_CHECK(cudaMalloc(&w.codes, n * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMemsetAsync(w.codes, 0, n * sizeof(uint32_t), stream_));
        for (int c = 0; c < 3; ++c) {
            BLUB_CUDA_CHECK(cudaMalloc(&w.r[c], n * sizeof(float)));
            BLUB_CUDA_CHECK(cudaMalloc(&w.s[c], n * sizeof(float)));
        }
        BLUB_CUDA_CHECK(cudaMalloc(&w.word_flags, (words + 1) * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&w.words, words * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&w.scan_sums, ((size_t)exclusive_scan_blocks((int64_t)words + 1) + 1024) * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&w.partials, 2 * 6 * (size_t)std::max(w.blocks, w.pair_blocks) * sizeof(float)));
        BLUB_CUDA_CHECK(cudaMalloc(&w.barrier, 256));
        BLUB_CUDA_CHECK(cudaMalloc(&w.block, sizeof(BlubViscosity)));
        BLUB_CUDA_CHECK(cudaMalloc(&w.info, sizeof(ViscositySolveInfo)));
        BLUB_CUDA_CHECK(cudaMemsetAsync(w.info, 0, sizeof(ViscositySolveInfo), stream_));
    } catch (...) {
        cudaStreamSynchronize(stream_); // the memsets may be in flight
        free_work(w);
        throw;
    }
    visc_ = w;
}

void HybridFluid::set_viscosity(const BlubViscosity *v) {
    if (slab_world_ > 1) throw std::invalid_argument("set_viscosity: z-slab ranks have no viscosity");
    if (mid_step_) throw std::invalid_argument("set_viscosity: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    const BlubViscosity next = v ? *v : kViscosityOff;
    check_viscosity(next);
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const bool was_on = viscosity_on();
    const uint32_t count = (uint32_t)tag_viscosities_.size();
    if (next.kinematic_viscosity > 0.0f || tag_viscosity_scale(tag_viscosities_.data(), count, 0.0f) > 0.0f) ensure_viscosity_work();
    // stream-ordered behind the steps already enqueued (the copies stage the values before they return)
    if (visc_.block) BLUB_CUDA_CHECK(cudaMemcpyAsync(visc_.block, &next, sizeof(next), cudaMemcpyHostToDevice, stream_));
    if (count) { // the fluid's nu is the value of the tags not in the table, and may be nu_scale
        const TagViscosityBlock b = make_tag_viscosity_block(tag_viscosities_.data(), count, next.kinematic_viscosity);
        BLUB_CUDA_CHECK(cudaMemcpyAsync(tv_.block, &b, sizeof(b), cudaMemcpyHostToDevice, stream_));
    }
    viscosity_ = next;
    if (viscosity_on() != was_on) destroy_graphs();
}

// Liquids of different viscosities (viscosity_kernels.cu).  Not in the reference.  The kernels read the table from a device block, so a new
// non-empty table replays the captured graphs; turning the table or the stage on or off changes the launches and drops them.
void HybridFluid::set_tag_viscosities(const BlubTagViscosity *table, uint32_t count) {
    if (slab_world_ > 1) throw std::invalid_argument("set_tag_viscosities: z-slab ranks have no viscosity");
    if (mid_step_) throw std::invalid_argument("set_tag_viscosities: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    check_tag_viscosities(table, count);
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const bool was_on = viscosity_on(), had_table = !tag_viscosities_.empty();
    if (count && !tv_.block) {
        TagViscosityWork w;
        const size_t n = (size_t)grid_.n, bytes = n * (sizeof(unsigned long long) + sizeof(uint32_t) + 13 * sizeof(float));
        try {
            char *mem = nullptr;
            BLUB_CUDA_CHECK(cudaMalloc(&mem, bytes));
            w.k[0] = reinterpret_cast<float4 *>(mem);
            BLUB_CUDA_CHECK(cudaMemsetAsync(mem, 0, bytes, stream_));
            for (int c = 1; c < 3; ++c) w.k[c] = w.k[0] + c * n;
            w.sum = reinterpret_cast<unsigned long long *>(w.k[0] + 3 * n);
            w.count = reinterpret_cast<uint32_t *>(w.sum + n);
            w.nu = reinterpret_cast<float *>(w.count + n);
            BLUB_CUDA_CHECK(cudaMalloc(&w.block, sizeof(TagViscosityBlock)));
        } catch (...) {
            cudaStreamSynchronize(stream_); // the memset may be in flight
            free_work(w);
            throw;
        }
        tv_ = w;
    }
    if (count && tag_viscosity_scale(table, count, viscosity_.kinematic_viscosity) > 0.0f) ensure_viscosity_work();
    if (tv_.block) { // stream-ordered behind the steps already enqueued (the copies stage the values before they return)
        const TagViscosityBlock b = make_tag_viscosity_block(table, count, viscosity_.kinematic_viscosity);
        BLUB_CUDA_CHECK(cudaMemcpyAsync(tv_.block, &b, sizeof(b), cudaMemcpyHostToDevice, stream_));
        if (!count) BLUB_CUDA_CHECK(cudaMemsetAsync(tv_.nu, 0, (size_t)grid_.n * sizeof(float), stream_)); // the tap reads zeros without a table
    }
    // the tolerance and the cap of a setting with nu = 0, for a table that turns the stage on
    if (visc_.block && !was_on) BLUB_CUDA_CHECK(cudaMemcpyAsync(visc_.block, &viscosity_, sizeof(viscosity_), cudaMemcpyHostToDevice, stream_));
    tag_viscosities_.assign(table, table + count);
    if (viscosity_on() != was_on || had_table != !tag_viscosities_.empty()) destroy_graphs();
}

void HybridFluid::run_viscosity() {
    const NvtxScope scope("apply viscosity");
    float *u[3] = {u_[0].ptr, u_[1].ptr, u_[2].ptr};
    if (tag_viscosities_.empty()) launch_viscosity(stream_, grid_, params_dev_, fluid_bits_, marker_.ptr, solid_volume(), u, visc_);
    else
        launch_viscosity(stream_, grid_, params_dev_, fluid_bits_, marker_.ptr, solid_volume(), u, visc_, &tv_, device_count_mode(), num_particles_,
                         device_count_mode() ? max_num_particles_ : num_particles_, pos_[cur_]);
}

void HybridFluid::last_viscosity_solve(int32_t *iterations, float max_error[3]) {
    ViscositySolveInfo info{};
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (visc_.info) BLUB_CUDA_CHECK(cudaMemcpyAsync(&info, visc_.info, sizeof(info), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    *iterations = info.iterations;
    for (int c = 0; c < 3; ++c) max_error[c] = info.max_error[c];
}

void HybridFluid::viscosity_only(double simulation_delta_seconds) {
    if (!viscosity_on()) throw std::invalid_argument("viscosity_only: the fluid has no viscosity");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    if (!(dt > 0.0f)) throw std::invalid_argument("simulation delta must be positive");
    upload_step_params(dt);
    refresh_fluid_bits();
    run_viscosity();
}

void HybridFluid::solve_only(int which, double simulation_delta_seconds) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    upload_step_params(dt);
    solver_->solve(stream_, field(which), which, marker_.ptr, params_dev_, quirks, which == 0 ? solve_weights() : nullptr);
}

// ---------------------------------------------------------------------------------------------------------------
// Sources and drains (flow_kernels.cu).  Not in the reference.
FlowBox clamp_box(const uint32_t dim[3], const float mn[3], const float mx[3], const char *what) {
    FlowBox b;
    for (int k = 0; k < 3; ++k) {
        if (!std::isfinite(mn[k]) || !std::isfinite(mx[k])) throw std::invalid_argument(std::string(what) + " corner is not finite");
        b.lo[k] = (int)clamp_to_grid(dim[k], mn[k]);
        b.hi[k] = (int)clamp_to_grid(dim[k], mx[k]);
        if (b.hi[k] <= b.lo[k]) throw std::invalid_argument(std::string(what) + " box is empty after clamping to the grid");
    }
    return b;
}

FlowSet make_flow_set(const uint32_t dim[3], const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources, const BlubFluidDrain *drains,
                      uint32_t num_drains) {
    if (num_sources > (uint32_t)FLOW_MAX_BOXES || num_drains > (uint32_t)FLOW_MAX_BOXES) throw std::invalid_argument("at most 16 sources and 16 drains");
    if ((num_sources && !sources) || (num_drains && !drains)) throw std::invalid_argument("NULL box array");
    FlowSet fs{};
    auto overlap = [](const FlowBox &a, const FlowBox &b) {
        for (int k = 0; k < 3; ++k)
            if (a.hi[k] <= b.lo[k] || b.hi[k] <= a.lo[k]) return false;
        return true;
    };
    fs.num_sources = (int)num_sources;
    fs.num_drains = (int)num_drains;
    for (uint32_t s = 0; s < num_sources; ++s) {
        fs.source[s] = clamp_box(dim, sources[s].min_grid, sources[s].max_grid, "source");
        fs.tag[s] = source_tags ? source_tags[s] : 0u;
        for (int k = 0; k < 3; ++k) {
            if (!std::isfinite(sources[s].velocity_grid[k])) throw std::invalid_argument("source velocity is not finite");
            fs.velocity[s][k] = sources[s].velocity_grid[k];
        }
        const FlowBox &b = fs.source[s];
        fs.source_base[s + 1] = fs.source_base[s] + (uint32_t)((b.hi[0] - b.lo[0]) * (b.hi[1] - b.lo[1]) * (b.hi[2] - b.lo[2]));
    }
    for (uint32_t s = num_sources; s < (uint32_t)FLOW_MAX_BOXES; ++s) fs.source_base[s + 1] = fs.source_base[s];
    for (uint32_t d = 0; d < num_drains; ++d) fs.drain[d] = clamp_box(dim, drains[d].min_grid, drains[d].max_grid, "drain");
    for (uint32_t s = 0; s < num_sources; ++s) {
        for (uint32_t t = s + 1; t < num_sources; ++t)
            if (overlap(fs.source[s], fs.source[t])) throw std::invalid_argument("two sources overlap");
        for (uint32_t d = 0; d < num_drains; ++d)
            if (overlap(fs.source[s], fs.drain[d])) throw std::invalid_argument("a source overlaps a drain");
    }
    return fs;
}

void HybridFluid::set_flow(const BlubFluidSource *sources, const uint32_t *source_tags, uint32_t num_sources, const BlubFluidDrain *drains,
                           uint32_t num_drains) {
    if (slab_world_ > 1) throw std::invalid_argument("set_flow: z-slab ranks have no sources or drains");
    if (mid_step_) throw std::invalid_argument("set_flow: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    restore_flow(make_flow_set(dim, sources, source_tags, num_sources, drains, num_drains), nullptr);
}

// Applies a validated set; counters != nullptr also sets the cumulative counters (state file load).
void HybridFluid::restore_flow(const FlowSet &fs, const uint64_t counters[3]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    const bool active = fs.num_sources > 0 || fs.num_drains > 0;
    FlowScratch &s = flow_scratch_;
    if (active) {
        if (!s.counters) {
            s.num_chunks = (max_num_particles_ + FLOW_CHUNK - 1) / FLOW_CHUNK;
            BLUB_CUDA_CHECK(cudaMalloc(&s.counters, 3 * sizeof(unsigned long long)));
            BLUB_CUDA_CHECK(cudaMemset(s.counters, 0, 3 * sizeof(unsigned long long)));
            BLUB_CUDA_CHECK(cudaMalloc(&s.scalars, 4 * sizeof(uint32_t)));
            BLUB_CUDA_CHECK(cudaMalloc(&s.chunk_drained, ((size_t)s.num_chunks + 1) * sizeof(uint32_t)));
        }
        const uint32_t cells = fs.source_base[FLOW_MAX_BOXES];
        if (cells > flow_scratch_cells_ || !s.scan_sums) {
            cudaFree(s.source_count);
            cudaFree(s.emit_offsets);
            cudaFree(s.scan_sums);
            s.source_count = s.emit_offsets = s.scan_sums = nullptr;
            const uint32_t room = std::max(cells, flow_scratch_cells_);
            BLUB_CUDA_CHECK(cudaMalloc(&s.source_count, ((size_t)room + 1) * sizeof(uint32_t)));
            BLUB_CUDA_CHECK(cudaMalloc(&s.emit_offsets, ((size_t)room + 1) * sizeof(uint32_t)));
            const int64_t longest = std::max<int64_t>((int64_t)room + 1, (int64_t)s.num_chunks);
            BLUB_CUDA_CHECK(cudaMalloc(&s.scan_sums, ((size_t)exclusive_scan_blocks(longest) + 1024) * sizeof(uint32_t)));
            flow_scratch_cells_ = room;
        }
        s.source_cells = cells;
        if (fs.num_drains && !row_alt_[0]) {
            const size_t pbytes = ((size_t)max_num_particles_ + 64) * sizeof(float4);
            for (int k = 0; k < 3; ++k) {
                BLUB_CUDA_CHECK(cudaMalloc(&row_alt_[k], pbytes));
                BLUB_CUDA_CHECK(cudaMemset(row_alt_[k], 0, pbytes));
            }
        }
    }
    if (counters) {
        if (!s.counters) throw std::invalid_argument("flow counters without a flow set");
        BLUB_CUDA_CHECK(cudaMemcpy(s.counters, counters, 3 * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    }
    if (active && !flow_active_) set_device_particle_count(num_particles_); // from now on the device owns the count
    if (!active && flow_active_) num_particles_ = num_particles();          // read it back once
    flow_ = fs;
    flow_active_ = active;
    destroy_graphs();
}

void HybridFluid::flow_counters(uint64_t out[3]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    out[0] = out[1] = out[2] = 0;
    if (!flow_scratch_.counters) return;
    BLUB_CUDA_CHECK(cudaMemcpyAsync(out, flow_scratch_.counters, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

void HybridFluid::run_flow_prologue() {
    launch_flow_prologue(stream_, grid_, params_dev_, max_num_particles_, flow_, flow_scratch_, pos_[cur_], pos_[1 - cur_], row_, row_alt_, solid_volume(), sched_.valid);
}

// ---------------------------------------------------------------------------------------------------------------
// Particle tags (flow_kernels.cu).  Not in the reference.  In device-count mode the kernels read the count from StepParams (a step or
// set_device_particle_count wrote it); otherwise the host count is passed, since StepParams may not have been uploaded yet.
void HybridFluid::paint_tags(const float min_grid[3], const float max_grid[3], uint32_t tag) {
    if (slab_world_ > 1) throw std::invalid_argument("paint_tags: z-slab ranks cannot paint");
    if (mid_step_) throw std::invalid_argument("paint_tags: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    const FlowBox box = clamp_box(dim, min_grid, max_grid, "paint");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const bool dev = device_count_mode();
    launch_paint_tags(stream_, grid_, dev ? params_dev_ : nullptr, num_particles_, dev ? max_num_particles_ : num_particles_, box, tag, pos_[cur_]);
}

void HybridFluid::tag_census(uint32_t first, uint32_t num_tags, BlubTagCensus *out) {
    if (num_tags == 0 || num_tags > TAG_CENSUS_MAX) throw std::invalid_argument("tag_census: num_tags must be 1 .. 256");
    if ((uint64_t)first + num_tags > (1ull << 32)) throw std::invalid_argument("tag_census: first_tag + num_tags exceeds 2^32");
    if (!out) throw std::invalid_argument("tag_census: NULL output");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (!census_dev_) BLUB_CUDA_CHECK(cudaMalloc(&census_dev_, TAG_CENSUS_MAX * sizeof(BlubTagCensus)));
    for (uint32_t t = 0; t < num_tags; ++t) {
        out[t] = BlubTagCensus{};
        for (int k = 0; k < 3; ++k) {
            out[t].cell_min[k] = INT32_MAX;
            out[t].cell_max[k] = INT32_MIN;
        }
    }
    const size_t bytes = (size_t)num_tags * sizeof(BlubTagCensus);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(census_dev_, out, bytes, cudaMemcpyHostToDevice, stream_));
    const bool dev = device_count_mode();
    launch_tag_census(stream_, grid_, dev ? params_dev_ : nullptr, num_particles_, dev ? max_num_particles_ : num_particles_, first, num_tags, pos_[cur_],
                      row_, census_dev_);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(out, census_dev_, bytes, cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// ---------------------------------------------------------------------------------------------------------------
// CFL-limited substeps (cfl_kernels.cu).  Not in the reference.  The count follows the tags' rule: the device count in device-count mode.
void HybridFluid::max_particle_velocity(float out[3]) {
    if (slab_world_ > 1) throw std::invalid_argument("max_particle_velocity: z-slab ranks cannot plan substeps");
    if (mid_step_) throw std::invalid_argument("max_particle_velocity: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (!max_velocity_dev_) BLUB_CUDA_CHECK(cudaMalloc(&max_velocity_dev_, 3 * sizeof(uint32_t)));
    const bool dev = device_count_mode();
    launch_max_particle_velocity(stream_, dev ? params_dev_ : nullptr, num_particles_, dev ? max_num_particles_ : num_particles_, row_, max_velocity_dev_);
    uint32_t bits[3];
    BLUB_CUDA_CHECK(cudaMemcpyAsync(bits, max_velocity_dev_, sizeof(bits), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    std::memcpy(out, bits, sizeof(bits));
}

uint64_t HybridFluid::plan_substep(uint64_t remaining_ns, const BlubTimeStepping &ts, float max_velocity_out[3]) {
    check_time_stepping(ts);
    if (remaining_ns == 0) throw std::invalid_argument("plan_substep: remaining_ns must be above 0");
    float v[3];
    max_particle_velocity(v);
    if (max_velocity_out) std::memcpy(max_velocity_out, v, sizeof(v));
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    // the larger of the two tensions: conservative for the interface, whose densities (at least 1/2 each) sum to at least 1
    const float s = std::max(surface_tension_, interfacial_tension_);
    if (!(s > 0.0f)) return tank_cfl_substep_ns(remaining_ns, v, gravity_, tank_frame(), dim, ts);
    const uint64_t cap = capillary_limit_ns(s);
    if (cap < ts.min_dt_ns)
        throw UnstableError("plan_substep: the capillary step limit of " + std::to_string(cap) + " ns at a surface tension of " + std::to_string(s) +
                            " cells^3/s^2 is below min_dt_ns = " + std::to_string(ts.min_dt_ns) + " ns");
    BlubTimeStepping capped = ts;
    capped.max_dt_ns = std::min(ts.max_dt_ns, cap);
    return tank_cfl_substep_ns(remaining_ns, v, gravity_, tank_frame(), dim, capped);
}

// ---------------------------------------------------------------------------------------------------------------
// Moving tanks (tank_kernels.cu).  Not in the reference.  The frame is host state only: every upload_step_params turns it into the step's
// constants, so a captured graph follows a new frame without a recapture; only the launch of tank_frame_kernel depends on whether it rotates.
void HybridFluid::set_tank_frame(const BlubTankFrame *frame) {
    if (slab_world_ > 1) throw std::invalid_argument("set_tank_frame: z-slab ranks cannot move their tank");
    if (mid_step_) throw std::invalid_argument("set_tank_frame: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    if (frame) {
        check_tank_frame(*frame);
        if (num_bodies_ > 0 && tank_frame_rotates(*frame))
            throw std::invalid_argument("set_tank_frame: a rotating frame is not supported with floating bodies (translation-only frames are)");
    }
    const bool was_rotating = tank_rotating();
    has_tank_frame_ = frame != nullptr;
    if (frame) tank_frame_ = *frame;
    if (tank_rotating() != was_rotating) destroy_graphs();
}

// ---------------------------------------------------------------------------------------------------------------
// Surface tension (surface_tension_kernels.cu).  Not in the reference.
void HybridFluid::set_surface_tension(float s) {
    if (slab_world_ > 1) throw std::invalid_argument("set_surface_tension: z-slab ranks have no surface tension");
    if (mid_step_) throw std::invalid_argument("set_surface_tension: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    if (!std::isfinite(s) || s < 0.0f) throw std::invalid_argument("set_surface_tension: the surface tension must be finite and not negative");
    if (s > 0.0f && !tag_densities_.empty())
        throw std::invalid_argument("set_surface_tension: not supported with a tag density table (the interfacial tension is not modelled)");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const bool on = s > 0.0f;
    if (on && !st_.sigma) {
        SurfaceTensionWork w;
        const size_t n = (size_t)grid_.n;
        try {
            BLUB_CUDA_CHECK(cudaMalloc(&w.psi, n * sizeof(long long)));
            BLUB_CUDA_CHECK(cudaMalloc(&w.kappa, n * sizeof(float)));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.kappa, 0, n * sizeof(float), stream_));
            BLUB_CUDA_CHECK(cudaMalloc(&w.sigma, sizeof(float)));
        } catch (...) {
            cudaStreamSynchronize(stream_); // the memset may be in flight
            free_work(w);
            throw;
        }
        st_ = w;
    }
    // stream-ordered behind the steps already enqueued (the copy stages the value before it returns)
    if (st_.sigma) BLUB_CUDA_CHECK(cudaMemcpyAsync(st_.sigma, &s, sizeof(s), cudaMemcpyHostToDevice, stream_));
    if (!on && st_.kappa) BLUB_CUDA_CHECK(cudaMemsetAsync(st_.kappa, 0, (size_t)grid_.n * sizeof(float), stream_)); // the tap reads zeros when off
    if (on != (surface_tension_ > 0.0f)) destroy_graphs();
    surface_tension_ = s;
}

// ---------------------------------------------------------------------------------------------------------------
// Interfacial tension (surface_tension_kernels.cu).  Not in the reference.  The kernels read the tension and the tag set from a device block,
// so a change between two settings above zero replays the captured graphs; turning it on or off changes the launches and drops them.
void check_interfacial_tension(const uint32_t *tags, uint32_t count, float s, const char *who) {
    const std::string w = who;
    if (!std::isfinite(s) || s < 0.0f) throw std::invalid_argument(w + ": the interfacial tension must be finite and not negative");
    if (count > (uint32_t)INTERFACE_TAGS_MAX) throw std::invalid_argument(w + ": more than " + std::to_string(INTERFACE_TAGS_MAX) + " tags");
    if (count && !tags) throw std::invalid_argument(w + ": NULL tags with count > 0");
    for (uint32_t a = 0; a < count; ++a)
        for (uint32_t b = 0; b < a; ++b)
            if (tags[a] == tags[b]) throw std::invalid_argument(w + ": tag " + std::to_string(tags[a]) + " is listed twice");
    if (s > 0.0f && !count) throw std::invalid_argument(w + ": an interfacial tension above 0 needs at least one tag");
}

void HybridFluid::set_interfacial_tension(const uint32_t *tags, uint32_t count, float s) {
    if (slab_world_ > 1) throw std::invalid_argument("set_interfacial_tension: z-slab ranks have no interfacial tension");
    if (mid_step_) throw std::invalid_argument("set_interfacial_tension: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    check_interfacial_tension(tags, count, s, "set_interfacial_tension");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const bool on = s > 0.0f;
    if (on && !it_.block) {
        InterfacialTensionWork w;
        const size_t n = (size_t)grid_.n;
        try {
            BLUB_CUDA_CHECK(cudaMalloc(&w.phi, n * sizeof(long long)));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.phi, 0, n * sizeof(long long), stream_));
            BLUB_CUDA_CHECK(cudaMalloc(&w.psi, n * sizeof(long long)));
            BLUB_CUDA_CHECK(cudaMalloc(&w.kappa, n * sizeof(float)));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.kappa, 0, n * sizeof(float), stream_));
            BLUB_CUDA_CHECK(cudaMalloc(&w.block, sizeof(InterfacialTensionBlock)));
        } catch (...) {
            cudaStreamSynchronize(stream_); // the memsets may be in flight
            free_work(w);
            throw;
        }
        it_ = w;
    }
    if (it_.block) { // stream-ordered behind the steps already enqueued (the copy stages the value before it returns)
        InterfacialTensionBlock b{};
        b.s = s;
        b.count = on ? count : 0u;
        for (uint32_t k = 0; k < b.count; ++k) b.tag[k] = tags[k];
        BLUB_CUDA_CHECK(cudaMemcpyAsync(it_.block, &b, sizeof(b), cudaMemcpyHostToDevice, stream_));
        if (!on) { // the taps read zeros when off
            BLUB_CUDA_CHECK(cudaMemsetAsync(it_.kappa, 0, (size_t)grid_.n * sizeof(float), stream_));
            BLUB_CUDA_CHECK(cudaMemsetAsync(it_.phi, 0, (size_t)grid_.n * sizeof(long long), stream_));
        }
    }
    if (on != (interfacial_tension_ > 0.0f)) destroy_graphs();
    interfacial_tension_ = s;
    if (on) interface_tags_.assign(tags, tags + count);
    else interface_tags_.clear();
}

// ---------------------------------------------------------------------------------------------------------------
// Whitewater (whitewater_kernels.cu).  Not in the reference.  The setting reaches the kernels by value, so every change drops the step graphs.
void check_whitewater(const BlubWhitewater &s, const char *who) {
    const std::string w = who;
    if (s.max_num_particles == 0) return;
    if (s.max_num_particles > BLUB_WHITEWATER_MAX_PARTICLES)
        throw std::invalid_argument(w + ": max_num_particles above " + std::to_string(BLUB_WHITEWATER_MAX_PARTICLES));
    const float values[] = {s.trapped_air_rate, s.wave_crest_rate, s.trapped_air_range[0], s.trapped_air_range[1], s.wave_crest_range[0],
                            s.wave_crest_range[1], s.energy_range[0], s.energy_range[1], s.lifetime_lo, s.lifetime_hi, s.buoyancy, s.drag};
    for (float v : values)
        if (!std::isfinite(v)) throw std::invalid_argument(w + ": every value must be finite");
    if (s.trapped_air_rate < 0.0f || s.wave_crest_rate < 0.0f) throw std::invalid_argument(w + ": a rate is negative");
    if (!(s.trapped_air_range[0] < s.trapped_air_range[1])) throw std::invalid_argument(w + ": trapped_air_range needs lo < hi");
    if (!(s.wave_crest_range[0] < s.wave_crest_range[1])) throw std::invalid_argument(w + ": wave_crest_range needs lo < hi");
    if (!(s.energy_range[0] < s.energy_range[1])) throw std::invalid_argument(w + ": energy_range needs lo < hi");
    if (s.lifetime_lo < 0.0f || !(s.lifetime_lo < s.lifetime_hi)) throw std::invalid_argument(w + ": the lifetime needs 0 <= lo < hi");
    if (!(s.drag >= 0.0f && s.drag <= 1.0f)) throw std::invalid_argument(w + ": drag must lie in [0, 1]");
    if (s.spray_below > s.bubble_from) throw std::invalid_argument(w + ": spray_below is above bubble_from");
    if (s.bubble_from > 27u) throw std::invalid_argument(w + ": bubble_from is above 27");
    if (s.max_per_cell > 16u) throw std::invalid_argument(w + ": max_per_cell is above 16");
}

void HybridFluid::set_whitewater(const BlubWhitewater *setting) {
    if (slab_world_ > 1) throw std::invalid_argument("set_whitewater: z-slab ranks have no whitewater");
    if (mid_step_) throw std::invalid_argument("set_whitewater: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    check_whitewater(setting ? *setting : BlubWhitewater{}, "set_whitewater");
    const BlubWhitewater s = setting && setting->max_num_particles ? *setting : BlubWhitewater{}; // off is stored as all zero
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (s.max_num_particles != ww_.capacity) {
        // the new storage first: a failed allocation throws with the fluid, its particles and its graphs as they were
        WhitewaterWork w;
        if (s.max_num_particles) {
            const size_t cap = s.max_num_particles, n = (size_t)grid_.n;
            try {
                for (int k = 0; k < 2; ++k) {
                    BLUB_CUDA_CHECK(cudaMalloc(&w.pos[k], cap * sizeof(float4)));
                    BLUB_CUDA_CHECK(cudaMalloc(&w.vel[k], cap * sizeof(float4)));
                }
                BLUB_CUDA_CHECK(cudaMalloc(&w.flags, (cap + 1) * sizeof(uint32_t)));
                BLUB_CUDA_CHECK(cudaMalloc(&w.cell_counts, (n + 1) * sizeof(uint32_t)));
                const int64_t longest = std::max<int64_t>((int64_t)cap + 1, (int64_t)n + 1);
                BLUB_CUDA_CHECK(cudaMalloc(&w.scan_sums, ((size_t)exclusive_scan_blocks(longest) + 1024) * sizeof(uint32_t)));
                BLUB_CUDA_CHECK(cudaMalloc(&w.counters, sizeof(WhitewaterCounters)));
                BLUB_CUDA_CHECK(cudaMemsetAsync(w.counters, 0, sizeof(WhitewaterCounters), stream_));
            } catch (...) {
                cudaStreamSynchronize(stream_); // the memset may be in flight
                free_work(w);
                throw;
            }
            w.capacity = s.max_num_particles;
        }
        if (ww_.counters) {
            BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // the enqueued steps may still use the old storage
            free_work(ww_);
        }
        ww_ = w;
    }
    whitewater_ = s;
    destroy_graphs();
}

void HybridFluid::whitewater_counters(uint64_t out[4]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    out[0] = out[1] = out[2] = out[3] = 0;
    if (!ww_.counters) return;
    WhitewaterCounters c;
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&c, ww_.counters, sizeof(c), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    out[0] = c.count;
    out[1] = c.emitted;
    out[2] = c.removed;
    out[3] = c.refused;
}

uint32_t HybridFluid::download_whitewater(float *pos4, float *vel4, uint32_t capacity) {
    uint64_t c[4];
    whitewater_counters(c);
    const uint32_t count = (uint32_t)c[0], n = std::min(count, capacity);
    if (n) {
        BLUB_CUDA_CHECK(cudaMemcpyAsync(pos4, ww_.pos[0], (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, stream_));
        BLUB_CUDA_CHECK(cudaMemcpyAsync(vel4, ww_.vel[0], (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, stream_));
        BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    return count;
}

void HybridFluid::restore_whitewater(const BlubWhitewater &s, const uint64_t counters[3], uint32_t count, const float *particles) {
    set_whitewater(&s);
    if (count > ww_.capacity) throw std::invalid_argument("restore_whitewater: more particles than the capacity");
    std::vector<float4> pos(count), vel(count);
    for (uint32_t i = 0; i < count; ++i) {
        std::memcpy(&pos[i], particles + 8ull * i, sizeof(float4));
        std::memcpy(&vel[i], particles + 8ull * i + 4, sizeof(float4));
    }
    WhitewaterCounters c{};
    c.emitted = counters[0];
    c.removed = counters[1];
    c.refused = counters[2];
    c.count = count;
    if (count) {
        BLUB_CUDA_CHECK(cudaMemcpyAsync(ww_.pos[0], pos.data(), (size_t)count * sizeof(float4), cudaMemcpyHostToDevice, stream_));
        BLUB_CUDA_CHECK(cudaMemcpyAsync(ww_.vel[0], vel.data(), (size_t)count * sizeof(float4), cudaMemcpyHostToDevice, stream_));
    }
    BLUB_CUDA_CHECK(cudaMemcpyAsync(ww_.counters, &c, sizeof(c), cudaMemcpyHostToDevice, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // the host copies are pageable
}

// ---------------------------------------------------------------------------------------------------------------
// Liquids of different densities (tag_density_kernels.cu).  Not in the reference.  The kernels read the table from a device block, so a new
// non-empty table replays the captured graphs; turning the feature on or off changes the launches and drops them.
void HybridFluid::set_tag_densities(const BlubTagDensity *table, uint32_t count) {
    if (slab_world_ > 1) throw std::invalid_argument("set_tag_densities: z-slab ranks have one density");
    if (mid_step_) throw std::invalid_argument("set_tag_densities: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    check_tag_densities(table, count);
    if (count && surface_tension_ > 0.0f)
        throw std::invalid_argument("set_tag_densities: not supported with surface tension (the interfacial tension is not modelled)");
    if (count && quirks.precond_mode != 0) throw std::invalid_argument("set_tag_densities: the variable-density solve needs precond_mode 0");
    // the bodies' coupling was measured not to hold with a table (a 0.9 box rose through a 0.8 layer instead of settling on the water below)
    if (count && num_bodies_ > 0) throw std::invalid_argument("set_tag_densities: not supported with floating bodies");
    if (count && !solver_->persistent_available()) throw std::invalid_argument("set_tag_densities: the variable-density solve needs cooperative launch");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    if (count && !td_.block) {
        TagDensityWork w;
        const size_t n = (size_t)grid_.n, vol = GridArray<float>::bytes_for(grid_);
        try {
            BLUB_CUDA_CHECK(cudaMalloc(&w.sum, n * sizeof(unsigned long long)));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.sum, 0, n * sizeof(unsigned long long), stream_));
            BLUB_CUDA_CHECK(cudaMalloc(&w.count, n * sizeof(uint32_t)));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.count, 0, n * sizeof(uint32_t), stream_));
            BLUB_CUDA_CHECK(cudaMalloc(&w.volumes, 6 * vol));
            BLUB_CUDA_CHECK(cudaMemsetAsync(w.volumes, 0, 6 * vol, stream_)); // the padding stays zero
            float *v[6];
            for (int k = 0; k < 6; ++k) v[k] = reinterpret_cast<float *>(static_cast<char *>(w.volumes) + k * vol) + grid_.pad;
            w.rho = v[0];
            for (int c = 0; c < 3; ++c) w.beta[c] = v[1 + c];
            w.diag = v[4];
            w.inv_diag2 = v[5];
            BLUB_CUDA_CHECK(cudaMalloc(&w.block, sizeof(TagDensityBlock)));
        } catch (...) {
            cudaStreamSynchronize(stream_); // the memsets may be in flight
            free_work(w);
            throw;
        }
        td_ = w;
    }
    if (td_.block) { // stream-ordered behind the steps already enqueued (the copy stages the value before it returns)
        const TagDensityBlock b = make_tag_density_block(table, count);
        BLUB_CUDA_CHECK(cudaMemcpyAsync(td_.block, &b, sizeof(b), cudaMemcpyHostToDevice, stream_));
    }
    if (!count && td_.rho) BLUB_CUDA_CHECK(cudaMemsetAsync(td_.rho, 0, (size_t)grid_.n * sizeof(float), stream_)); // the tap reads zeros when off
    if ((count != 0) != !tag_densities_.empty()) destroy_graphs();
    tag_densities_.assign(table, table + count);
}

// ---------------------------------------------------------------------------------------------------------------
// Solid load probes (load_kernels.cu).  Not in the reference.  The records stay on the device; the host only keeps the step numbers it
// recorded, so that a step never synchronises and load_history knows which ring slots hold what.
static int clamp_to_closed_grid(uint32_t dim, float v) { // clamp_to_grid's conversion, clamped to [0, dim]: the border cells are walls
    const uint32_t u = !(v > 0.0f) ? 0u : (v >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)v);
    return (int)(u < dim ? u : dim);
}

LoadProbeBox clamp_load_probe(const uint32_t dim[3], const BlubLoadProbe &probe) {
    LoadProbeBox b;
    for (int k = 0; k < 3; ++k) {
        if (!std::isfinite(probe.min_grid[k]) || !std::isfinite(probe.max_grid[k])) throw std::invalid_argument("load probe corner is not finite");
        if (!std::isfinite(probe.pivot_grid[k])) throw std::invalid_argument("load probe pivot is not finite");
        b.lo[k] = clamp_to_closed_grid(dim[k], probe.min_grid[k]);
        b.hi[k] = clamp_to_closed_grid(dim[k], probe.max_grid[k]);
        if (b.hi[k] <= b.lo[k]) throw std::invalid_argument("load probe box is empty after clamping to the grid");
        b.pivot[k] = probe.pivot_grid[k];
    }
    return b;
}

void HybridFluid::set_load_probes(const BlubLoadProbe *probes, uint32_t num_probes) {
    if (slab_world_ > 1) throw std::invalid_argument("set_load_probes: z-slab ranks have no load probes");
    if (mid_step_) throw std::invalid_argument("set_load_probes: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    if (num_probes > (uint32_t)LOAD_PROBES_MAX) throw std::invalid_argument("set_load_probes: at most 16 probes");
    if (num_probes && !probes) throw std::invalid_argument("set_load_probes: NULL probe array");
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    LoadProbeBox boxes[LOAD_PROBES_MAX];
    uint32_t max_cells = 0;
    for (uint32_t p = 0; p < num_probes; ++p) {
        boxes[p] = clamp_load_probe(dim, probes[p]);
        const LoadProbeBox &b = boxes[p];
        max_cells = std::max(max_cells, (uint32_t)(b.hi[0] - b.lo[0]) * (uint32_t)(b.hi[1] - b.lo[1]) * (uint32_t)(b.hi[2] - b.lo[2]));
    }
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // no step in flight reads the old boxes or writes the ring
    if (num_probes > 0) {
        const size_t ring_bytes = (size_t)LOAD_PROBES_MAX * LOAD_HISTORY_LENGTH * sizeof(BlubSolidLoad);
        if (!load_ring_) {
            BLUB_CUDA_CHECK(cudaMalloc(&load_probes_dev_, LOAD_PROBES_MAX * sizeof(LoadProbeBox)));
            BLUB_CUDA_CHECK(cudaMalloc(&load_ring_, ring_bytes));
        }
        BLUB_CUDA_CHECK(cudaMemcpy(load_probes_dev_, boxes, num_probes * sizeof(LoadProbeBox), cudaMemcpyHostToDevice));
        BLUB_CUDA_CHECK(cudaMemset(load_ring_, 0, ring_bytes));
    }
    num_load_probes_ = num_probes;
    load_max_cells_ = max_cells;
    load_steps_.clear();
    destroy_graphs();
}

void HybridFluid::note_load_record(uint32_t step) { note_record(load_steps_, step, LOAD_HISTORY_LENGTH); }

uint32_t HybridFluid::load_history(uint32_t probe, BlubSolidLoad *out, uint32_t capacity) {
    if (probe >= num_load_probes_) throw std::invalid_argument("load_history: no such load probe");
    if (capacity && !out) throw std::invalid_argument("load_history: NULL output");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    std::vector<BlubSolidLoad> ring(LOAD_HISTORY_LENGTH);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(ring.data(), load_ring_ + (size_t)probe * LOAD_HISTORY_LENGTH, LOAD_HISTORY_LENGTH * sizeof(BlubSolidLoad),
                                    cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    // the recorded steps increase and lie within LOAD_HISTORY_LENGTH of each other: they fill distinct slots
    const uint32_t n = std::min<uint32_t>(capacity, (uint32_t)load_steps_.size());
    const size_t first = load_steps_.size() - n;
    for (uint32_t k = 0; k < n; ++k) out[k] = ring[load_steps_[first + k] % LOAD_HISTORY_LENGTH];
    return n;
}

// ---------------------------------------------------------------------------------------------------------------
// Floating bodies (body_kernels.cu).  Not in the reference.  The poses live on the device and move inside the step; the host keeps only the
// step numbers it recorded, as it does for the probes.
std::vector<BlubBody> make_body_set(const uint32_t dim[3], const BlubBody *bodies, uint32_t num_bodies, bool loaded) {
    if (num_bodies > (uint32_t)BODIES_MAX) throw std::invalid_argument("set_bodies: at most 16 bodies");
    if (num_bodies && !bodies) throw std::invalid_argument("set_bodies: NULL body array");
    std::vector<BlubBody> out(bodies, bodies + num_bodies);
    for (BlubBody &b : out) {
        bool finite = std::isfinite(b.relative_density);
        for (int k = 0; k < 4; ++k) finite = finite && std::isfinite(b.rotation[k]);
        for (int k = 0; k < 3; ++k)
            finite = finite && std::isfinite(b.half_extent[k]) && std::isfinite(b.centre[k]) && std::isfinite(b.velocity[k]) && std::isfinite(b.angular_velocity[k]);
        if (!finite) throw std::invalid_argument("set_bodies: a body value is not finite");
        if (b.shape != 0 && b.shape != 1) throw std::invalid_argument("set_bodies: shape must be 0 (box) or 1 (sphere)");
        for (int k = 0; k < (b.shape == 1 ? 1 : 3); ++k)
            if (!(b.half_extent[k] >= 1.0f)) throw std::invalid_argument("set_bodies: a half extent or radius is below 1 cell");
        if (!(b.relative_density > 0.0f)) throw std::invalid_argument("set_bodies: relative_density must be > 0");
        const float *q = b.rotation;
        const double norm = std::sqrt((double)q[0] * q[0] + (double)q[1] * q[1] + (double)q[2] * q[2] + (double)q[3] * q[3]);
        if (!(std::fabs(norm - 1.0) <= 1e-3)) throw std::invalid_argument("set_bodies: the rotation quaternion is not of unit norm (within 1e-3)");
        if (!loaded)
            for (int k = 0; k < 4; ++k) b.rotation[k] = (float)(q[k] / norm);
        float e[3];
        body_bounding_extents(b, e);
        const float slack = loaded ? 1e-3f : 0.0f;
        for (int k = 0; k < 3 && dim; ++k)
            if (b.centre[k] - e[k] < 1.0f - slack || b.centre[k] + e[k] > (float)dim[k] - 1.0f + slack)
                throw std::invalid_argument("set_bodies: a body's bounding box leaves [1, dim - 1]");
    }
    return out;
}

void HybridFluid::set_bodies(const BlubBody *bodies, uint32_t num_bodies) {
    if (slab_world_ > 1) throw std::invalid_argument("set_bodies: z-slab ranks have no floating bodies");
    if (mid_step_) throw std::invalid_argument("set_bodies: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    if (num_bodies > 0 && tank_rotating()) throw std::invalid_argument("set_bodies: floating bodies are not supported in a rotating tank frame");
    if (num_bodies > 0 && !tag_densities_.empty()) throw std::invalid_argument("set_bodies: floating bodies are not supported with a tag density table");
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    restore_bodies(make_body_set(dim, bodies, num_bodies, false));
}

void HybridFluid::set_bodies_meshes(const BlubBody *bodies, const BlubMesh *const *meshes, const float *scales, uint32_t num_bodies) {
    if (num_bodies > (uint32_t)BODIES_MAX) throw std::invalid_argument("set_bodies: at most 16 bodies");
    if (num_bodies && (!bodies || !meshes || !scales)) throw std::invalid_argument("set_bodies: NULL body, mesh or scale array");
    std::vector<HostMesh> host(num_bodies);
    for (uint32_t i = 0; i < num_bodies; ++i) {
        if (!meshes[i]) continue;
        if (mesh_device(*meshes[i]) != device_) throw std::invalid_argument("set_bodies: a mesh lives on another device");
        host[i].present = true;
        host[i].scale = scales[i];
        mesh_download(*meshes[i], host[i].positions, host[i].indices);
    }
    set_bodies_host(bodies, host);
}

void HybridFluid::set_bodies_host(const BlubBody *bodies, const std::vector<HostMesh> &meshes) {
    if (slab_world_ > 1) throw std::invalid_argument("set_bodies: z-slab ranks have no floating bodies");
    if (mid_step_) throw std::invalid_argument("set_bodies: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    const uint32_t num_bodies = (uint32_t)meshes.size();
    if (num_bodies > 0 && tank_rotating()) throw std::invalid_argument("set_bodies: floating bodies are not supported in a rotating tank frame");
    if (num_bodies > 0 && !tag_densities_.empty()) throw std::invalid_argument("set_bodies: floating bodies are not supported with a tag density table");
    if (num_bodies > (uint32_t)BODIES_MAX) throw std::invalid_argument("set_bodies: at most 16 bodies");
    if (num_bodies && !bodies) throw std::invalid_argument("set_bodies: NULL body array");
    const uint32_t dim[3] = {(uint32_t)grid_.nx, (uint32_t)grid_.ny, (uint32_t)grid_.nz};
    std::vector<BlubBody> set(num_bodies);
    std::vector<MeshBodyHost> host = make_mesh_body_set(dim, bodies, meshes, set);
    restore_bodies(set, std::move(host));
}

std::vector<MeshBodyHost> make_mesh_body_set(const uint32_t dim[3], const BlubBody *bodies, const std::vector<HostMesh> &meshes, std::vector<BlubBody> &set) {
    const size_t n = meshes.size();
    set.assign(n, BlubBody{});
    std::vector<MeshBodyHost> host(n);
    size_t vertices = 0, triangles = 0;
    bool any = false;
    for (size_t i = 0; i < n; ++i) {
        if (!meshes[i].present) {
            set[i] = make_body_set(dim, bodies + i, 1, false)[0];
            continue;
        }
        const HostMesh &m = meshes[i];
        host[i] = make_mesh_body(dim, bodies[i], m.positions.data(), (uint32_t)(m.positions.size() / 3), m.indices.data(), (uint32_t)m.indices.size(),
                                 m.scale, set[i]);
        vertices += m.positions.size() / 3;
        triangles += m.indices.size() / 3;
        any = true;
    }
    if (vertices > (size_t)BLUB_MESH_BODY_MAX_VERTICES || triangles > (size_t)BLUB_MESH_BODY_MAX_TRIANGLES)
        throw std::invalid_argument("set_bodies: the mesh bodies hold more than " + std::to_string(BLUB_MESH_BODY_MAX_VERTICES) + " vertices or " +
                                    std::to_string(BLUB_MESH_BODY_MAX_TRIANGLES) + " triangles");
    if (!any) host.clear();
    return host;
}

BlubMeshBodyProperties HybridFluid::body_mass_properties(uint32_t body) const {
    if (body >= num_bodies_ || mesh_bodies_.empty() || mesh_bodies_[body].vertices.empty())
        throw std::invalid_argument("body_mass_properties: not a mesh body");
    return mesh_bodies_[body].props;
}

void HybridFluid::free_mesh_bodies() {
    cudaFree(mesh_.info);
    cudaFree(mesh_.body_vertices);
    cudaFree(mesh_.grid_vertices);
    cudaFree(mesh_.indices);
    cudaFree(mesh_.bits);
    cudaFree(mesh_.origin);
    mesh_ = MeshBodySet{};
    mesh_bodies_.clear();
}

void HybridFluid::restore_bodies(const std::vector<BlubBody> &set, std::vector<MeshBodyHost> meshes) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // no step in flight reads the old bodies or writes the ring
    uint32_t cube = 0;
    for (size_t i = 0; i < set.size(); ++i)
        cube = std::max(cube, meshes.empty() || meshes[i].vertices.empty() ? body_cube_side(set[i]) : mesh_body_cube_side(set[i].half_extent, meshes[i].mid));
    free_mesh_bodies();
    if (!meshes.empty()) {
        std::vector<MeshBodyDev> info(BODIES_MAX, MeshBodyDev{});
        std::vector<float> vb;
        std::vector<uint32_t> idx;
        for (size_t i = 0; i < meshes.size(); ++i) {
            const MeshBodyHost &m = meshes[i];
            MeshBodyDev &d = info[i];
            d.first_vertex = (uint32_t)(vb.size() / 3);
            d.first_triangle = (uint32_t)(idx.size() / 3);
            d.num_vertices = (uint32_t)(m.vertices.size() / 3);
            d.num_triangles = (uint32_t)(m.indices.size() / 3);
            d.mass = m.props.mass;
            for (int k = 0; k < 3; ++k) d.inertia[k] = m.props.moments[k], d.mid[k] = m.mid[k];
            vb.insert(vb.end(), m.vertices.begin(), m.vertices.end());
            for (uint32_t v : m.indices) idx.push_back(d.first_vertex + v);
            mesh_.max_vertices = std::max(mesh_.max_vertices, d.num_vertices);
            mesh_.max_triangles = std::max(mesh_.max_triangles, d.num_triangles);
        }
        mesh_.words = (cube + 31) / 32;
        const size_t bit_words = set.size() * (size_t)cube * cube * mesh_.words;
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.info, BODIES_MAX * sizeof(MeshBodyDev)));
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.body_vertices, vb.size() * sizeof(float)));
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.grid_vertices, vb.size() * sizeof(float)));
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.indices, idx.size() * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.bits, bit_words * sizeof(uint32_t)));
        BLUB_CUDA_CHECK(cudaMalloc(&mesh_.origin, BODIES_MAX * 3 * sizeof(int)));
        BLUB_CUDA_CHECK(cudaMemset(mesh_.origin, 0, BODIES_MAX * 3 * sizeof(int)));
        BLUB_CUDA_CHECK(cudaMemcpy(mesh_.info, info.data(), BODIES_MAX * sizeof(MeshBodyDev), cudaMemcpyHostToDevice));
        BLUB_CUDA_CHECK(cudaMemcpy(mesh_.body_vertices, vb.data(), vb.size() * sizeof(float), cudaMemcpyHostToDevice));
        BLUB_CUDA_CHECK(cudaMemcpy(mesh_.indices, idx.data(), idx.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        BLUB_CUDA_CHECK(cudaMemset(mesh_.bits, 0, bit_words * sizeof(uint32_t)));
        mesh_bodies_ = std::move(meshes);
    }
    if (!set.empty()) {
        const size_t ring_bytes = (size_t)BODIES_MAX * BODY_HISTORY_LENGTH * sizeof(BlubBodyRecord);
        if (!bodies_dev_) {
            BLUB_CUDA_CHECK(cudaMalloc(&bodies_dev_, BODIES_MAX * sizeof(BlubBody)));
            BLUB_CUDA_CHECK(cudaMalloc(&body_sums_, BODIES_MAX * 8 * sizeof(unsigned long long)));
            BLUB_CUDA_CHECK(cudaMalloc(&body_ring_, ring_bytes));
            BLUB_CUDA_CHECK(cudaMalloc(&composite_, (size_t)grid_.n * sizeof(uint2)));
            BLUB_CUDA_CHECK(cudaMemset(composite_, 0, (size_t)grid_.n * sizeof(uint2)));
        }
        BLUB_CUDA_CHECK(cudaMemcpy(bodies_dev_, set.data(), set.size() * sizeof(BlubBody), cudaMemcpyHostToDevice));
        BLUB_CUDA_CHECK(cudaMemset(body_sums_, 0, BODIES_MAX * 8 * sizeof(unsigned long long)));
        BLUB_CUDA_CHECK(cudaMemset(body_ring_, 0, ring_bytes));
    }
    num_bodies_ = (uint32_t)set.size();
    body_cube_ = cube;
    body_steps_.clear();
    destroy_graphs();
}

uint32_t HybridFluid::bodies(BlubBody *out, uint32_t capacity) {
    if (capacity && !out) throw std::invalid_argument("bodies: NULL output");
    const uint32_t n = std::min(capacity, num_bodies_);
    if (n == 0) return num_bodies_;
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaMemcpyAsync(out, bodies_dev_, n * sizeof(BlubBody), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    return num_bodies_;
}

uint32_t HybridFluid::body_history(uint32_t body, BlubBodyRecord *out, uint32_t capacity) {
    if (body >= num_bodies_) throw std::invalid_argument("body_history: no such body");
    if (capacity && !out) throw std::invalid_argument("body_history: NULL output");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    std::vector<BlubBodyRecord> ring(BODY_HISTORY_LENGTH);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(ring.data(), body_ring_ + (size_t)body * BODY_HISTORY_LENGTH, BODY_HISTORY_LENGTH * sizeof(BlubBodyRecord),
                                    cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    const uint32_t n = std::min<uint32_t>(capacity, (uint32_t)body_steps_.size());
    const size_t first = body_steps_.size() - n;
    for (uint32_t k = 0; k < n; ++k) out[k] = ring[body_steps_[first + k] % BODY_HISTORY_LENGTH];
    return n;
}

std::unique_ptr<HybridFluid> create_fluid_from_config(const SceneConfig &cfg, int device, cudaStream_t stream) {
    std::unique_ptr<HybridFluid> f(new HybridFluid(cfg.grid_dimension[0], cfg.grid_dimension[1], cfg.grid_dimension[2], cfg.max_num_particles, device, stream));
    const float scale = cfg.grid_to_world_scale;
    for (const SceneBox &b : cfg.fluid_cubes) { // src/scene/mod.rs:132-138
        const float mn[3] = {b.min[0] / scale, b.min[1] / scale, b.min[2] / scale};
        const float mx[3] = {b.max[0] / scale, b.max[1] / scale, b.max[2] / scale};
        f->add_fluid_cube(mn, mx, b.tag);
    }
    const float g[3] = {cfg.gravity[0] / scale, cfg.gravity[1] / scale, cfg.gravity[2] / scale}; // :139
    f->set_gravity_grid(g);
    if (!cfg.sources.empty() || !cfg.drains.empty()) { // after the cubes
        std::vector<BlubFluidSource> src(cfg.sources.size());
        std::vector<BlubFluidDrain> drn(cfg.drains.size());
        std::vector<uint32_t> tags(cfg.sources.size());
        for (size_t i = 0; i < src.size(); ++i) {
            tags[i] = cfg.sources[i].tag;
            for (int k = 0; k < 3; ++k) {
                src[i].min_grid[k] = cfg.sources[i].min[k] / scale;
                src[i].max_grid[k] = cfg.sources[i].max[k] / scale;
                src[i].velocity_grid[k] = cfg.sources[i].velocity[k] / scale;
            }
        }
        for (size_t i = 0; i < drn.size(); ++i)
            for (int k = 0; k < 3; ++k) {
                drn[i].min_grid[k] = cfg.drains[i].min[k] / scale;
                drn[i].max_grid[k] = cfg.drains[i].max[k] / scale;
            }
        f->set_flow(src.data(), tags.data(), (uint32_t)src.size(), drn.data(), (uint32_t)drn.size());
    }
    if (cfg.viscosity > 0.0f) {
        BlubViscosity v = kViscosityOff;
        v.kinematic_viscosity = scene_viscosity_grid(cfg);
        f->set_viscosity(&v);
    }
    if (!cfg.tag_viscosities.empty()) {
        const std::vector<BlubTagViscosity> t = scene_tag_viscosities_grid(cfg);
        f->set_tag_viscosities(t.data(), (uint32_t)t.size());
    }
    if (cfg.surface_tension > 0.0f) f->set_surface_tension(scene_surface_tension_grid(cfg));
    if (!cfg.tag_densities.empty()) f->set_tag_densities(cfg.tag_densities.data(), (uint32_t)cfg.tag_densities.size());
    if (cfg.has_whitewater) f->set_whitewater(&cfg.whitewater);
    if (cfg.interfacial_tension > 0.0f) f->set_interfacial_tension(cfg.interface_tags.data(), (uint32_t)cfg.interface_tags.size(), scene_interfacial_tension_grid(cfg));
    if (!cfg.load_probes.empty()) {
        const std::vector<BlubLoadProbe> probes = scene_load_probes_grid(cfg);
        f->set_load_probes(probes.data(), (uint32_t)probes.size());
    }
    if (!cfg.bodies.empty()) {
        const std::vector<BlubBody> bodies = scene_bodies_grid(cfg);
        bool mesh = false;
        for (const SceneBody &b : cfg.bodies) mesh = mesh || b.shape == 2;
        if (mesh) f->set_bodies_host(bodies.data(), scene_body_meshes(cfg));
        else f->set_bodies(bodies.data(), (uint32_t)bodies.size());
    }
    return f;
}

std::vector<BlubBody> scene_bodies_grid(const SceneConfig &cfg) {
    const float scale = cfg.grid_to_world_scale;
    std::vector<BlubBody> out(cfg.bodies.size());
    for (size_t i = 0; i < out.size(); ++i) {
        const SceneBody &s = cfg.bodies[i];
        BlubBody &b = out[i];
        b.shape = s.shape;
        b.relative_density = s.relative_density;
        for (int k = 0; k < 3; ++k) { // as the static objects are placed (models.rs:196-216)
            b.centre[k] = (s.position[k] - cfg.world_position[k]) / scale;
            b.half_extent[k] = s.half_extent[k] / scale;
            b.velocity[k] = s.velocity[k] / scale;
            b.angular_velocity[k] = s.angular_velocity[k];
        }
        quat_from_euler_deg_wxyz(s.rotation_angles_deg, b.rotation);
    }
    return out;
}

std::vector<HostMesh> scene_body_meshes(const SceneConfig &cfg) {
    std::vector<HostMesh> out(cfg.bodies.size());
    for (size_t i = 0; i < out.size(); ++i) {
        const SceneBody &s = cfg.bodies[i];
        if (s.shape != 2) continue;
        out[i].present = true;
        out[i].scale = s.model_scale / cfg.grid_to_world_scale;
        read_obj(s.model, out[i].positions, out[i].indices);
    }
    return out;
}

std::vector<BlubLoadProbe> scene_load_probes_grid(const SceneConfig &cfg) {
    const float scale = cfg.grid_to_world_scale;
    std::vector<BlubLoadProbe> out(cfg.load_probes.size());
    for (size_t i = 0; i < out.size(); ++i) {
        const SceneLoadProbe &p = cfg.load_probes[i];
        for (int k = 0; k < 3; ++k) {
            out[i].min_grid[k] = p.min[k] / scale;
            out[i].max_grid[k] = p.max[k] / scale;
            out[i].pivot_grid[k] = p.has_pivot ? p.pivot[k] / scale : 0.5f * (out[i].min_grid[k] + out[i].max_grid[k]);
        }
    }
    return out;
}

} // namespace blub
