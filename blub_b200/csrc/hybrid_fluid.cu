// hybrid_fluid.cu -- host side of the fluid: allocation, particle seeding and the recording of one step.
// Counterpart of src/simulation/hybrid_fluid.rs (HybridFluid::{new, add_fluid_cube, step, ...}).
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>

#include <nvtx3/nvToolsExt.h>

#include "blub_core.hpp"
#include "fluid_kernels.hpp"

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
    BLUB_CUDA_CHECK(cudaMallocHost(&params_host_, sizeof(StepParams) * 64));
    for (int k = 0; k < 64; ++k) BLUB_CUDA_CHECK(cudaEventCreateWithFlags(&param_events_[k], cudaEventDisableTiming));
    BLUB_CUDA_CHECK(cudaDeviceSynchronize());
    if (const char *rs = std::getenv("BLUB_RESORT_EVERY")) internal_resort_every_ = (uint32_t)std::atoi(rs);
    const char *ng = std::getenv("BLUB_NO_GRAPH");
    if (ng && ng[0] == '1') use_graph = false;
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
    if (solver_ && solver_->comm.seq) cudaFree(solver_->comm.seq);
    solver_.reset();
    field_velocity_.reset();
    field_density_.reset();
    if (window_) cudaFree(window_);
    for (int k = 0; k < 3; ++k) cudaFree(row_alt_[k]);
    cudaFree(mig_counters_);
    if (slab_error_host_) cudaFreeHost(slab_error_host_);
    cudaFree(params_dev_);
    cudaFreeHost(params_host_);
    for (int k = 0; k < 64; ++k) cudaEventDestroy(param_events_[k]);
    if (owns_stream_) cudaStreamDestroy(stream_);
}

// ---------------------------------------------------------------------------------------------------------------
// Particle seeding, hybrid_fluid.rs:609-678.  The jitter stream is rand 0.8.5 `SmallRng` (xoshiro256++ seeded from a
// u64 through SplitMix64) drawing cgmath::Vector3<f32> as x, y, z with f32 = (next_u32 >> 8) * 2^-24 and next_u32 = high
// half of next_u64 -- third-party crates that are not vendored in the reference checkout (Cargo.lock: rand 0.8.5,
// rand_core 0.6.4, cgmath 0.18.0); restated from their published algorithms.
namespace {
struct Xoshiro256pp {
    uint64_t s[4];
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    explicit Xoshiro256pp(uint64_t state) {
        for (int i = 0; i < 4; ++i) {
            state += 0x9e3779b97f4a7c15ull;
            uint64_t z = state;
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            s[i] = z ^ (z >> 31);
        }
    }
    uint64_t next_u64() {
        const uint64_t result = rotl(s[0] + s[3], 23) + s[0];
        const uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return result;
    }
    float next_f32() { return (float)((uint32_t)(next_u64() >> 32) >> 8) * (1.0f / 16777216.0f); }
};

uint32_t clamp_to_grid(uint32_t dim, float v) { // hybrid_fluid.rs:609-617; Rust `as u32` saturates, NaN -> 0
    uint32_t u = !(v > 0.0f) ? 0u : (v >= 4294967040.0f ? 0xFFFFFFFFu : (uint32_t)v);
    uint32_t m = dim - 1 < u ? dim - 1 : u;
    return m < 1 ? 1 : m;
}
} // namespace

bool HybridFluid::add_fluid_cube(const float min_grid[3], const float max_grid[3]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
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
    if (slab_world_ > 1) return add_fluid_cube_slab(mn, ext);
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
        fresh[i] = make_float4(p[0], p[1], p[2], 0.0f);
    }
    BLUB_CUDA_CHECK(cudaMemcpyAsync(pos_[cur_] + num_particles_, fresh.data(), (size_t)num_new * sizeof(float4), cudaMemcpyHostToDevice, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_)); // `fresh` is pageable: finish before it dies (queue.write_buffer semantics)
    num_particles_ += num_new;
    return truncated;
}

// Slab rank: the same particle stream as the single-GPU seeding (same RNG draws in the same order -- the seed is the GLOBAL
// particle count, hybrid_fluid.rs:637), of which this rank keeps the particles whose cell lies in its planes, re-based to
// local z.  `seeded_global_` mirrors the reference's running num_particles for the seed of the next cube.
bool HybridFluid::add_fluid_cube_slab(const uint32_t mn[3], const uint32_t ext[3]) {
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
        if (cz >= z0 && cz < z1) fresh.push_back(make_float4(p[0], p[1], p[2] - (float)z0 + (float)SLAB_HALO, 0.0f));
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

void HybridFluid::set_device_particle_count(uint32_t n) {
    BLUB_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<char *>(params_dev_) + offsetof(StepParams, num_particles), &n, sizeof(uint32_t),
                                    cudaMemcpyHostToDevice, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

uint32_t HybridFluid::num_particles() const {
    if (slab_world_ <= 1) return num_particles_;
    uint32_t n = 0; // authoritative count lives on the device (migration)
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
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    num_particles_ = count;
    if (slab_world_ > 1) set_device_particle_count(count);
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
    for (int c = 0; c < 3; ++c) h->gravity_dt[c] = gravity_[c] * dt;
    h->tolerance[0] = field_velocity_->config.error_tolerance / dt; // pressure_solver.rs:193-201
    h->tolerance[1] = field_density_->config.error_tolerance / dt;
    h->num_particles = num_particles_;
    // sharded: the particle count changes on the device (migration) and is the last field: leave it alone
    const size_t bytes = slab_world_ > 1 ? offsetof(StepParams, num_particles) : sizeof(StepParams);
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
    const uint32_t np = slab_world_ > 1 ? max_num_particles_ : num_particles_; // sharded: the device-side count guards the kernels
    const NvtxScope scope(stage >= 0 && stage < 14 ? kScopeLabels[stage] : "stage");
    switch (stage) {
    case 0: // transfer particle velocity to grid (:806-833)
        if (!shard && !use_scatter_) {
            // cell lists -> marker (+ FLUID bits) -> one gather per component; deterministic, no accumulator volumes
            launch_cell_lists(stream_, grid_, params_dev_, np, pos_[cur_], 1.0f, lists_);
            launch_marker_from_lists(stream_, grid_, lists_, marker_.ptr, voxels_, bits);
            fluid_bits_stale_ = false;
            if (np > 0) launch_p2g_gather(stream_, grid_, params_dev_, lists_, pos_[cur_], row_, marker_.ptr, u);
            else for (int c = 0; c < 3; ++c) BLUB_CUDA_CHECK(cudaMemsetAsync(u[c], 0, (size_t)grid_.n * sizeof(float), stream_));
        } else if (!shard) {
            launch_p2g_scatter(stream_, grid_, params_dev_, np, pos_[cur_], row_, nw, marker_.ptr, false);
            launch_p2g_finish(stream_, grid_, params_dev_, u, nw, marker_.ptr, voxels_, bits, particle_words_);
            fluid_bits_stale_ = false;
        } else {
            launch_p2g_scatter(stream_, grid_, params_dev_, np, pos_[cur_], row_, nw, marker_.ptr, true);
            const SlabHaloItem items[4] = {{nw[0], sizeof(longlong2), 0}, {nw[1], sizeof(longlong2), 0}, {nw[2], sizeof(longlong2), 0}, {marker_.ptr, 1, 1}};
            slab_halo_exchange(items, 4); // X1
            launch_p2g_finish(stream_, grid_, params_dev_, u, nw, marker_.ptr, voxels_, bits, particle_words_);
            fluid_bits_stale_ = false;
        }
        break;
    case 1: // compute divergence -> PCG residual (:835-840)
        refresh_fluid_bits();
        launch_divergence_compute(stream_, grid_, bits, marker_.ptr, u, voxels_, solver_->residual());
        break;
    case 2: // primary pressure solver (:843-852)
        solver_->solve(stream_, *field_velocity_, 0, marker_.ptr, params_dev_, quirks);
        if (!capturing_) field_velocity_->enqueue_error_buffer_read(stream_, dt); // the scalars live until this field's next solve
        break;
    case 3: // particle binning every n-th step, including step 0 (:854-894)
        if (binning_step()) {
            launch_binning(stream_, grid_, params_dev_, np, pos_[cur_], pos_[1 - cur_], lists_);
            if (np > 0) cur_ = 1 - cur_; // ping-pong instead of the reference's full-buffer copy-back (:884-892)
        }
        break;
    case 4: // make velocity grid divergence free (:901-904)
        refresh_fluid_bits();
        launch_divergence_remove(stream_, grid_, bits, marker_.ptr, field_velocity_->pressure(), voxels_, u);
        break;
    case 5: // extrapolate velocity grid (:906-909)
        refresh_fluid_bits();
        launch_extrapolate(stream_, grid_, bits, u);
        if (shard) {
            const SlabHaloItem items[3] = {{u[0], sizeof(float), 2}, {u[1], sizeof(float), 2}, {u[2], sizeof(float), 2}};
            slab_halo_exchange(items, 3); // X2
        }
        break;
    case 6: // clear marker (& linked list) grids (:911-916)
        launch_clear_marker(stream_, grid_, marker_.ptr);
        break;
    case 7: // advect particles (:917-921)
        if (!shard) {
            launch_advect(stream_, grid_, params_dev_, np, pos_[cur_], row_, u, voxels_, marker_.ptr);
        } else {
            launch_advect_migrate(stream_, grid_, params_dev_, np, pos_[cur_], row_, u, voxels_, marker_.ptr, slab_migrate_targets());
            slab_migrate_finish();
            const SlabHaloItem items[1] = {{marker_.ptr, 1, 1}};
            slab_halo_exchange(items, 1); // X3
        }
        break;
    case 8: // density projection: set boundary marker (:923-927)
        launch_boundary_marker(stream_, grid_, marker_.ptr, voxels_, bits);
        fluid_bits_stale_ = false;
        break;
    case 9: // density projection: compute density error (:928-932)
        if (!shard) {
            launch_density_rhs(stream_, grid_, params_dev_, np, pos_[cur_], marker_.ptr, density_.ptr, solver_->residual());
        } else {
            launch_density_scatter(stream_, grid_, params_dev_, np, pos_[cur_], density_.ptr);
            const SlabHaloItem items[1] = {{density_.ptr, sizeof(long long), 0}};
            slab_halo_exchange(items, 1); // X4
            launch_density_finish(stream_, grid_, params_dev_, marker_.ptr, density_.ptr, solver_->residual());
        }
        break;
    case 10: // secondary pressure solver (:940-949)
        solver_->solve(stream_, *field_density_, 1, marker_.ptr, params_dev_, quirks);
        if (!capturing_) field_density_->enqueue_error_buffer_read(stream_, dt);
        break;
    case 11: // compute position change (:959-962)
        refresh_fluid_bits();
        launch_position_change(stream_, grid_, bits, params_dev_, marker_.ptr, field_density_->pressure(), u);
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
    if (!use_graph) {
        for (int s = 0; s < 14; ++s) run_stage(s, dt);
        return;
    }
    GraphSignature sig;
    sig.num_particles = num_particles_;
    sig.voxels = voxels_;
    sig.precond_mode = quirks.precond_mode;
    sig.max_it[0] = field_velocity_->config.max_num_iterations; sig.freq[0] = field_velocity_->config.error_check_frequency;
    sig.max_it[1] = field_density_->config.max_num_iterations; sig.freq[1] = field_density_->config.error_check_frequency;
    if (!(sig == graph_signature_)) {
        destroy_graphs();
        graph_signature_ = sig;
    }
    const bool binning = binning_step() && num_particles_ > 0;
    // Host-side buffer roles that a captured step bakes in (and changes): the graph is keyed by them.
    struct Roles {
        int cur, row_parity;
        uint32_t exchange_index, step_counter;
        float4 *row[3], *row_alt[3];
    };
    auto save_roles = [&]() {
        Roles r{cur_, row_parity_, slab_exchange_index_, step_counter_, {row_[0], row_[1], row_[2]}, {row_alt_[0], row_alt_[1], row_alt_[2]}};
        return r;
    };
    auto restore_roles = [&](const Roles &r) {
        cur_ = r.cur; row_parity_ = r.row_parity; slab_exchange_index_ = r.exchange_index; step_counter_ = r.step_counter;
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
        graph_roles_after_[before.cur][kb][before.row_parity][kx] = {cur_, row_parity_, slab_exchange_index_ - before.exchange_index};
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
    step_counter_ = before.step_counter + 1;
    field_velocity_->enqueue_error_buffer_read(stream_, dt);
    field_density_->enqueue_error_buffer_read(stream_, dt);
}

void HybridFluid::step_stages(double simulation_delta_seconds, int from, int to) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    if (!(dt > 0.0f)) throw std::invalid_argument("simulation delta must be positive");
    upload_step_params(dt);
    for (int s = from; s < to && s < 14; ++s) run_stage(s, dt);
    mid_step_ = to < 14;
}

void HybridFluid::step_timed(double simulation_delta_seconds, float ms[14]) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    upload_step_params(dt);
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

void HybridFluid::solve_only(int which, double simulation_delta_seconds) {
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    const float dt = (float)simulation_delta_seconds;
    upload_step_params(dt);
    solver_->solve(stream_, field(which), which, marker_.ptr, params_dev_, quirks);
}

std::unique_ptr<HybridFluid> create_fluid_from_config(const SceneConfig &cfg, int device, cudaStream_t stream) {
    std::unique_ptr<HybridFluid> f(new HybridFluid(cfg.grid_dimension[0], cfg.grid_dimension[1], cfg.grid_dimension[2], cfg.max_num_particles, device, stream));
    const float scale = cfg.grid_to_world_scale;
    for (const SceneBox &b : cfg.fluid_cubes) { // src/scene/mod.rs:132-138
        const float mn[3] = {b.min[0] / scale, b.min[1] / scale, b.min[2] / scale};
        const float mx[3] = {b.max[0] / scale, b.max[1] / scale, b.max[2] / scale};
        f->add_fluid_cube(mn, mx);
    }
    const float g[3] = {cfg.gravity[0] / scale, cfg.gravity[1] / scale, cfg.gravity[2] / scale}; // :139
    f->set_gravity_grid(g);
    return f;
}

} // namespace blub
