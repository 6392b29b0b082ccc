// state_file.cpp -- checkpoint / restart of a single-GPU fluid: HybridFluid::save_state / load_state and the host-only reader behind
// blub_state_info.  The file layout is documented in DESIGN.md §8 (checkpoint / restart); tests/test_state_file.py writes files from that
// description.  Arrays travel between the device and the file through one pinned staging buffer of fixed size, so the host memory a
// save or load needs does not grow with the fluid.
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>

#include "blub_core.hpp"

namespace blub {

namespace {

static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the state file is little-endian and written as the host lays it out");

constexpr char kMagic[8] = {'B', 'L', 'U', 'B', 'S', 'T', 'A', 'T'};
constexpr uint32_t kFormatVersion = 1;
constexpr uint32_t kNumSections = 13;
constexpr size_t kStagingBytes = 64u << 20; // two halves: one is filled while the other one is copied

enum : uint32_t {
    SEC_POSITIONS = 1, SEC_VELOCITY_X, SEC_VELOCITY_Y, SEC_VELOCITY_Z, SEC_GRID_VELOCITY_X, SEC_GRID_VELOCITY_Y, SEC_GRID_VELOCITY_Z,
    SEC_MARKER, SEC_PRESSURE_VELOCITY, SEC_PRESSURE_DENSITY, SEC_SOLVER_SCALARS, SEC_STATS_VELOCITY, SEC_STATS_DENSITY
};

struct StateHeader {
    char magic[8];
    uint32_t format_version;
    char library_version[32]; // blub_version(), NUL-padded; informational
    uint32_t grid_dimension[3];
    uint32_t max_num_particles, num_particles, step_count;
    uint32_t resort_every;          // internal re-sort cadence (BLUB_RESORT_EVERY when the run started)
    uint32_t rebin_frequency;       // DynamicSettings::particle_rebinning_step_frequency
    float gravity[3];               // grid units
    SolverConfig solver[2];         // velocity, density
    int32_t precond_mode;
    uint32_t transfer_path;         // blub_fluid_set_transfer_path value
    uint32_t solver_path;           // blub_fluid_set_solver_path value
    uint32_t graph_replay;
    uint32_t num_stats[2];          // samples in the statistics history of the velocity / density solve (<= 100)
    uint32_t num_sections;
    uint32_t header_crc;            // CRC-32 of the 140 bytes before it
};
static_assert(sizeof(SolverConfig) == 12 && sizeof(StateHeader) == 144, "state header layout");
static_assert(sizeof(PcgScalars) == 32 && sizeof(SolverStatisticSample) == 8, "state section layout");

struct SectionHead {
    uint32_t id, reserved;
    uint64_t length; // payload bytes; the payload is followed by its CRC-32 (4 bytes)
};
static_assert(sizeof(SectionHead) == 16, "section head layout");

struct Section {
    uint32_t id;
    uint64_t length;
};

// The sections of a file in their order, with the lengths its header implies.
void expected_sections(const StateHeader &h, Section out[kNumSections]) {
    const uint64_t np = (uint64_t)h.num_particles * 16, n = (uint64_t)h.grid_dimension[0] * h.grid_dimension[1] * h.grid_dimension[2];
    const Section s[kNumSections] = {{SEC_POSITIONS, np}, {SEC_VELOCITY_X, np}, {SEC_VELOCITY_Y, np}, {SEC_VELOCITY_Z, np},
                                     {SEC_GRID_VELOCITY_X, 4 * n}, {SEC_GRID_VELOCITY_Y, 4 * n}, {SEC_GRID_VELOCITY_Z, 4 * n}, {SEC_MARKER, n},
                                     {SEC_PRESSURE_VELOCITY, 4 * n}, {SEC_PRESSURE_DENSITY, 4 * n}, {SEC_SOLVER_SCALARS, 2 * sizeof(PcgScalars)},
                                     {SEC_STATS_VELOCITY, 8ull * h.num_stats[0]}, {SEC_STATS_DENSITY, 8ull * h.num_stats[1]}};
    std::memcpy(out, s, sizeof(s));
}

uint32_t crc_of(const void *p, size_t n, uint32_t crc = 0) { return (uint32_t)crc32_z(crc, static_cast<const Bytef *>(p), n); }

std::string errno_text() { return std::strerror(errno); }

struct File {
    FILE *f = nullptr;
    std::string path;
    File(const std::string &p, const char *mode) : path(p) {
        f = std::fopen(p.c_str(), mode);
        if (!f) throw IoError("cannot open " + p + ": " + errno_text());
    }
    ~File() {
        if (f) std::fclose(f);
    }
    void write(const void *p, size_t n) {
        if (n && std::fwrite(p, 1, n, f) != n) throw IoError("cannot write " + path + ": " + errno_text());
    }
    // a short read is a truncated file (the header check compares the file size first, so this is a file that shrank meanwhile)
    void read(void *p, size_t n) {
        if (n && std::fread(p, 1, n, f) != n) {
            if (std::ferror(f)) throw IoError("cannot read " + path + ": " + errno_text());
            throw ParseError(path + ": truncated state file");
        }
    }
    uint64_t size() {
        struct stat st;
        if (fstat(fileno(f), &st) != 0) throw IoError("cannot stat " + path + ": " + errno_text());
        return (uint64_t)st.st_size;
    }
};

// Staging memory of the array sections: pinned halves with an event each when the arrays come from / go to the device, plain host memory
// for the host-only reader.
struct Staging {
    char *half[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    std::vector<char> host;
    static constexpr size_t kHalf = kStagingBytes / 2;
    explicit Staging(bool pinned) {
        if (!pinned) {
            host.resize(kStagingBytes);
            half[0] = host.data();
            half[1] = host.data() + kHalf;
            return;
        }
        BLUB_CUDA_CHECK(cudaMallocHost(reinterpret_cast<void **>(&half[0]), kStagingBytes));
        half[1] = half[0] + kHalf;
        for (auto &e : done) BLUB_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    ~Staging() { // after an error copies may still be in flight: wait for them before the memory goes
        for (auto &e : done)
            if (e) {
                cudaEventSynchronize(e);
                cudaEventDestroy(e);
            }
        if (host.empty() && half[0]) cudaFreeHost(half[0]);
    }
    void wait(int k) {
        if (done[k]) BLUB_CUDA_CHECK(cudaEventSynchronize(done[k]));
    }
};

// Header checks: everything a reader needs to trust before it allocates anything.  Leaves `f` at the first section.
StateHeader read_header(File &f) {
    StateHeader h;
    const uint64_t size = f.size();
    if (size < sizeof(StateHeader)) throw ParseError(f.path + ": truncated state file (" + std::to_string(size) + " bytes)");
    f.read(&h, sizeof(h));
    if (std::memcmp(h.magic, kMagic, sizeof(kMagic)) != 0) throw ParseError(f.path + ": not a blub state file (bad magic)");
    if (h.format_version != kFormatVersion)
        throw ParseError(f.path + ": state format version " + std::to_string(h.format_version) + " is not supported (this library reads version " +
                         std::to_string(kFormatVersion) + ")");
    if (crc_of(&h, offsetof(StateHeader, header_crc)) != h.header_crc) throw ParseError(f.path + ": header checksum mismatch");
    const uint32_t *d = h.grid_dimension;
    if (d[0] == 0 || d[1] == 0 || d[2] == 0 || d[0] % 8 || d[1] % 8 || d[2] % 8)
        throw ParseError(f.path + ": grid dimensions must be positive multiples of 8");
    const uint64_t cells = (uint64_t)d[0] * d[1] * d[2];
    if (cells <= 16384 || cells >= (1ull << 31)) throw ParseError(f.path + ": grid must have more than 16384 and fewer than 2^31 cells");
    if (h.num_particles > h.max_num_particles) throw ParseError(f.path + ": num_particles exceeds max_num_particles");
    if (h.num_stats[0] > PressureField::SOLVER_STATISTIC_HISTORY_LENGTH || h.num_stats[1] > PressureField::SOLVER_STATISTIC_HISTORY_LENGTH)
        throw ParseError(f.path + ": statistics history longer than 100 samples");
    if (h.precond_mode < 0 || h.precond_mode > 1 || h.transfer_path > 1 || h.graph_replay > 1)
        throw ParseError(f.path + ": precond_mode, transfer path or graph replay flag out of range");
    const uint32_t sp = h.solver_path;
    if (sp > 6 || sp == 3 || sp == 5 || (sp == 2 && d[0] % 128)) throw ParseError(f.path + ": solver path out of range");
    if (h.num_sections != kNumSections) throw ParseError(f.path + ": " + std::to_string(h.num_sections) + " sections, expected 13");
    Section sec[kNumSections];
    expected_sections(h, sec);
    uint64_t total = sizeof(StateHeader);
    for (const Section &s : sec) total += sizeof(SectionHead) + s.length + 4;
    if (size != total)
        throw ParseError(f.path + ": the file has " + std::to_string(size) + " bytes, its header describes " + std::to_string(total));
    return h;
}

// Reads one section whose id and length must be `s`, in chunks of at most one staging half; sink(slot, data, bytes, offset) receives
// every chunk (it must be done with the half `slot` before that half's event is waited on again), then the CRC is checked.
template <class Sink> void read_section(File &f, const Section &s, Staging &st, Sink sink) {
    SectionHead head;
    f.read(&head, sizeof(head));
    if (head.id != s.id) throw ParseError(f.path + ": section " + std::to_string(s.id) + " expected, found " + std::to_string(head.id));
    if (head.length != s.length)
        throw ParseError(f.path + ": section " + std::to_string(s.id) + " has " + std::to_string(head.length) + " bytes, the header implies " +
                         std::to_string(s.length));
    uint32_t crc = crc_of(nullptr, 0);
    uint64_t off = 0;
    for (int k = 0; off < s.length; k ^= 1) {
        const size_t n = (size_t)std::min<uint64_t>(Staging::kHalf, s.length - off);
        st.wait(k);
        f.read(st.half[k], n);
        crc = crc_of(st.half[k], n, crc);
        sink(k, st.half[k], n, off);
        off += n;
    }
    uint32_t stored = 0;
    f.read(&stored, 4);
    if (stored != crc) throw ParseError(f.path + ": checksum mismatch in section " + std::to_string(s.id));
}

// A section from device memory: the copy of chunk k+1 runs while chunk k is checksummed and written.
void write_device_section(File &f, uint32_t id, const void *src, uint64_t bytes, Staging &st, cudaStream_t stream) {
    const SectionHead head{id, 0, bytes};
    f.write(&head, sizeof(head));
    uint32_t crc = crc_of(nullptr, 0);
    auto enqueue = [&](int k, uint64_t off) {
        const size_t n = (size_t)std::min<uint64_t>(Staging::kHalf, bytes - off);
        BLUB_CUDA_CHECK(cudaMemcpyAsync(st.half[k], static_cast<const char *>(src) + off, n, cudaMemcpyDeviceToHost, stream));
        BLUB_CUDA_CHECK(cudaEventRecord(st.done[k], stream));
    };
    if (bytes) enqueue(0, 0);
    for (uint64_t off = 0, k = 0; off < bytes; k ^= 1) {
        const size_t n = (size_t)std::min<uint64_t>(Staging::kHalf, bytes - off);
        if (off + n < bytes) enqueue((int)(k ^ 1), off + n);
        st.wait((int)k);
        crc = crc_of(st.half[k], n, crc);
        f.write(st.half[k], n);
        off += n;
    }
    f.write(&crc, 4);
}

void write_host_section(File &f, uint32_t id, const void *src, uint64_t bytes) {
    const SectionHead head{id, 0, bytes};
    f.write(&head, sizeof(head));
    const uint32_t crc = crc_of(src, (size_t)bytes);
    f.write(src, (size_t)bytes);
    f.write(&crc, 4);
}

} // namespace

StateInfo read_state_info(const std::string &path) {
    File f(path, "rb");
    const StateHeader h = read_header(f);
    Section sec[kNumSections];
    expected_sections(h, sec);
    Staging st(false);
    for (const Section &s : sec) read_section(f, s, st, [](int, const char *, size_t, uint64_t) {});
    StateInfo info;
    std::memcpy(info.grid_dimension, h.grid_dimension, sizeof(info.grid_dimension));
    info.max_num_particles = h.max_num_particles;
    info.num_particles = h.num_particles;
    info.step_count = h.step_count;
    info.format_version = h.format_version;
    return info;
}

void HybridFluid::save_state(const std::string &path) {
    if (slab_world_ > 1) throw std::invalid_argument("save_state: z-slab ranks cannot be saved");
    if (mid_step_) throw std::invalid_argument("save_state: the fluid is inside a step (the last step_stages call did not end at stage 14)");
    BLUB_CUDA_CHECK(cudaSetDevice(device_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    update_statistics(); // every finished solve is in the history now
    StateHeader h{}; // no padding: every byte written is a field or zero
    std::memcpy(h.magic, kMagic, sizeof(kMagic));
    h.format_version = kFormatVersion;
    std::strncpy(h.library_version, blub_version(), sizeof(h.library_version) - 1);
    h.grid_dimension[0] = (uint32_t)grid_.nx;
    h.grid_dimension[1] = (uint32_t)grid_.ny;
    h.grid_dimension[2] = (uint32_t)grid_.nz;
    h.max_num_particles = max_num_particles_;
    h.num_particles = num_particles_;
    h.step_count = step_counter_;
    h.resort_every = internal_resort_every_;
    h.rebin_frequency = dynamic_settings_.particle_rebinning_step_frequency;
    for (int c = 0; c < 3; ++c) h.gravity[c] = gravity_[c];
    h.solver[0] = field_velocity_->config;
    h.solver[1] = field_density_->config;
    h.precond_mode = quirks.precond_mode;
    h.transfer_path = use_scatter_ ? 1 : 0;
    h.solver_path = (uint32_t)solver_->path();
    h.graph_replay = use_graph ? 1 : 0;
    h.num_stats[0] = (uint32_t)field_velocity_->stats.size();
    h.num_stats[1] = (uint32_t)field_density_->stats.size();
    h.num_sections = kNumSections;
    h.header_crc = crc_of(&h, offsetof(StateHeader, header_crc));

    PcgScalars scalars[2];
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&scalars[0], field_velocity_->scalars, sizeof(PcgScalars), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaMemcpyAsync(&scalars[1], field_density_->scalars, sizeof(PcgScalars), cudaMemcpyDeviceToHost, stream_));
    BLUB_CUDA_CHECK(cudaStreamSynchronize(stream_));
    std::vector<SolverStatisticSample> stats[2] = {{field_velocity_->stats.begin(), field_velocity_->stats.end()},
                                                   {field_density_->stats.begin(), field_density_->stats.end()}};

    // path.tmp first, made durable, then renamed over `path`: a crash during the save leaves the previous file intact
    const std::string tmp = path + ".tmp";
    try {
        Staging st(true);
        File f(tmp, "wb");
        f.write(&h, sizeof(h));
        const uint64_t np = (uint64_t)num_particles_ * sizeof(float4), n = (uint64_t)grid_.n;
        write_device_section(f, SEC_POSITIONS, pos_[cur_], np, st, stream_);
        for (int c = 0; c < 3; ++c) write_device_section(f, SEC_VELOCITY_X + c, row_[c], np, st, stream_);
        for (int c = 0; c < 3; ++c) write_device_section(f, SEC_GRID_VELOCITY_X + c, u_[c].ptr, 4 * n, st, stream_);
        write_device_section(f, SEC_MARKER, marker_.ptr, n, st, stream_);
        write_device_section(f, SEC_PRESSURE_VELOCITY, field_velocity_->pressure(), 4 * n, st, stream_);
        write_device_section(f, SEC_PRESSURE_DENSITY, field_density_->pressure(), 4 * n, st, stream_);
        write_host_section(f, SEC_SOLVER_SCALARS, scalars, sizeof(scalars));
        write_host_section(f, SEC_STATS_VELOCITY, stats[0].data(), stats[0].size() * sizeof(SolverStatisticSample));
        write_host_section(f, SEC_STATS_DENSITY, stats[1].data(), stats[1].size() * sizeof(SolverStatisticSample));
        if (std::fflush(f.f) != 0 || fsync(fileno(f.f)) != 0) throw IoError("cannot flush " + tmp + ": " + errno_text());
        FILE *raw = f.f;
        f.f = nullptr;
        if (std::fclose(raw) != 0) throw IoError("cannot close " + tmp + ": " + errno_text());
        if (std::rename(tmp.c_str(), path.c_str()) != 0) throw IoError("cannot rename " + tmp + " to " + path + ": " + errno_text());
    } catch (...) {
        std::remove(tmp.c_str());
        throw;
    }
}

std::unique_ptr<HybridFluid> HybridFluid::load_state(const std::string &path, int device, cudaStream_t stream) {
    File f(path, "rb");
    const StateHeader h = read_header(f); // every size is checked before anything is allocated
    Section sec[kNumSections];
    expected_sections(h, sec);
    std::unique_ptr<HybridFluid> fluid(
        new HybridFluid(h.grid_dimension[0], h.grid_dimension[1], h.grid_dimension[2], h.max_num_particles, device, stream));
    HybridFluid &x = *fluid;
    // the file's settings win over the environment the constructor read (BLUB_P2G, BLUB_RESORT_EVERY, BLUB_NO_GRAPH, BLUB_PCG)
    x.num_particles_ = h.num_particles;
    x.step_counter_ = h.step_count;
    x.internal_resort_every_ = h.resort_every;
    x.dynamic_settings_.particle_rebinning_step_frequency = h.rebin_frequency;
    x.set_gravity_grid(h.gravity);
    x.field_velocity_->config = h.solver[0];
    x.field_density_->config = h.solver[1];
    x.quirks.precond_mode = h.precond_mode;
    x.set_transfer_path((int)h.transfer_path);
    x.solver_->set_path((int)h.solver_path);
    x.use_graph = h.graph_replay != 0;

    Staging st(true);
    auto to_device = [&](const Section &s, void *dst) {
        read_section(f, s, st, [&](int k, const char *data, size_t n, uint64_t off) {
            BLUB_CUDA_CHECK(cudaMemcpyAsync(static_cast<char *>(dst) + off, data, n, cudaMemcpyHostToDevice, x.stream_));
            BLUB_CUDA_CHECK(cudaEventRecord(st.done[k], x.stream_));
        });
    };
    x.cur_ = 0;
    void *const arrays[10] = {x.pos_[0], x.row_[0], x.row_[1], x.row_[2], x.u_[0].ptr, x.u_[1].ptr, x.u_[2].ptr, x.marker_.ptr,
                              x.field_velocity_->pressure(), x.field_density_->pressure()};
    for (int k = 0; k < 10; ++k) to_device(sec[k], arrays[k]);
    auto to_host = [&](const Section &s, void *dst) {
        read_section(f, s, st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(static_cast<char *>(dst) + off, data, n); });
    };
    PcgScalars scalars[2];
    to_host(sec[10], scalars);
    BLUB_CUDA_CHECK(cudaMemcpyAsync(x.field_velocity_->scalars, &scalars[0], sizeof(PcgScalars), cudaMemcpyHostToDevice, x.stream_));
    BLUB_CUDA_CHECK(cudaMemcpyAsync(x.field_density_->scalars, &scalars[1], sizeof(PcgScalars), cudaMemcpyHostToDevice, x.stream_));
    for (int which = 0; which < 2; ++which) {
        std::vector<SolverStatisticSample> samples(h.num_stats[which]);
        to_host(sec[11 + which], samples.data());
        x.field(which).stats.assign(samples.begin(), samples.end());
    }
    x.fluid_bits_stale_ = true; // rebuilt from the restored marker volume before the next grid pass that reads it
    BLUB_CUDA_CHECK(cudaStreamSynchronize(x.stream_));
    return fluid;
}

} // namespace blub
