// state_file.cpp -- checkpoint / restart of a single-GPU fluid: HybridFluid::save_state / load_state and the host-only reader behind
// blub_state_info.  The file layout is documented in DESIGN.md §8 (checkpoint / restart); tests/test_state_file.py writes files from that
// description.  Arrays travel between the device and the file through one pinned staging buffer of fixed size, so the host memory a
// save or load needs does not grow with the fluid.
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "blub_core.hpp"

namespace blub {

namespace {

static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the state file is little-endian and written as the host lays it out");

constexpr char kMagic[8] = {'B', 'L', 'U', 'B', 'S', 'T', 'A', 'T'};
// version 1: a fluid without sources or drains, 13 sections; version 2: the same plus section 14, the flow set and its counters; version 4:
// section 14 followed by the sources' particle tags (written only when one of them is not 0).  Version 3 is not a format: no build writes
// it and readers refuse it.  Version 8: a fluid with floating bodies; the version-4 layout (section 14 may describe an empty flow set) plus
// section 15, the bodies.  Versions 3, 5, 6 and 7 are not formats either.  Version 16: a fluid with at least one mesh body; the version-8
// layout plus section 16, the mesh bodies' geometry and mass properties (its length is what the file holds beyond section 15).  Version 32: a
// fluid with viscosity; the layout it would otherwise have, promoted to 13 sections, or 14 (section 14 in its version-4 form, possibly an empty
// set), 15 or 16, plus a last section 17, the viscosity setting: num_sections (14 to 17) tells which.  Versions 17 to 31 are not formats.
constexpr uint32_t kFormatVersionFlow = 2, kFormatVersionSourceTags = 4, kFormatVersionBodies = 8, kFormatVersionMeshBodies = 16, kFormatVersionViscosity = 32;
constexpr uint32_t kNumSections = 17; // at most
constexpr size_t kStagingBytes = 64u << 20; // two halves: one is filled while the other one is copied

enum : uint32_t {
    SEC_POSITIONS = 1, SEC_VELOCITY_X, SEC_VELOCITY_Y, SEC_VELOCITY_Z, SEC_GRID_VELOCITY_X, SEC_GRID_VELOCITY_Y, SEC_GRID_VELOCITY_Z,
    SEC_MARKER, SEC_PRESSURE_VELOCITY, SEC_PRESSURE_DENSITY, SEC_SOLVER_SCALARS, SEC_STATS_VELOCITY, SEC_STATS_DENSITY, SEC_FLOW, SEC_BODIES,
    SEC_MESH_BODIES, SEC_VISCOSITY
};

// Section 14 (version 2): the flow set as clamped integer cell corners [lo, hi), unused slots zero, and the cumulative counters.
struct FlowSection {
    uint32_t num_sources, num_drains;
    int32_t source[16][6]; // lo x, y, z, hi x, y, z
    float velocity[16][3]; // cells/s
    int32_t drain[16][6];
    uint64_t counters[3];  // emitted, drained, refused for capacity
};
static_assert(sizeof(FlowSection) == 992 && FLOW_MAX_BOXES == 16, "flow section layout");
// Section 14 of version 4
struct FlowSectionTagged {
    FlowSection flow;
    uint32_t source_tags[16]; // unused slots zero
};
static_assert(sizeof(FlowSectionTagged) == 1056, "tagged flow section layout");
// Section 15 (version 8): the bodies, unused slots zero
struct BodySection {
    uint32_t num_bodies;
    BlubBody body[16];
};
static_assert(sizeof(BodySection) == 1156 && BODIES_MAX == 16, "body section layout");
// Section 16 (version 16): u32 num_mesh_bodies, u32 reserved, then per mesh body in body order this record followed by its float32 body-frame
// vertices (3 per vertex) and its uint32 indices (3 per triangle, into its own vertices)
struct MeshBodyRecordHead {
    uint32_t body, num_vertices, num_triangles, reserved;
    float mass, moments[3];           // as stored: the integrator's m and I_b
    float bounds_lo[3], bounds_hi[3]; // body-frame bounds
    float scale, reserved2;
    double volume, centroid[3], principal_moments[3], principal_rotation[4], inertia[9];
};
static_assert(sizeof(MeshBodyRecordHead) == 224, "mesh body record layout");
// Section 17 (version 32): the BlubViscosity as set, kinematic_viscosity > 0
static_assert(sizeof(BlubViscosity) == 16, "viscosity section layout");

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

// The sections of a file in their order, with the lengths its header implies; returns their number (0: a version-32 header whose
// num_sections names no layout).  The base sections come first: base_sections() of them, then section 17 in a version-32 file.
uint32_t base_sections(const StateHeader &h) {
    if (h.format_version == kFormatVersionViscosity) return h.num_sections >= 14 && h.num_sections <= 17 ? h.num_sections - 1 : 0;
    return h.format_version == kFormatVersionMeshBodies ? 16 : h.format_version == kFormatVersionBodies ? 15 : h.format_version >= kFormatVersionFlow ? 14 : 13;
}
uint32_t expected_sections(const StateHeader &h, Section out[kNumSections]) {
    const uint64_t np = (uint64_t)h.num_particles * 16, n = (uint64_t)h.grid_dimension[0] * h.grid_dimension[1] * h.grid_dimension[2];
    const Section s[kNumSections] = {{SEC_POSITIONS, np}, {SEC_VELOCITY_X, np}, {SEC_VELOCITY_Y, np}, {SEC_VELOCITY_Z, np},
                                     {SEC_GRID_VELOCITY_X, 4 * n}, {SEC_GRID_VELOCITY_Y, 4 * n}, {SEC_GRID_VELOCITY_Z, 4 * n}, {SEC_MARKER, n},
                                     {SEC_PRESSURE_VELOCITY, 4 * n}, {SEC_PRESSURE_DENSITY, 4 * n}, {SEC_SOLVER_SCALARS, 2 * sizeof(PcgScalars)},
                                     {SEC_STATS_VELOCITY, 8ull * h.num_stats[0]}, {SEC_STATS_DENSITY, 8ull * h.num_stats[1]},
                                     {SEC_FLOW, h.format_version >= kFormatVersionSourceTags ? sizeof(FlowSectionTagged) : sizeof(FlowSection)},
                                     {SEC_BODIES, sizeof(BodySection)}, {SEC_MESH_BODIES, 0}, // section 16: the file's bytes beyond the others
                                     {SEC_VISCOSITY, sizeof(BlubViscosity)}};
    std::memcpy(out, s, sizeof(s));
    const uint32_t nb = base_sections(h);
    if (h.format_version != kFormatVersionViscosity || nb == 0) return nb;
    out[nb] = s[16];
    return nb + 1;
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
    if (h.format_version != 1 && h.format_version != kFormatVersionFlow && h.format_version != kFormatVersionSourceTags &&
        h.format_version != kFormatVersionBodies && h.format_version != kFormatVersionMeshBodies && h.format_version != kFormatVersionViscosity)
        throw ParseError(f.path + ": state format version " + std::to_string(h.format_version) +
                         " is not supported (this library reads versions 1, 2, 4, 8, 16 and 32)");
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
    Section sec[kNumSections];
    const uint32_t ns = expected_sections(h, sec);
    if (h.num_sections != ns)
        throw ParseError(f.path + ": " + std::to_string(h.num_sections) + " sections, format version " + std::to_string(h.format_version) + " has " +
                         (ns ? std::to_string(ns) : std::string("14 to 17")));
    uint64_t total = sizeof(StateHeader);
    for (uint32_t k = 0; k < ns; ++k) total += sizeof(SectionHead) + sec[k].length + 4;
    // version 16: section 16 holds at least its count and one mesh body record
    if (base_sections(h) == 16 ? size < total + 8 + sizeof(MeshBodyRecordHead) : size != total)
        throw ParseError(f.path + ": the file has " + std::to_string(size) + " bytes, its header describes " + std::to_string(total));
    return h;
}

// Reads one section whose id and length must be `s`, in chunks of at most one staging half; sink(slot, data, bytes, offset) receives
// every chunk (it must be done with the half `slot` before that half's event is waited on again), then the CRC is checked.
// the length of section 16 when the file has one: what the file holds beyond section 15, its head and its CRC
uint64_t mesh_section_length(File &f, const StateHeader &h) {
    if (base_sections(h) != 16) return 0;
    Section sec[kNumSections];
    const uint32_t ns = expected_sections(h, sec);
    uint64_t total = sizeof(StateHeader);
    for (uint32_t k = 0; k < ns; ++k) total += sizeof(SectionHead) + sec[k].length + 4; // section 16 counted empty
    return f.size() - total;
}

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

// The flow set of section 14, checked with the rules of set_flow: the corners must be what clamping them again gives.  tags: the sources'
// particle tags (version 4), or nullptr.  Versions 8, 16 and 32 may describe an empty set.
FlowSet flow_set_of(const FlowSection &fl, const uint32_t *tags, const StateHeader &h, const std::string &path) {
    if (fl.num_sources > 16 || fl.num_drains > 16 || (fl.num_sources + fl.num_drains == 0 && h.format_version < kFormatVersionBodies))
        throw ParseError(path + ": section 14 must hold at most 16 boxes of each kind and at least one box");
    std::vector<BlubFluidSource> src(fl.num_sources);
    std::vector<BlubFluidDrain> drn(fl.num_drains);
    for (uint32_t b = 0; b < fl.num_sources; ++b)
        for (int k = 0; k < 3; ++k) {
            src[b].min_grid[k] = (float)fl.source[b][k];
            src[b].max_grid[k] = (float)fl.source[b][3 + k];
            src[b].velocity_grid[k] = fl.velocity[b][k];
        }
    for (uint32_t b = 0; b < fl.num_drains; ++b)
        for (int k = 0; k < 3; ++k) {
            drn[b].min_grid[k] = (float)fl.drain[b][k];
            drn[b].max_grid[k] = (float)fl.drain[b][3 + k];
        }
    FlowSet fs;
    try {
        fs = make_flow_set(h.grid_dimension, src.data(), tags, fl.num_sources, drn.data(), fl.num_drains);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 14: " + e.what());
    }
    for (uint32_t b = 0; b < fl.num_sources; ++b)
        for (int k = 0; k < 3; ++k)
            if (fs.source[b].lo[k] != fl.source[b][k] || fs.source[b].hi[k] != fl.source[b][3 + k])
                throw ParseError(path + ": section 14: a source corner lies outside [1, dim - 1]");
    for (uint32_t b = 0; b < fl.num_drains; ++b)
        for (int k = 0; k < 3; ++k)
            if (fs.drain[b].lo[k] != fl.drain[b][k] || fs.drain[b].hi[k] != fl.drain[b][3 + k])
                throw ParseError(path + ": section 14: a drain corner lies outside [1, dim - 1]");
    return fs;
}

// The bodies of section 15, checked with the rules of set_bodies; the poses are kept bit for bit.
std::vector<BlubBody> body_set_of(const BodySection &bs, const StateHeader &h, const std::string &path) {
    if (bs.num_bodies > 16) throw ParseError(path + ": section 15 holds more than 16 bodies");
    try {
        return make_body_set(h.grid_dimension, bs.body, bs.num_bodies, true);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 15: " + e.what());
    }
}

// Version 16: the bodies of section 15 with the mesh bodies of section 16 (bytes), kept bit for bit.  A mesh body's placement is checked as
// set_bodies checks a body (bounding box within 1e-3 of [1, dim - 1], on the box centred on c + R mid), its record for sizes, index ranges,
// finite values, positive mass and moments, bounds at least 1 cell thick that match its vertices and its half extents.
std::vector<BlubBody> mesh_body_set_of(const BodySection &bs, const std::vector<char> &bytes, const StateHeader &h, const std::string &path,
                                       std::vector<MeshBodyHost> &meshes) {
    auto bad = [&](const std::string &what) { return ParseError(path + ": section 16: " + what); };
    if (bs.num_bodies == 0 || bs.num_bodies > 16) throw ParseError(path + ": section 15 must hold 1 to 16 bodies");
    uint32_t count = 0;
    std::memcpy(&count, bytes.data(), 4);
    if (count == 0) throw bad("a version-16 file holds at least one mesh body");
    size_t off = 8;
    meshes.assign(bs.num_bodies, MeshBodyHost{});
    size_t vertices = 0, triangles = 0;
    for (uint32_t r = 0; r < count; ++r) {
        MeshBodyRecordHead m;
        if (bytes.size() - off < sizeof(m)) throw bad("truncated record");
        std::memcpy(&m, bytes.data() + off, sizeof(m));
        off += sizeof(m);
        if (m.body >= bs.num_bodies || bs.body[m.body].shape != 2 || !meshes[m.body].vertices.empty())
            throw bad("a record names no mesh body of section 15, or one twice");
        if (m.num_vertices == 0 || m.num_triangles == 0 || m.num_vertices > (uint32_t)BLUB_MESH_BODY_MAX_VERTICES ||
            m.num_triangles > (uint32_t)BLUB_MESH_BODY_MAX_TRIANGLES)
            throw bad("vertex or triangle count out of range");
        vertices += m.num_vertices;
        triangles += m.num_triangles;
        const size_t need = 12ull * m.num_vertices + 12ull * m.num_triangles;
        if (bytes.size() - off < need) throw bad("truncated geometry");
        MeshBodyHost &host = meshes[m.body];
        host.vertices.resize(3ull * m.num_vertices);
        host.indices.resize(3ull * m.num_triangles);
        std::memcpy(host.vertices.data(), bytes.data() + off, 12ull * m.num_vertices);
        std::memcpy(host.indices.data(), bytes.data() + off + 12ull * m.num_vertices, 12ull * m.num_triangles);
        off += need;
        for (uint32_t v : host.indices)
            if (v >= m.num_vertices) throw bad("an index is out of range");
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (size_t k = 0; k < host.vertices.size(); ++k) {
            if (!std::isfinite(host.vertices[k])) throw bad("a vertex is not finite");
            lo[k % 3] = std::min(lo[k % 3], host.vertices[k]);
            hi[k % 3] = std::max(hi[k % 3], host.vertices[k]);
        }
        BlubMeshBodyProperties &p = host.props;
        p.volume = m.volume;
        std::memcpy(p.centroid, m.centroid, sizeof(p.centroid));
        std::memcpy(p.inertia, m.inertia, sizeof(p.inertia));
        std::memcpy(p.principal_moments, m.principal_moments, sizeof(p.principal_moments));
        std::memcpy(p.principal_rotation, m.principal_rotation, sizeof(p.principal_rotation));
        p.mass = m.mass;
        p.scale = m.scale;
        p.num_vertices = m.num_vertices;
        p.num_triangles = m.num_triangles;
        bool ok = std::isfinite(m.mass) && m.mass > 0.0f && std::isfinite(m.scale) && m.scale > 0.0f && m.volume > 0.0;
        for (int k = 0; k < 3; ++k) {
            p.moments[k] = m.moments[k];
            p.bounds_lo[k] = m.bounds_lo[k];
            p.bounds_hi[k] = m.bounds_hi[k];
            ok = ok && std::isfinite(m.moments[k]) && m.moments[k] > 0.0f && m.bounds_lo[k] == lo[k] && m.bounds_hi[k] == hi[k] &&
                 hi[k] - lo[k] >= 1.0f && bs.body[m.body].half_extent[k] == 0.5f * (hi[k] - lo[k]);
            host.mid[k] = 0.5f * (lo[k] + hi[k]);
        }
        if (!ok) throw bad("a mass, moment, scale or bound is out of range or does not match the vertices");
    }
    if (off != bytes.size()) throw bad("bytes beyond the last record");
    if (vertices > (size_t)BLUB_MESH_BODY_MAX_VERTICES || triangles > (size_t)BLUB_MESH_BODY_MAX_TRIANGLES) throw bad("over the vertex or triangle limit");
    std::vector<BlubBody> set(bs.body, bs.body + bs.num_bodies);
    for (uint32_t i = 0; i < bs.num_bodies; ++i) {
        const bool mesh = set[i].shape == 2;
        if (mesh != !meshes[i].vertices.empty()) throw bad("a mesh body of section 15 has no record");
        BlubBody b = set[i];
        if (mesh) b.shape = 0, b.half_extent[0] = b.half_extent[1] = b.half_extent[2] = 1.0f; // its shape was checked above
        try {
            make_body_set(mesh ? nullptr : h.grid_dimension, &b, 1, true); // a mesh body's box is checked below
        } catch (const std::invalid_argument &e) {
            throw ParseError(path + ": section 15: " + e.what());
        }
        if (!mesh) continue;
        float e[3], o[3];
        mesh_body_box(set[i], meshes[i].mid, e, o);
        for (int k = 0; k < 3; ++k)
            if (set[i].centre[k] + o[k] - e[k] < 1.0f - 1e-3f || set[i].centre[k] + o[k] + e[k] > (float)h.grid_dimension[k] - 1.0f + 1e-3f)
                throw ParseError(path + ": section 15: a body's bounding box leaves [1, dim - 1]");
    }
    return set;
}

// The setting of section 17, checked with the rules of set_viscosity; a version-32 file has viscosity.
BlubViscosity viscosity_of(const BlubViscosity &v, const std::string &path) {
    try {
        check_viscosity(v);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 17: " + e.what());
    }
    if (!(v.kinematic_viscosity > 0.0f)) throw ParseError(path + ": section 17: a version-32 file holds a viscosity above 0");
    return v;
}

} // namespace

StateInfo read_state_info(const std::string &path) {
    File f(path, "rb");
    const StateHeader h = read_header(f);
    Section sec[kNumSections];
    const uint32_t ns = expected_sections(h, sec), nb = base_sections(h);
    Staging st(false);
    for (uint32_t k = 0; k < 13; ++k) read_section(f, sec[k], st, [](int, const char *, size_t, uint64_t) {});
    if (nb >= 14) {
        FlowSectionTagged fl{};
        read_section(f, sec[13], st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(reinterpret_cast<char *>(&fl) + off, data, n); });
        flow_set_of(fl.flow, fl.source_tags, h, f.path);
    }
    if (nb >= 15) {
        BodySection bs{};
        read_section(f, sec[14], st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(reinterpret_cast<char *>(&bs) + off, data, n); });
        if (nb == 15) body_set_of(bs, h, f.path);
        else {
            std::vector<char> bytes(mesh_section_length(f, h));
            read_section(f, {SEC_MESH_BODIES, bytes.size()}, st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(bytes.data() + off, data, n); });
            std::vector<MeshBodyHost> meshes;
            mesh_body_set_of(bs, bytes, h, f.path, meshes);
        }
    }
    if (ns > nb) {
        BlubViscosity v{};
        read_section(f, sec[nb], st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(reinterpret_cast<char *>(&v) + off, data, n); });
        viscosity_of(v, f.path);
    }
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
    bool source_tags = false;
    for (int b = 0; b < flow_.num_sources; ++b) source_tags = source_tags || flow_.tag[b] != 0u;
    const bool with_bodies = num_bodies_ > 0;
    const bool viscous = viscosity_.kinematic_viscosity > 0.0f;
    h.format_version = viscous ? kFormatVersionViscosity : has_mesh_bodies() ? kFormatVersionMeshBodies : with_bodies ? kFormatVersionBodies : !flow_active_ ? 1 : source_tags ? kFormatVersionSourceTags : kFormatVersionFlow;
    std::strncpy(h.library_version, blub_version(), sizeof(h.library_version) - 1);
    h.grid_dimension[0] = (uint32_t)grid_.nx;
    h.grid_dimension[1] = (uint32_t)grid_.ny;
    h.grid_dimension[2] = (uint32_t)grid_.nz;
    h.max_num_particles = max_num_particles_;
    h.num_particles = num_particles(); // the device count while sources or drains are set
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
    h.num_sections = (has_mesh_bodies() ? 16 : with_bodies ? 15 : flow_active_ ? 14 : 13) + (viscous ? 1 : 0);
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
        const uint64_t np = (uint64_t)h.num_particles * sizeof(float4), n = (uint64_t)grid_.n;
        write_device_section(f, SEC_POSITIONS, pos_[cur_], np, st, stream_);
        for (int c = 0; c < 3; ++c) write_device_section(f, SEC_VELOCITY_X + c, row_[c], np, st, stream_);
        for (int c = 0; c < 3; ++c) write_device_section(f, SEC_GRID_VELOCITY_X + c, u_[c].ptr, 4 * n, st, stream_);
        write_device_section(f, SEC_MARKER, marker_.ptr, n, st, stream_);
        write_device_section(f, SEC_PRESSURE_VELOCITY, field_velocity_->pressure(), 4 * n, st, stream_);
        write_device_section(f, SEC_PRESSURE_DENSITY, field_density_->pressure(), 4 * n, st, stream_);
        write_host_section(f, SEC_SOLVER_SCALARS, scalars, sizeof(scalars));
        write_host_section(f, SEC_STATS_VELOCITY, stats[0].data(), stats[0].size() * sizeof(SolverStatisticSample));
        write_host_section(f, SEC_STATS_DENSITY, stats[1].data(), stats[1].size() * sizeof(SolverStatisticSample));
        if (flow_active_ || with_bodies) {
            FlowSectionTagged tagged{};
            FlowSection &fl = tagged.flow;
            fl.num_sources = (uint32_t)flow_.num_sources;
            fl.num_drains = (uint32_t)flow_.num_drains;
            for (int b = 0; b < FLOW_MAX_BOXES; ++b)
                for (int k = 0; k < 3; ++k) {
                    if (b < flow_.num_sources) {
                        tagged.source_tags[b] = flow_.tag[b];
                        fl.source[b][k] = flow_.source[b].lo[k];
                        fl.source[b][3 + k] = flow_.source[b].hi[k];
                        fl.velocity[b][k] = flow_.velocity[b][k];
                    }
                    if (b < flow_.num_drains) {
                        fl.drain[b][k] = flow_.drain[b].lo[k];
                        fl.drain[b][3 + k] = flow_.drain[b].hi[k];
                    }
                }
            flow_counters(fl.counters);
            write_host_section(f, SEC_FLOW, &tagged, source_tags || with_bodies || viscous ? sizeof(tagged) : sizeof(fl));
        }
        if (with_bodies) {
            BodySection bs{};
            bs.num_bodies = bodies(bs.body, BODIES_MAX);
            write_host_section(f, SEC_BODIES, &bs, sizeof(bs));
        }
        if (has_mesh_bodies()) {
            std::vector<char> bytes(8, 0);
            uint32_t count = 0;
            for (const MeshBodyHost &m : mesh_bodies_) count += m.vertices.empty() ? 0 : 1;
            std::memcpy(bytes.data(), &count, 4);
            for (uint32_t i = 0; i < (uint32_t)mesh_bodies_.size(); ++i) {
                const MeshBodyHost &m = mesh_bodies_[i];
                if (m.vertices.empty()) continue;
                const BlubMeshBodyProperties &p = m.props;
                MeshBodyRecordHead r{};
                r.body = i;
                r.num_vertices = (uint32_t)(m.vertices.size() / 3);
                r.num_triangles = (uint32_t)(m.indices.size() / 3);
                r.mass = p.mass;
                r.scale = p.scale;
                r.volume = p.volume;
                for (int k = 0; k < 3; ++k) {
                    r.moments[k] = p.moments[k];
                    r.bounds_lo[k] = p.bounds_lo[k];
                    r.bounds_hi[k] = p.bounds_hi[k];
                    r.centroid[k] = p.centroid[k];
                    r.principal_moments[k] = p.principal_moments[k];
                }
                std::memcpy(r.principal_rotation, p.principal_rotation, sizeof(r.principal_rotation));
                std::memcpy(r.inertia, p.inertia, sizeof(r.inertia));
                const char *rb = reinterpret_cast<const char *>(&r);
                bytes.insert(bytes.end(), rb, rb + sizeof(r));
                const char *vb = reinterpret_cast<const char *>(m.vertices.data()), *ib = reinterpret_cast<const char *>(m.indices.data());
                bytes.insert(bytes.end(), vb, vb + m.vertices.size() * sizeof(float));
                bytes.insert(bytes.end(), ib, ib + m.indices.size() * sizeof(uint32_t));
            }
            write_host_section(f, SEC_MESH_BODIES, bytes.data(), bytes.size());
        }
        if (viscous) write_host_section(f, SEC_VISCOSITY, &viscosity_, sizeof(viscosity_));
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
    const uint32_t ns = expected_sections(h, sec), nb = base_sections(h);
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
    if (nb >= 14) {
        FlowSectionTagged fl{};
        to_host(sec[13], &fl);
        const FlowSet fs = flow_set_of(fl.flow, fl.source_tags, h, f.path);
        BLUB_CUDA_CHECK(cudaStreamSynchronize(x.stream_));
        if (fs.num_sources + fs.num_drains > 0) x.restore_flow(fs, fl.flow.counters); // the device takes over the restored count
    }
    if (nb >= 15) { // the history ring is not state: a loaded fluid starts with an empty one
        BodySection bs{};
        to_host(sec[14], &bs);
        if (nb == 15) x.restore_bodies(body_set_of(bs, h, f.path));
        else {
            std::vector<char> bytes(mesh_section_length(f, h));
            to_host({SEC_MESH_BODIES, bytes.size()}, bytes.data());
            std::vector<MeshBodyHost> meshes;
            const std::vector<BlubBody> set = mesh_body_set_of(bs, bytes, h, f.path, meshes);
            x.restore_bodies(set, std::move(meshes));
        }
    }
    if (ns > nb) { // the working volumes and the last solve are not state
        BlubViscosity v{};
        to_host(sec[nb], &v);
        v = viscosity_of(v, f.path);
        x.set_viscosity(&v);
    }
    BLUB_CUDA_CHECK(cudaStreamSynchronize(x.stream_));
    return fluid;
}

} // namespace blub
