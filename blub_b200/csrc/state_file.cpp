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
// The layout rule (DESIGN.md §8): a header, sections 1 to 13 at the lengths the header implies, then a strictly ascending selection of the
// optional sections 14 to 21 of kOptional.  Section 15 needs 14 and 16 needs 15, so num_sections, which counts every section, tells how many of
// 14, 15 and 16 a file holds; the sections from 17 on are found by their ids.  format_version is the largest version that introduced one of the
// file's sections, or 1 when it has none; section 14 counts as version 4 when a source tag is not 0, and it is 992 bytes long in a version-2
// file only.  Every other version number is not a format.  The rules between sections are checked with the payloads.
constexpr uint32_t kFormatVersionFlow = 2, kFormatVersionSourceTags = 4;
constexpr size_t kStagingBytes = 64u << 20; // two halves: one is filled while the other one is copied

enum : uint32_t {
    SEC_POSITIONS = 1, SEC_VELOCITY_X, SEC_VELOCITY_Y, SEC_VELOCITY_Z, SEC_GRID_VELOCITY_X, SEC_GRID_VELOCITY_Y, SEC_GRID_VELOCITY_Z,
    SEC_MARKER, SEC_PRESSURE_VELOCITY, SEC_PRESSURE_DENSITY, SEC_SOLVER_SCALARS, SEC_STATS_VELOCITY, SEC_STATS_DENSITY, SEC_FLOW, SEC_BODIES,
    SEC_MESH_BODIES, SEC_VISCOSITY, SEC_SURFACE_TENSION, SEC_TAG_DENSITIES, SEC_TAG_VISCOSITIES, SEC_INTERFACIAL_TENSION, SEC_WHITEWATER
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
// Section 18 (version 64): the kinematic surface tension as set, above 0 (cells^3/s^2)
struct SurfaceTensionSection {
    float surface_tension;
    uint32_t reserved; // 0
};
static_assert(sizeof(SurfaceTensionSection) == 8, "surface tension section layout");
// Section 19 (version 128): the tag density table in the order it was set, unused entries zero
struct TagDensitySection {
    uint32_t count;
    uint32_t reserved; // 0
    BlubTagDensity entry[16];
};
static_assert(sizeof(TagDensitySection) == 136 && TAG_DENSITIES_MAX == 16, "tag density section layout");
// Section 20 (version 256): the tag viscosity table in the order it was set, unused entries zero
struct TagViscositySection {
    uint32_t count;
    uint32_t reserved; // 0
    BlubTagViscosity entry[16];
};
static_assert(sizeof(TagViscositySection) == 136 && TAG_VISCOSITIES_MAX == 16, "tag viscosity section layout");
// Section 21 (version 512): the kinematic interfacial tension as set, above 0 (cells^3/s^2), and phase B's tags in the order they were set,
// unused entries zero
struct InterfacialTensionSection {
    float tension;
    uint32_t count;
    uint32_t tag[16];
};
static_assert(sizeof(InterfacialTensionSection) == 72 && INTERFACE_TAGS_MAX == 16, "interfacial tension section layout");
// Section 22 (version 1024): this head, then `count` particles of 32 bytes each (the position float4, then the velocity float4)
struct WhitewaterSectionHead {
    BlubWhitewater setting;    // as set, capacity above 0
    uint64_t counters[3];      // emitted, removed, refused for capacity
    uint32_t count;            // live particles, at most the capacity
};
static_assert(sizeof(BlubWhitewater) == 64 && offsetof(WhitewaterSectionHead, count) == 88, "whitewater section layout");
constexpr uint64_t kWhitewaterHeadBytes = 92; // the head without its tail padding

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

// The optional sections in id order: the format version that introduced each one and its payload length.
struct OptionalSection {
    uint32_t id, version;
    uint64_t length; // section 14: in every version but 2 (fixed_length); sections 16 and 22: 0, their length is stored
    const char *name;
};
constexpr OptionalSection kOptional[] = {
    {SEC_FLOW, kFormatVersionFlow, sizeof(FlowSectionTagged), "the flow set"},
    {SEC_BODIES, 8, sizeof(BodySection), "the bodies"},
    {SEC_MESH_BODIES, 16, 0, "the mesh bodies"},
    {SEC_VISCOSITY, 32, sizeof(BlubViscosity), "the viscosity"},
    {SEC_SURFACE_TENSION, 64, sizeof(SurfaceTensionSection), "the surface tension"},
    {SEC_TAG_DENSITIES, 128, sizeof(TagDensitySection), "the tag densities"},
    {SEC_TAG_VISCOSITIES, 256, sizeof(TagViscositySection), "the tag viscosities"},
    {SEC_INTERFACIAL_TENSION, 512, sizeof(InterfacialTensionSection), "the interfacial tension"},
    {SEC_WHITEWATER, 1024, 0, "the whitewater"},
};
constexpr uint32_t kLastSection = SEC_WHITEWATER;
static_assert(sizeof(kOptional) / sizeof(kOptional[0]) == kLastSection - SEC_FLOW + 1, "one row per optional section");
const OptionalSection &optional_section(uint32_t id) { return kOptional[id - SEC_FLOW]; }

constexpr uint32_t bit(uint32_t id) { return 1u << id; }

// The payload length of a section the rule fixes: sections 14, 15 and 17 to 21.  Sections 16 and 22 are as long as they say.
uint64_t fixed_length(uint32_t id, uint32_t version) {
    return id == SEC_FLOW && version == kFormatVersionFlow ? sizeof(FlowSection) : optional_section(id).length;
}

// The format version of a file with the sections `sections` (bits 1 << id); source_tags: section 14 holds a source tag that is not 0.
uint32_t format_version_of(uint32_t sections, bool source_tags) {
    uint32_t v = 1;
    for (const OptionalSection &s : kOptional)
        if (sections & bit(s.id)) v = std::max(v, s.id == SEC_FLOW && source_tags ? kFormatVersionSourceTags : s.version);
    return v;
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
    uint64_t tell() { return (uint64_t)ftello(f); }
    void seek(uint64_t at) {
        if (fseeko(f, (off_t)at, SEEK_SET) != 0) throw IoError("cannot seek in " + path + ": " + errno_text());
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

// Header checks: everything a reader needs to trust before it walks the sections.  Leaves `f` at the first section.
StateHeader read_header(File &f) {
    StateHeader h;
    const uint64_t size = f.size();
    if (size < sizeof(StateHeader)) throw ParseError(f.path + ": truncated state file (" + std::to_string(size) + " bytes)");
    f.read(&h, sizeof(h));
    if (std::memcmp(h.magic, kMagic, sizeof(kMagic)) != 0) throw ParseError(f.path + ": not a blub state file (bad magic)");
    std::string versions = "1";
    bool known = h.format_version == 1 || h.format_version == kFormatVersionSourceTags;
    for (const OptionalSection &s : kOptional) {
        versions += (s.id == kLastSection ? " and " : ", ") + std::to_string(s.version) + (s.id == SEC_FLOW ? ", 4" : "");
        known = known || h.format_version == s.version;
    }
    if (!known)
        throw ParseError(f.path + ": state format version " + std::to_string(h.format_version) + " is not supported (this library reads versions " +
                         versions + ")");
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
    return h;
}

// The sections of the file in their order with the lengths the rule gives them, checked against the header and the file size before anything
// is allocated.  Sections 1 to 13 take the lengths the header implies.  The walk then reads the heads after section 13 in ascending-id order and
// ends at the first one that is not a later section the format version may hold.  It advances over each section by the rule's length, over
// section 16 by its stored one, so a wrong stored length of another section is reported as that section's length error and does not end the
// walk early.  The sections from 17 on are the walk's; num_sections tells how many of 14, 15 and 16 precede them.  Leaves `f` at the first
// section.
std::vector<Section> layout_of(File &f, const StateHeader &h) {
    const uint32_t v = h.format_version;
    const uint64_t np = (uint64_t)h.num_particles * 16, n = (uint64_t)h.grid_dimension[0] * h.grid_dimension[1] * h.grid_dimension[2];
    std::vector<Section> sec = {{SEC_POSITIONS, np}, {SEC_VELOCITY_X, np}, {SEC_VELOCITY_Y, np}, {SEC_VELOCITY_Z, np},
                                {SEC_GRID_VELOCITY_X, 4 * n}, {SEC_GRID_VELOCITY_Y, 4 * n}, {SEC_GRID_VELOCITY_Z, 4 * n}, {SEC_MARKER, n},
                                {SEC_PRESSURE_VELOCITY, 4 * n}, {SEC_PRESSURE_DENSITY, 4 * n}, {SEC_SOLVER_SCALARS, 2 * sizeof(PcgScalars)},
                                {SEC_STATS_VELOCITY, 8ull * h.num_stats[0]}, {SEC_STATS_DENSITY, 8ull * h.num_stats[1]}};
    const uint64_t first = f.tell(), size = f.size();
    uint64_t at = first;
    for (const Section &s : sec) at += sizeof(SectionHead) + s.length + 4;
    std::vector<Section> settings;
    for (uint32_t last = SEC_STATS_DENSITY; at + sizeof(SectionHead) <= size;) {
        SectionHead head;
        f.seek(at);
        f.read(&head, sizeof(head));
        if (head.id <= last || head.id > kLastSection || optional_section(head.id).version > v) break;
        // 18 and 19 never go together: a version-128 file has no section 18, and in later versions the check of section 19 refuses the pair
        if (head.id == SEC_SURFACE_TENSION && v == optional_section(SEC_TAG_DENSITIES).version) break;
        const uint64_t length = head.id == SEC_MESH_BODIES || head.id == SEC_WHITEWATER ? head.length : fixed_length(head.id, v);
        if (length > size - at) break;
        if (head.id >= SEC_VISCOSITY) settings.push_back({head.id, length});
        last = head.id;
        at += sizeof(SectionHead) + length + 4;
    }
    f.seek(first);
    // of 14, 15 and 16 the file holds those up to the last one its version may hold, or, in a version that introduced a setting section, fewer
    uint32_t hi = SEC_STATS_DENSITY;
    while (hi < SEC_MESH_BODIES && optional_section(hi + 1).version <= v) ++hi;
    const uint32_t lo = v >= optional_section(SEC_VISCOSITY).version ? SEC_STATS_DENSITY : hi, extra = (uint32_t)settings.size();
    if (h.num_sections < lo + extra || h.num_sections > hi + extra)
        throw ParseError(f.path + ": " + std::to_string(h.num_sections) + " sections, format version " + std::to_string(v) + " has " +
                         std::to_string(lo + extra) + (lo == hi ? "" : " to " + std::to_string(hi + extra)));
    const uint32_t base = h.num_sections - extra;
    for (uint32_t id = SEC_FLOW; id <= base; ++id) sec.push_back({id, id == SEC_MESH_BODIES ? 0 : fixed_length(id, v)});
    sec.insert(sec.end(), settings.begin(), settings.end());
    uint64_t total = sizeof(StateHeader);
    for (const Section &s : sec) total += sizeof(SectionHead) + s.length + 4;
    // section 16 holds at least its count and one mesh body record
    if (base == SEC_MESH_BODIES ? size < total + 8 + sizeof(MeshBodyRecordHead) : size != total)
        throw ParseError(f.path + ": the file has " + std::to_string(size) + " bytes, its header describes " + std::to_string(total));
    if (base == SEC_MESH_BODIES) sec[SEC_MESH_BODIES - 1].length = size - total;
    // the walk took no section newer than the version and the count placed 14, 15 and 16: only the version's own setting section can be
    // missing (section 14 of a version-4 file counts as version 4)
    uint32_t ids = 0;
    for (const Section &s : sec) ids |= bit(s.id);
    if (format_version_of(ids, v == kFormatVersionSourceTags) != v) {
        const OptionalSection &own = *std::find_if(std::begin(kOptional), std::end(kOptional), [&](const OptionalSection &s) { return s.version == v; });
        throw ParseError(f.path + ": format version " + std::to_string(v) + " ends with section " + std::to_string(own.id) + " (" + own.name +
                         "), the file has none");
    }
    return sec;
}

// The whitewater of section 22, checked with the rules of set_whitewater: a capacity above 0, at most that many particles, and a length that
// holds exactly them.  particles: count x 8 floats.
WhitewaterSectionHead whitewater_of(const std::vector<char> &bytes, std::vector<float> &particles, const std::string &path) {
    WhitewaterSectionHead w{};
    if (bytes.size() < kWhitewaterHeadBytes) throw ParseError(path + ": section 22 is shorter than its head");
    std::memcpy(&w, bytes.data(), kWhitewaterHeadBytes);
    if (w.setting.max_num_particles == 0) throw ParseError(path + ": section 22: the capacity must be above 0");
    try {
        check_whitewater(w.setting, "section 22");
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": " + e.what());
    }
    if (w.count > w.setting.max_num_particles) throw ParseError(path + ": section 22 holds more particles than its capacity");
    if (bytes.size() != kWhitewaterHeadBytes + 32ull * w.count)
        throw ParseError(path + ": section 22 has " + std::to_string(bytes.size()) + " bytes, " + std::to_string(w.count) + " particles take " +
                         std::to_string(kWhitewaterHeadBytes + 32ull * w.count));
    particles.resize(8ull * w.count);
    if (w.count) std::memcpy(particles.data(), bytes.data() + kWhitewaterHeadBytes, 32ull * w.count);
    return w;
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

// The flow set of section 14, checked with the rules of set_flow: the corners must be what clamping them again gives.  tags: the sources'
// particle tags (version 4), or nullptr.  From version 8 on it may describe an empty set.
FlowSet flow_set_of(const FlowSection &fl, const uint32_t *tags, const StateHeader &h, const std::string &path) {
    if (fl.num_sources > 16 || fl.num_drains > 16 || (fl.num_sources + fl.num_drains == 0 && h.format_version < optional_section(SEC_BODIES).version))
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

// The setting of section 17, checked with the rules of set_viscosity; it holds a viscosity above 0 unless the file has a section 20 (the tags
// not in that table are inviscid).  sections: the file's section ids, bits 1 << id.
BlubViscosity viscosity_of(const BlubViscosity &v, uint32_t sections, const std::string &path) {
    try {
        check_viscosity(v);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 17: " + e.what());
    }
    if (!(sections & bit(SEC_TAG_VISCOSITIES)) && !(v.kinematic_viscosity > 0.0f))
        throw ParseError(path + ": section 17: without a section 20 section 17 holds a viscosity above 0");
    return v;
}

// The setting of section 18, checked with the rules of set_surface_tension; a version-64 file has surface tension.
float surface_tension_of(const SurfaceTensionSection &s, const std::string &path) {
    if (!std::isfinite(s.surface_tension) || !(s.surface_tension > 0.0f)) throw ParseError(path + ": section 18: the surface tension must be finite and above 0");
    if (s.reserved != 0u) throw ParseError(path + ": section 18: reserved must be 0");
    return s.surface_tension;
}

// The table of section 19, checked with the rules of set_tag_densities: precond_mode 0, no surface tension and no floating bodies.
std::vector<BlubTagDensity> tag_densities_of(const TagDensitySection &s, const StateHeader &h, uint32_t sections, const std::string &path) {
    if (h.precond_mode != 0) throw ParseError(path + ": section 19: a tag density table needs precond_mode 0");
    if (sections & bit(SEC_SURFACE_TENSION)) throw ParseError(path + ": section 19: a tag density table is not supported with surface tension");
    if (sections & bit(SEC_BODIES)) throw ParseError(path + ": section 19: a tag density table is not supported with floating bodies");
    if (s.count == 0 || s.count > 16) throw ParseError(path + ": section 19 must hold 1 to 16 entries");
    if (s.reserved != 0u) throw ParseError(path + ": section 19: reserved must be 0");
    try {
        check_tag_densities(s.entry, s.count);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 19: " + e.what());
    }
    const BlubTagDensity zero{};
    for (uint32_t k = s.count; k < 16; ++k)
        if (std::memcmp(&s.entry[k], &zero, sizeof(zero)) != 0) throw ParseError(path + ": section 19: the unused entries must be zero");
    return std::vector<BlubTagDensity>(s.entry, s.entry + s.count);
}

// The table of section 20, checked with the rules of set_tag_viscosities; a version-256 file has a table.
std::vector<BlubTagViscosity> tag_viscosities_of(const TagViscositySection &s, const std::string &path) {
    if (s.count == 0 || s.count > 16) throw ParseError(path + ": section 20 must hold 1 to 16 entries");
    if (s.reserved != 0u) throw ParseError(path + ": section 20: reserved must be 0");
    try {
        check_tag_viscosities(s.entry, s.count);
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": section 20: " + e.what());
    }
    const BlubTagViscosity zero{};
    for (uint32_t k = s.count; k < 16; ++k)
        if (std::memcmp(&s.entry[k], &zero, sizeof(zero)) != 0) throw ParseError(path + ": section 20: the unused entries must be zero");
    return std::vector<BlubTagViscosity>(s.entry, s.entry + s.count);
}

// The setting of section 21, checked with the rules of set_interfacial_tension; a version-512 file has an interfacial tension above 0.
void interfacial_tension_of(const InterfacialTensionSection &s, const std::string &path) {
    if (!(s.tension > 0.0f)) throw ParseError(path + ": section 21: the interfacial tension must be above 0");
    if (s.count > 16) throw ParseError(path + ": section 21 must hold 1 to 16 tags");
    try {
        check_interfacial_tension(s.tag, s.count, s.tension, "section 21");
    } catch (const std::invalid_argument &e) {
        throw ParseError(path + ": " + e.what());
    }
    for (uint32_t k = s.count; k < 16; ++k)
        if (s.tag[k] != 0u) throw ParseError(path + ": section 21: the unused entries must be zero");
}

// What a state file holds besides its header and its ten arrays, checked with the setters' rules.
struct StateContents {
    uint32_t sections = 0; // the file's section ids, bits 1 << id
    PcgScalars scalars[2];
    std::vector<SolverStatisticSample> stats[2];
    FlowSet flow{};
    uint64_t flow_counters[3] = {0, 0, 0};
    std::vector<BlubBody> bodies;
    std::vector<MeshBodyHost> meshes;
    BlubViscosity viscosity{};
    SurfaceTensionSection surface_tension{};
    TagDensitySection densities{};
    TagViscositySection viscosities{};
    InterfacialTensionSection interfacial{};
    WhitewaterSectionHead whitewater{};
    std::vector<float> whitewater_particles;
};

// Reads the sections of `layout` (layout_of) in their order, `f` at the first one.  The ten array sections go to
// to_array(id, slot, data, bytes, offset), which is read_section's sink with the section id in front; the others are checked and returned.
template <class ArraySink>
StateContents read_sections(File &f, const StateHeader &h, const std::vector<Section> &layout, Staging &st, ArraySink to_array) {
    StateContents c;
    for (const Section &s : layout) c.sections |= bit(s.id);
    auto to_host = [&](const Section &s, void *dst) {
        read_section(f, s, st, [&](int, const char *data, size_t n, uint64_t off) { std::memcpy(static_cast<char *>(dst) + off, data, n); });
    };
    FlowSectionTagged fl{};
    BodySection bs{};
    std::vector<char> mesh_bytes;
    for (const Section &s : layout) {
        switch (s.id) {
        case SEC_SOLVER_SCALARS: to_host(s, c.scalars); break;
        case SEC_STATS_VELOCITY:
        case SEC_STATS_DENSITY: {
            std::vector<SolverStatisticSample> &stats = c.stats[s.id - SEC_STATS_VELOCITY];
            stats.resize(s.length / sizeof(SolverStatisticSample));
            to_host(s, stats.data());
            break;
        }
        case SEC_FLOW:
            to_host(s, &fl);
            c.flow = flow_set_of(fl.flow, fl.source_tags, h, f.path);
            std::memcpy(c.flow_counters, fl.flow.counters, sizeof(c.flow_counters));
            break;
        case SEC_BODIES:
            to_host(s, &bs);
            if (!(c.sections & bit(SEC_MESH_BODIES))) c.bodies = body_set_of(bs, h, f.path);
            break;
        case SEC_MESH_BODIES:
            mesh_bytes.resize(s.length);
            to_host(s, mesh_bytes.data());
            c.bodies = mesh_body_set_of(bs, mesh_bytes, h, f.path, c.meshes);
            break;
        case SEC_VISCOSITY:
            to_host(s, &c.viscosity);
            viscosity_of(c.viscosity, c.sections, f.path);
            break;
        case SEC_SURFACE_TENSION:
            to_host(s, &c.surface_tension);
            surface_tension_of(c.surface_tension, f.path);
            break;
        case SEC_TAG_DENSITIES:
            to_host(s, &c.densities);
            tag_densities_of(c.densities, h, c.sections, f.path);
            break;
        case SEC_TAG_VISCOSITIES:
            to_host(s, &c.viscosities);
            tag_viscosities_of(c.viscosities, f.path);
            if (!(c.sections & bit(SEC_VISCOSITY))) throw ParseError(f.path + ": section 20 needs a section 17 before it");
            break;
        case SEC_INTERFACIAL_TENSION:
            to_host(s, &c.interfacial);
            interfacial_tension_of(c.interfacial, f.path);
            break;
        case SEC_WHITEWATER: {
            std::vector<char> bytes(s.length);
            to_host(s, bytes.data());
            c.whitewater = whitewater_of(bytes, c.whitewater_particles, f.path);
            break;
        }
        default: read_section(f, s, st, [&](int k, const char *data, size_t n, uint64_t off) { to_array(s.id, k, data, n, off); });
        }
    }
    return c;
}

} // namespace

StateInfo read_state_info(const std::string &path) {
    File f(path, "rb");
    const StateHeader h = read_header(f);
    const std::vector<Section> layout = layout_of(f, h);
    Staging st(false);
    read_sections(f, h, layout, st, [](uint32_t, int, const char *, size_t, uint64_t) {});
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
    // the sections the fluid writes, bits 1 << id: 1 to 13 always, then the optional ones its features need
    uint32_t sections = bit(SEC_FLOW) - bit(SEC_POSITIONS);
    const bool with_bodies = num_bodies_ > 0;
    if (flow_active_ || with_bodies) sections |= bit(SEC_FLOW); // a fluid with bodies writes a flow section, possibly of an empty set
    if (with_bodies) sections |= bit(SEC_BODIES);
    if (has_mesh_bodies()) sections |= bit(SEC_MESH_BODIES);
    if (viscosity_.kinematic_viscosity > 0.0f || !tag_viscosities_.empty()) sections |= bit(SEC_VISCOSITY); // section 20 needs section 17
    if (surface_tension_ > 0.0f) sections |= bit(SEC_SURFACE_TENSION);
    if (!tag_densities_.empty()) sections |= bit(SEC_TAG_DENSITIES);
    if (!tag_viscosities_.empty()) sections |= bit(SEC_TAG_VISCOSITIES);
    if (interfacial_tension_ > 0.0f) sections |= bit(SEC_INTERFACIAL_TENSION);
    if (whitewater_on()) sections |= bit(SEC_WHITEWATER);
    h.format_version = format_version_of(sections, source_tags);
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
    h.num_sections = (uint32_t)__builtin_popcount(sections);
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
        if (sections & bit(SEC_FLOW)) {
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
            write_host_section(f, SEC_FLOW, &tagged, fixed_length(SEC_FLOW, h.format_version));
        }
        if (sections & bit(SEC_BODIES)) {
            BodySection bs{};
            bs.num_bodies = bodies(bs.body, BODIES_MAX);
            write_host_section(f, SEC_BODIES, &bs, sizeof(bs));
        }
        if (sections & bit(SEC_MESH_BODIES)) {
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
        if (sections & bit(SEC_VISCOSITY)) write_host_section(f, SEC_VISCOSITY, &viscosity_, sizeof(viscosity_));
        if (sections & bit(SEC_SURFACE_TENSION)) {
            const SurfaceTensionSection sts = {surface_tension_, 0u};
            write_host_section(f, SEC_SURFACE_TENSION, &sts, sizeof(sts));
        }
        if (sections & bit(SEC_TAG_DENSITIES)) {
            TagDensitySection tds{};
            tds.count = (uint32_t)tag_densities_.size();
            for (uint32_t k = 0; k < tds.count; ++k) tds.entry[k] = tag_densities_[k];
            write_host_section(f, SEC_TAG_DENSITIES, &tds, sizeof(tds));
        }
        if (sections & bit(SEC_TAG_VISCOSITIES)) {
            TagViscositySection tvs{};
            tvs.count = (uint32_t)tag_viscosities_.size();
            for (uint32_t k = 0; k < tvs.count; ++k) tvs.entry[k] = tag_viscosities_[k];
            write_host_section(f, SEC_TAG_VISCOSITIES, &tvs, sizeof(tvs));
        }
        if (sections & bit(SEC_INTERFACIAL_TENSION)) {
            InterfacialTensionSection its{};
            its.tension = interfacial_tension_;
            its.count = (uint32_t)interface_tags_.size();
            for (uint32_t k = 0; k < its.count; ++k) its.tag[k] = interface_tags_[k];
            write_host_section(f, SEC_INTERFACIAL_TENSION, &its, sizeof(its));
        }
        if (sections & bit(SEC_WHITEWATER)) {
            uint64_t counters[4];
            whitewater_counters(counters);
            WhitewaterSectionHead wh{};
            wh.setting = whitewater_;
            for (int k = 0; k < 3; ++k) wh.counters[k] = counters[1 + k];
            wh.count = (uint32_t)counters[0];
            std::vector<char> bytes(kWhitewaterHeadBytes + 32ull * wh.count);
            std::memcpy(bytes.data(), &wh, kWhitewaterHeadBytes);
            std::vector<float> pos(4ull * wh.count), vel(4ull * wh.count);
            download_whitewater(pos.data(), vel.data(), wh.count);
            for (uint32_t i = 0; i < wh.count; ++i) {
                std::memcpy(bytes.data() + kWhitewaterHeadBytes + 32ull * i, &pos[4ull * i], 16);
                std::memcpy(bytes.data() + kWhitewaterHeadBytes + 32ull * i + 16, &vel[4ull * i], 16);
            }
            write_host_section(f, SEC_WHITEWATER, bytes.data(), bytes.size());
        }
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
    const StateHeader h = read_header(f);
    const std::vector<Section> layout = layout_of(f, h); // every size is checked before anything is allocated
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
    x.cur_ = 0;
    void *const arrays[10] = {x.pos_[0], x.row_[0], x.row_[1], x.row_[2], x.u_[0].ptr, x.u_[1].ptr, x.u_[2].ptr, x.marker_.ptr,
                              x.field_velocity_->pressure(), x.field_density_->pressure()};
    StateContents c = read_sections(f, h, layout, st, [&](uint32_t id, int k, const char *data, size_t n, uint64_t off) {
        BLUB_CUDA_CHECK(cudaMemcpyAsync(static_cast<char *>(arrays[id - SEC_POSITIONS]) + off, data, n, cudaMemcpyHostToDevice, x.stream_));
        BLUB_CUDA_CHECK(cudaEventRecord(st.done[k], x.stream_));
    });
    BLUB_CUDA_CHECK(cudaMemcpyAsync(x.field_velocity_->scalars, &c.scalars[0], sizeof(PcgScalars), cudaMemcpyHostToDevice, x.stream_));
    BLUB_CUDA_CHECK(cudaMemcpyAsync(x.field_density_->scalars, &c.scalars[1], sizeof(PcgScalars), cudaMemcpyHostToDevice, x.stream_));
    for (int which = 0; which < 2; ++which) x.field(which).stats.assign(c.stats[which].begin(), c.stats[which].end());
    x.fluid_bits_stale_ = true; // rebuilt from the restored marker volume before the next grid pass that reads it
    if (c.sections & bit(SEC_FLOW)) {
        BLUB_CUDA_CHECK(cudaStreamSynchronize(x.stream_));
        if (c.flow.num_sources + c.flow.num_drains > 0) x.restore_flow(c.flow, c.flow_counters); // the device takes over the restored count
    }
    // the history ring is not state: a loaded fluid starts with an empty one
    if (c.sections & bit(SEC_BODIES)) x.restore_bodies(c.bodies, std::move(c.meshes));
    // the working volumes, the last viscosity solve, the curvature, the cell densities, viscosities and coefficients are not state: the steps
    // form them again
    if (c.sections & bit(SEC_VISCOSITY)) x.set_viscosity(&c.viscosity);
    if (c.sections & bit(SEC_SURFACE_TENSION)) x.set_surface_tension(c.surface_tension.surface_tension);
    if (c.sections & bit(SEC_TAG_DENSITIES)) x.set_tag_densities(c.densities.entry, c.densities.count);
    if (c.sections & bit(SEC_TAG_VISCOSITIES)) x.set_tag_viscosities(c.viscosities.entry, c.viscosities.count);
    if (c.sections & bit(SEC_INTERFACIAL_TENSION)) x.set_interfacial_tension(c.interfacial.tag, c.interfacial.count, c.interfacial.tension);
    if (c.sections & bit(SEC_WHITEWATER))
        x.restore_whitewater(c.whitewater.setting, c.whitewater.counters, c.whitewater.count, c.whitewater_particles.data());
    BLUB_CUDA_CHECK(cudaStreamSynchronize(x.stream_));
    return fluid;
}

} // namespace blub
