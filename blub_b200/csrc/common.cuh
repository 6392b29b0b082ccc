// common.cuh -- shared device/host helpers of libblubcore (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace blub {

// marker values, shader/simulation/hybrid_fluid.glsl:20-23
constexpr int CELL_SOLID = 0;
constexpr int CELL_FLUID = 1;
constexpr int CELL_AIR = -1;

struct CudaError : std::runtime_error {
    explicit CudaError(const std::string &what) : std::runtime_error(what) {}
};

#define BLUB_CUDA_CHECK(expr)                                                                                          \
    do {                                                                                                               \
        cudaError_t err__ = (expr);                                                                                    \
        if (err__ != cudaSuccess) {                                                                                    \
            throw ::blub::CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(err__) + " (" + __FILE__ +   \
                                    ":" + std::to_string(__LINE__) + ")");                                             \
        }                                                                                                              \
    } while (0)

extern std::atomic<uint64_t> g_kernel_launches;

// SM count of the current device, queried once per device: grids sized "so many blocks per SM" follow the GPU they run on.
inline int device_sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0, n = 0;
    BLUB_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64 && (n = cache[dev].load(std::memory_order_relaxed)) > 0) return n;
    BLUB_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
    return n;
}

// Every kernel launch of the library goes through this macro so that bench.py can report gpu_launches.
#define BLUB_LAUNCH(kernel, grid, block, smem, stream, ...)                                                            \
    do {                                                                                                               \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                                                    \
        ::blub::g_kernel_launches.fetch_add(1, std::memory_order_relaxed);                                             \
        BLUB_CUDA_CHECK(cudaGetLastError());                                                                           \
    } while (0)

// Dense grid in linear x-fastest order.  Every grid array is allocated with `pad` elements of slack on both sides
// (zero-filled for markers) so that +-1 neighbour loads in x, y and z never leave the allocation; a border cell is never
// FLUID (transfer_set_boundary_marker.comp:14-16), hence whatever such a load returns is masked away, which reproduces
// the reference's "out-of-bounds texel fetch returns 0 == SOLID" convention (hybrid_fluid.glsl:20-21).
struct GridDim {
    int nx, ny, nz;
    int sy;      // stride of +1 in y (= nx)
    int sz;      // stride of +1 in z (= nx * ny)
    int64_t n;   // cells
    int64_t pad; // slack elements before/after each array
    // z walls: cells with z <= z_wall_lo or z >= z_wall_hi are SOLID and particles are kept in
    // [z_wall_lo + 1.001, z_wall_hi - 0.001].  Single GPU: 0 and nz-1 (transfer_set_boundary_marker.comp:14-16,
    // advect_particles.comp:137); interior ranks of a z-slab decomposition have no z wall (+-2^20).
    int z_wall_lo, z_wall_hi;
    // z-slab ranks: after the density correction a particle may overhang its slab by at most half a cell (the halo sums
    // cover that); single GPU: +-3e38 (no effect).
    float z_keep_lo, z_keep_hi;
};

inline GridDim make_grid(int nx, int ny, int nz) {
    GridDim g;
    g.nx = nx; g.ny = ny; g.nz = nz;
    g.sy = nx; g.sz = nx * ny;
    g.n = (int64_t)nx * ny * nz;
    g.pad = (((int64_t)nx * ny + 8) + 255) / 256 * 256;
    g.z_wall_lo = 0;
    g.z_wall_hi = nz - 1;
    g.z_keep_lo = -3.0e38f;
    g.z_keep_hi = 3.0e38f;
    return g;
}

// Per-step parameters living in DEVICE memory so that a captured CUDA graph can be replayed with a new dt:
// the host fills a pinned copy and enqueues one small H2D copy in front of every step.
struct StepParams {
    float dt;
    float gravity_dt[3]; // GravityGridSpace * Time.SimulationDelta (transfer_gather_velocity.comp:121)
    float tolerance[2];  // error_tolerance / dt per field (pressure_solver.rs:193-201)
    float inv_dt;
    float gravity[3];       // GravityGridSpace itself (the floating bodies' integrator)
    uint32_t step_count;    // whole steps taken before this one (seeds the source emission)
    float tank_q[9];        // moving tanks, row major: the Coriolis rotation Q of the step (identity at rest; read only by tank_frame_kernel)
    float tank_k[9];        //   the position-dependent velocity increment K (zero at rest)
    float tank_pivot[3];    //   the frame's pivot, grid cells
    uint32_t num_particles; // last: left alone by the upload when the count lives on the device
};

// Scalars of one PCG solve (the reference's 64-byte ReduceResultAndMainDispatchBuffer, pressure_init.comp:8-15).
struct PcgScalars {
    float alpha;          // sigma / (s.As +- eps)            pressure_reduce.comp:73-75
    float beta;           // sigma' / (sigma +- eps)          pressure_reduce.comp:77-80
    float sigma;          // z.r
    float max_error;      // statistics                       pressure_reduce.comp:86
    int num_iterations;   // statistics; 0 == "no stats yet"  pressure_reduce.comp:84-87
    int done;             // replaces zeroing the indirect dispatch arguments (pressure_reduce.comp:89-92)
    unsigned int ticket;  // last-block-done counter of the grid-wide reductions
    int pad_;
};

// z-slab sharding of the pressure solve (SURVEY.md section 8e; the reference is single-GPU).  Every rank owns `owned_nz` planes
// of the global grid and keeps SLAB_HALO ghost planes on both sides; local plane SLAB_HALO is the first owned one.
// Ghost planes of r and p are written by the NEIGHBOUR's kernels (P2P stores into this rank's memory over NVLink);
// scalars are all-reduced through per-rank mailboxes that every peer writes into directly.
constexpr int SLAB_HALO = 4;  // == PCG_TZ: owned planes start on a tile boundary
constexpr int SLAB_MAX_WORLD = 8;
struct SlabComm {
    int rank = 0, world = 1;
    int halo = 0;                 // 0 = not sharded
    int owned_nz = 0;
    unsigned long long *mailbox[SLAB_MAX_WORLD] = {}; // mailbox[k] = rank k's mailbox as mapped here (own one included)
    float *peer_r[2] = {nullptr, nullptr};            // residual volume of the lower / upper neighbour (cell 0), or null
    float *peer_p[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}}; // [field][lower/upper]
    unsigned int *seq = nullptr;  // device counter of all-reduce rounds done so far (identical on every rank)
};

// One mailbox round: round `seq` uses slot seq & 1.  Rank k stores {value bits, seq} as ONE 64-bit word per value, two values, into
// entry k of every rank's mailbox (P2P store over NVLink), then polls entry j of its OWN mailbox for every rank j until it carries `seq`.
// Two slots suffice: a rank can only be one round ahead of the slowest one, because finishing round n needs everybody's n-th message.
// The PCG all-reduces (pcg.cu) and the stream-ordered slab barrier (slab.cu) share the slots and the round counter SlabComm::seq.
constexpr long long MAILBOX_SPIN_LIMIT = 40LL * 1000 * 1000; // ~10 s: a dead peer ends the round with an error instead of hanging the GPU
__device__ __forceinline__ unsigned long long *mailbox_entry(unsigned long long *mailbox, unsigned seq, int rank) {
    return mailbox + (int)(seq & 1u) * 2 * SLAB_MAX_WORLD + 2 * rank;
}
// The system-scope fence first publishes everything this GPU wrote before (what other blocks wrote: as far as the caller has ordered it
// before this thread, by a grid barrier or an arrival counter).
__device__ __forceinline__ void mailbox_post(unsigned long long *entry, unsigned seq, unsigned v0, unsigned v1) {
    __threadfence_system();
    volatile unsigned long long *dst = entry;
    dst[0] = ((unsigned long long)seq << 32) | (unsigned long long)v0;
    dst[1] = ((unsigned long long)seq << 32) | (unsigned long long)v1;
}
// Spins until both words of `entry` carry `seq`, at most spin_limit times, and at least once but no longer once the block's dead flag is
// set; sets the flag when the words never came.  v0 / v1: the words last read.  The system-scope fence after it is the acquire of what the
// peers wrote before their posts.
__device__ __forceinline__ void mailbox_poll(const unsigned long long *entry, unsigned seq, long long spin_limit, int *dead, unsigned long long &v0,
                                             unsigned long long &v1) {
    const volatile unsigned long long *src = entry;
    long long spins = 0;
    bool ok = false;
    while (!*dead || spins == 0) {
        v0 = src[0];
        v1 = src[1];
        if ((unsigned)(v0 >> 32) == seq && (unsigned)(v1 >> 32) == seq) { ok = true; break; }
        if (++spins > spin_limit) break;
    }
    if (!ok) *dead = 1;
    __threadfence_system();
}

// A particle on its way to the neighbouring slab: 64 B.
struct MigrantRecord {
    float4 pos, rx, ry, rz;
};
// Where the advection kernel of a slab rank puts its results: stayers are compacted into the spare arrays, leavers go
// straight into the neighbour's receive buffer (P2P stores), z re-based by -+zshift.  counters: [0] stay, [1] down, [2] up,
// [3] overflow flag.
struct MigrateOut {
    float4 *pos, *rx, *ry, *rz;
    MigrantRecord *peer_down, *peer_up;
    unsigned int *counters;
    float z_lo, z_hi, zshift;
    unsigned int capacity;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float saturatef(float x) { return __saturatef(x); }

// Accumulators of the scatter kernels: 64-bit fixed point.  Integer additions are associative, so a sum does not depend on the order in
// which the atomics arrive: the same input gives the same step, bit for bit, run after run.  Sums of w * value carry 36 fractional bits
// (range +-2^27), sums of weights 40 (range +-2^23); a contribution is rounded to 2^-36 / 2^-40, far below float resolution for the
// weights that matter (a face with a total weight of 1e-6 keeps a relative precision of 1e-6).
constexpr int FIXED_VALUE_BITS = 36, FIXED_WEIGHT_BITS = 40;
template <int FRAC> __device__ __forceinline__ long long to_fixed(float v) { return __float2ll_rn(v * (float)(1ull << FRAC)); }
template <int FRAC> __device__ __forceinline__ double from_fixed(long long a) { return (double)a / (double)(1ull << FRAC); }
__device__ __forceinline__ void fixed_add(long long *dst, long long v) {
    atomicAdd(reinterpret_cast<unsigned long long *>(dst), (unsigned long long)v); // two's complement: signed sums come out right
}

// RGBA16F solid voxel texel: xyz = velocity in cells/s, w != 0 => solid (src/scene/voxelization.rs:17)
struct Voxel {
    float x, y, z, w;
};
__device__ __forceinline__ Voxel load_voxel(const uint2 *__restrict__ vox, int64_t i) {
    Voxel v;
    if (vox == nullptr) {
        v.x = v.y = v.z = v.w = 0.0f;
        return v;
    }
    uint2 raw = __ldg(vox + i);
    __half2 a = *reinterpret_cast<__half2 *>(&raw.x), b = *reinterpret_cast<__half2 *>(&raw.y);
    float2 fa = __half22float2(a), fb = __half22float2(b);
    v.x = fa.x; v.y = fa.y; v.z = fb.x; v.w = fb.y;
    return v;
}

} // namespace blub
