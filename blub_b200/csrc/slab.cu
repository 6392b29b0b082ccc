// slab.cu -- z-slab sharding of the WHOLE step across GPUs (SURVEY.md section 8e; the reference is single-GPU).
//
// Rank k owns the global planes [k*zs, (k+1)*zs); its local grid carries SLAB_HALO ghost planes on both sides and all
// stage kernels run unchanged on that local grid.  What crosses the slab faces, per step:
//   X1  after the P2G scatter      SUM of the (num, weight) accumulators and MAX of the markers over the 4 planes around
//                                  each face (both ranks send their partials of the same 4 global planes and add)
//   PCG                            boundary planes of r / p pushed from inside the persistent kernel (pcg.cu)
//   X2  after extrapolation        COPY of the first two owned planes of u into the neighbour's ghost planes
//   MIG inside the advection       the advection kernel itself compacts the stayers and writes the leavers into the
//                                  neighbour's buffer (positions re-based by +-zs); counts + arrivals are appended afterwards
//   X3  after advection            MAX of the markers
//   X4  after the density scatter  SUM of the density accumulator
//   X5  after extrapolation #2     COPY of the displacement field planes
// Transport: stream-ordered cudaMemcpyAsync straight into the neighbour's (double-buffered) receive area inside its
// peer-visible window, one mailbox barrier kernel per exchange, then a local combine kernel.  No host synchronisation,
// no NCCL.  Particles keep their owner until they cross a face; up to half a cell of overhang (density correction) is
// tolerated by the 4-plane overlap.
#include <cstring>

#include "blub_core.hpp"
#include "fluid_kernels.hpp"

namespace blub {
namespace {

// one empty mailbox round (common.cuh): stream-ordered barrier; a peer that never answers sets the error flag, and the round still counts
__global__ void slab_barrier_kernel(SlabComm c, int *error_flag) {
    __shared__ int dead;
    const int tid = threadIdx.x;
    if (tid == 0) dead = 0;
    __syncthreads();
    const unsigned seq = *c.seq + 1u;
    if (tid < c.world) {
        mailbox_post(mailbox_entry(c.mailbox[tid], seq, c.rank), seq, 0u, 0u);
        unsigned long long v0, v1;
        mailbox_poll(mailbox_entry(c.mailbox[c.rank], seq, tid), seq, MAILBOX_SPIN_LIMIT, &dead, v0, v1);
    }
    __syncthreads();
    if (tid == 0) {
        *c.seq = seq;
        if (dead && error_flag) *error_flag = 1;
    }
}

__global__ void __launch_bounds__(256) halo_add_kernel(long long *__restrict__ dst, const long long *__restrict__ src, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) dst[i] += src[i];
}
__global__ void __launch_bounds__(256) halo_max_kernel(int8_t *__restrict__ dst, const int8_t *__restrict__ src, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) dst[i] = max(dst[i], src[i]);
}

// publish how many particles were sent (into the neighbours' windows) and start the new local count
__global__ void migrate_publish_kernel(unsigned int *counters, unsigned int *peer_count_down, unsigned int *peer_count_up, unsigned int capacity) {
    if (threadIdx.x != 0) return;
    if (peer_count_down) *peer_count_down = min(counters[1], capacity);
    if (peer_count_up) *peer_count_up = min(counters[2], capacity);
    __threadfence_system();
}

__global__ void __launch_bounds__(256) migrate_append_kernel(const MigrantRecord *__restrict__ recv_lo, const MigrantRecord *__restrict__ recv_hi,
                                                             const unsigned int *__restrict__ recv_counts, const unsigned int *__restrict__ counters,
                                                             float4 *__restrict__ opos, float4 *__restrict__ orx, float4 *__restrict__ ory,
                                                             float4 *__restrict__ orz, unsigned int max_particles) {
    const unsigned n_lo = recv_counts[0], n_hi = recv_counts[1], stay = counters[0];
    const unsigned i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n_lo + n_hi) return;
    const MigrantRecord rec = i < n_lo ? recv_lo[i] : recv_hi[i - n_lo];
    const unsigned dst = stay + i;
    if (dst >= max_particles) return;
    opos[dst] = rec.pos;
    orx[dst] = rec.rx;
    ory[dst] = rec.ry;
    orz[dst] = rec.rz;
}

__global__ void migrate_finish_kernel(StepParams *params, unsigned int *counters, unsigned int *recv_counts, unsigned int max_particles, int *error_flag) {
    if (threadIdx.x != 0) return;
    unsigned n = counters[0] + recv_counts[0] + recv_counts[1];
    if (n > max_particles) {
        n = max_particles;
        if (error_flag) *error_flag = 2;
    }
    if (counters[3] && error_flag) *error_flag = 3;
    params->num_particles = n;
    counters[0] = counters[1] = counters[2] = counters[3] = 0;
    recv_counts[0] = recv_counts[1] = 0;
}

inline int blocks_for(int64_t n, int per) { return (int)((n + per - 1) / per); }

} // namespace

// ---------------------------------------------------------------------------------------------------------------
size_t HybridFluid::slab_extra_window_bytes() const {
    const size_t cols = (size_t)grid_.nx * grid_.ny;
    const size_t halo = (cols * 196 + 255) / 256 * 256;                              // 3 x longlong2 x 4 planes + marker x 4 planes
    const size_t part = ((size_t)slab_migrant_capacity() * sizeof(MigrantRecord) + 255) / 256 * 256;
    return 4 * halo + 2 * part + 256;
}

uint32_t HybridFluid::slab_migrant_capacity() const { return (uint32_t)grid_.nx * grid_.ny * 8u * 3u; } // three planes' worth

void HybridFluid::slab_layout(void *window, char *&halo0, size_t &halo_bytes, char *&part0, size_t &part_bytes, unsigned int *&counts) const {
    const size_t vol = GridArray<float>::bytes_for(grid_);
    const size_t cols = (size_t)grid_.nx * grid_.ny;
    halo_bytes = (cols * 196 + 255) / 256 * 256;
    part_bytes = ((size_t)slab_migrant_capacity() * sizeof(MigrantRecord) + 255) / 256 * 256;
    char *w = static_cast<char *>(window) + 4096 + 3 * vol;
    halo0 = w;
    part0 = w + 4 * halo_bytes;
    counts = reinterpret_cast<unsigned int *>(part0 + 2 * part_bytes);
}

void HybridFluid::slab_barrier() {
    BLUB_LAUNCH(slab_barrier_kernel, 1, 32, 0, stream_, solver_->comm, slab_error_);
}

// items: {cell-0 pointer, bytes per cell}.  kind 0: SUM over the 4 overlap planes (float data), 1: MAX (int8), 2: COPY of the
// two outermost owned planes into the neighbour's two innermost ghost planes.
void HybridFluid::slab_halo_exchange(const SlabHaloItem *items, int n_items) {
    const SlabComm &c = solver_->comm;
    if (c.world <= 1) return;
    const int H = SLAB_HALO, zs = c.owned_nz;
    const size_t plane_cells = (size_t)grid_.nx * grid_.ny;
    const int buf = (int)(slab_exchange_index_++ & 1u);
    char *halo0;
    size_t hb, pb;
    char *part0;
    unsigned int *counts;
    slab_layout(window_, halo0, hb, part0, pb, counts);
    // receive areas: [face 0 = from the lower neighbour, face 1 = from the upper neighbour][buffer]
    auto local_recv = [&](int face) { return halo0 + (size_t)(face * 2 + buf) * hb; };
    auto peer_recv = [&](int side) -> char * { // my message to the neighbour on `side` lands in ITS area for the opposite face
        if (!slab_peer_window_[side]) return nullptr;
        char *ph0, *pp0;
        size_t phb, ppb;
        unsigned int *pc;
        slab_layout(slab_peer_window_[side], ph0, phb, pp0, ppb, pc);
        return ph0 + (size_t)((1 - side) * 2 + buf) * phb;
    };
    // 1) send
    for (int side = 0; side < 2; ++side) {
        char *dst = peer_recv(side);
        if (!dst) continue;
        size_t off = 0;
        for (int k = 0; k < n_items; ++k) {
            const SlabHaloItem &it = items[k];
            const int planes = it.kind == 2 ? 2 : 4;
            int first;
            if (it.kind == 2) first = side == 0 ? H : H + zs - 2;        // my outermost owned planes
            else first = side == 0 ? H - 2 : H + zs - 2;                 // the 4 planes around the face
            const size_t bytes = (size_t)planes * plane_cells * it.bytes_per_cell;
            const char *src = static_cast<const char *>(it.cell0) + (size_t)first * plane_cells * it.bytes_per_cell;
            BLUB_CUDA_CHECK(cudaMemcpyAsync(dst + off, src, bytes, cudaMemcpyDeviceToDevice, stream_));
            off += (bytes + 255) / 256 * 256;
        }
    }
    // 2) everybody's messages have landed
    slab_barrier();
    // 3) combine
    for (int face = 0; face < 2; ++face) {
        const int nb = slab_rank_ + (face == 0 ? -1 : 1);
        if (nb < 0 || nb >= c.world) continue;
        const char *src = local_recv(face);
        size_t off = 0;
        for (int k = 0; k < n_items; ++k) {
            const SlabHaloItem &it = items[k];
            const int planes = it.kind == 2 ? 2 : 4;
            int first;
            if (it.kind == 2) first = face == 0 ? H - 2 : H + zs;        // my innermost ghost planes
            else first = face == 0 ? H - 2 : H + zs - 2;
            const size_t bytes = (size_t)planes * plane_cells * it.bytes_per_cell;
            char *dst = static_cast<char *>(it.cell0) + (size_t)first * plane_cells * it.bytes_per_cell;
            if (it.kind == 0) {
                const int64_t n = (int64_t)(bytes / sizeof(long long)); // fixed-point sums: exact, the same on both sides of the face
                BLUB_LAUNCH(halo_add_kernel, blocks_for(n, 256), 256, 0, stream_, reinterpret_cast<long long *>(dst), reinterpret_cast<const long long *>(src + off), n);
            } else if (it.kind == 1) {
                BLUB_LAUNCH(halo_max_kernel, blocks_for((int64_t)bytes, 256), 256, 0, stream_, reinterpret_cast<int8_t *>(dst),
                            reinterpret_cast<const int8_t *>(src + off), (int64_t)bytes);
            } else {
                BLUB_CUDA_CHECK(cudaMemcpyAsync(dst, src + off, bytes, cudaMemcpyDeviceToDevice, stream_));
            }
            off += (bytes + 255) / 256 * 256;
        }
    }
}

// Migration.  The advection kernel of a slab rank already sorted its results (advect_kernel<true>): stayers compacted into
// the spare arrays, leavers written into the neighbours' receive buffers.  What is left: publish the counts, wait for
// everybody, append the arrivals, swap the buffers.
MigrateOut HybridFluid::slab_migrate_targets() {
    const SlabComm &c = solver_->comm;
    char *halo0, *part0;
    size_t hb, pb;
    unsigned int *counts;
    slab_layout(window_, halo0, hb, part0, pb, counts);
    MigrateOut m{};
    m.pos = pos_[1 - cur_];
    m.rx = row_alt_[0]; m.ry = row_alt_[1]; m.rz = row_alt_[2];
    for (int side = 0; side < 2; ++side) {
        if (!slab_peer_window_[side]) continue;
        char *ph0, *pp0;
        size_t phb, ppb;
        unsigned int *pc;
        slab_layout(slab_peer_window_[side], ph0, phb, pp0, ppb, pc);
        MigrantRecord *buf = reinterpret_cast<MigrantRecord *>(pp0 + (size_t)(1 - side) * ppb); // lands in its area for the opposite face
        if (side == 0) m.peer_down = buf; else m.peer_up = buf;
    }
    m.counters = mig_counters_;
    m.z_lo = (float)SLAB_HALO;
    m.z_hi = (float)(SLAB_HALO + c.owned_nz);
    m.zshift = (float)c.owned_nz;
    m.capacity = slab_migrant_capacity();
    return m;
}

void HybridFluid::slab_migrate_finish() {
    const SlabComm &c = solver_->comm;
    if (c.world <= 1) return;
    char *halo0, *part0;
    size_t hb, pb;
    unsigned int *counts;
    slab_layout(window_, halo0, hb, part0, pb, counts);
    unsigned int *peer_cnt[2] = {nullptr, nullptr};
    for (int side = 0; side < 2; ++side) {
        if (!slab_peer_window_[side]) continue;
        char *ph0, *pp0;
        size_t phb, ppb;
        unsigned int *pc;
        slab_layout(slab_peer_window_[side], ph0, phb, pp0, ppb, pc);
        peer_cnt[side] = pc + (1 - side);
    }
    const uint32_t cap = slab_migrant_capacity();
    float4 *opos = pos_[1 - cur_];
    BLUB_LAUNCH(migrate_publish_kernel, 1, 32, 0, stream_, mig_counters_, peer_cnt[0], peer_cnt[1], cap);
    slab_barrier();
    BLUB_LAUNCH(migrate_append_kernel, blocks_for(2 * (int64_t)cap, 256), 256, 0, stream_, reinterpret_cast<const MigrantRecord *>(part0),
                reinterpret_cast<const MigrantRecord *>(part0 + pb), counts, mig_counters_, opos, row_alt_[0], row_alt_[1], row_alt_[2], max_num_particles_);
    BLUB_LAUNCH(migrate_finish_kernel, 1, 32, 0, stream_, params_dev_, mig_counters_, counts, max_num_particles_, slab_error_);
    cur_ = 1 - cur_;
    for (int k = 0; k < 3; ++k) std::swap(row_[k], row_alt_[k]);
    row_parity_ ^= 1;
}

} // namespace blub
