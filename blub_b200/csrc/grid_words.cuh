// grid_words.cuh -- the shape of the grid passes (fluid_kernels.cu, viscosity_kernels.cu): one thread per 32-cell word of the FLUID bit mask,
// the warp walks the words that have something to do.
#pragma once
#include "fluid_kernels.hpp"

namespace blub {
namespace {

constexpr int PT = 256; // threads per block for particle and cell kernels

// Cell indices fit 32 bits (HybridFluid::new rejects grids of 2^31 cells or more): no 64-bit multiplies / divisions in the
// per-cell and per-particle kernels.
__device__ __forceinline__ int lin(const GridDim &g, int x, int y, int z) { return (z * g.ny + y) * g.nx + x; }

// All grid passes work on the 1-bit-per-cell FLUID mask (FluidBits, rebuilt with every finished marker volume): one thread per 32-cell
// word of a row decides from a handful of mask words whether any of its cells has anything to do (in a dam break ~85 % of the words
// have not), then the WARP walks the words that have, lane = cell, so that the loads and stores of a word are coalesced.  Cells that
// are more than one cell away from every FLUID cell are not visited at all: the reference's full-grid passes write 0 there, and no
// particle in a FLUID cell reads them (the extrapolation fills the one-cell ring G2P can reach).  With a solid volume a particle can sit
// in a SOLID cell: an eaten one is moved one cell before G2P and reads faces up to two cells from its own, one left in a solid by the
// advection's push reads faces one cell from its own in the correction.  So the projection also visits the cells within two cells of a
// SOLID cell that holds a particle, the position change those within one (near_stray_word), and writes there what the reference writes.
__device__ __forceinline__ unsigned fbits(const GridDim &g, const FluidBits &b, int xw, int y, int z) {
    if (xw < 0 || xw >= b.wpr || y < 0 || y >= g.ny || z < 0 || z >= g.nz) return 0u;
    return __ldg(b.words + (z * g.ny + y) * b.wpr + xw);
}
struct WordPos {
    int xw, y, z, cells;
    bool inside;
};
__device__ __forceinline__ WordPos word_of_thread(const GridDim &g, const FluidBits &b) {
    const int w = blockIdx.x * PT + threadIdx.x;
    WordPos p;
    p.inside = w < b.wpr * g.ny * g.nz;
    p.xw = p.inside ? w % b.wpr : 0;
    const int rowi = p.inside ? w / b.wpr : 0;
    p.y = rowi % g.ny;
    p.z = rowi / g.ny;
    p.cells = min(32, g.nx - p.xw * 32);
    return p;
}
__device__ __forceinline__ unsigned cells_mask(const WordPos &p) { return p.cells == 32 ? 0xffffffffu : ((1u << p.cells) - 1u); }
// FLUID cells of the word dilated by one cell in every dimension
__device__ __forceinline__ unsigned near_fluid_word(const GridDim &g, const FluidBits &b, const WordPos &p) {
    unsigned near = 0;
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const unsigned f = fbits(g, b, p.xw, p.y + dy, p.z + dz);
            near |= f | (f << 1) | (f >> 1) | (fbits(g, b, p.xw - 1, p.y + dy, p.z + dz) >> 31) | (fbits(g, b, p.xw + 1, p.y + dy, p.z + dz) << 31);
        }
    return near & cells_mask(p);
}
// SOLID cells that hold a particle (particle words of the last marker pass minus the FLUID bits), dilated by R cells in every dimension
__device__ __forceinline__ unsigned stray_bits(const GridDim &g, const FluidBits &b, const uint32_t *__restrict__ pw, int xw, int y, int z) {
    if (xw < 0 || xw >= b.wpr || y < 0 || y >= g.ny || z < 0 || z >= g.nz) return 0u;
    const int w = (z * g.ny + y) * b.wpr + xw;
    return __ldg(pw + w) & ~__ldg(b.words + w);
}
template <int R>
__device__ __forceinline__ unsigned near_stray_word(const GridDim &g, const FluidBits &b, const uint32_t *__restrict__ pw, const WordPos &p) {
    unsigned near = 0;
#pragma unroll
    for (int dz = -R; dz <= R; ++dz)
#pragma unroll
        for (int dy = -R; dy <= R; ++dy) {
            const unsigned s = stray_bits(g, b, pw, p.xw, p.y + dy, p.z + dz);
            const unsigned l = stray_bits(g, b, pw, p.xw - 1, p.y + dy, p.z + dz), r = stray_bits(g, b, pw, p.xw + 1, p.y + dy, p.z + dz);
            near |= s;
#pragma unroll
            for (int k = 1; k <= R; ++k) near |= (s << k) | (s >> k) | (l >> (32 - k)) | (r << (32 - k));
        }
    return near & cells_mask(p);
}
// The warp walks the words whose `todo` mask is not empty; body(cell index, x, y, z, lane of the word's owner) runs with lane = cell on the
// set bits.  All 32 lanes of the warp must call this.
template <class Body>
__device__ __forceinline__ void warp_walk(const GridDim &g, unsigned todo, const WordPos &p, Body &&body) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    unsigned words = __ballot_sync(full, todo != 0u);
    while (words) {
        const int src = __ffs(words) - 1;
        words &= words - 1;
        const unsigned tw = __shfl_sync(full, todo, src);
        const int xw = __shfl_sync(full, p.xw, src), y = __shfl_sync(full, p.y, src), z = __shfl_sync(full, p.z, src);
        body((tw >> lane) & 1u, xw * 32 + lane, y, z, src);
    }
}

} // namespace
} // namespace blub
