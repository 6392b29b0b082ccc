"""How many reductions (RED lane-ops) does the P2G / density scatter issue per particle under each warp aggregation scheme?

Pure NumPy on particle positions in ARRAY ORDER (no GPU, no oracle import: positions come from a file or from the caller --
tests/test_variants_emulated.py feeds positions of the CPU oracle's dam break, re-sorted by primal cell every 8 steps as the CUDA path does).

    python tools/red_stats.py snapshots.npz NX NY        # arrays of shape [n, 3] (grid units), one line per array

Schemes: none = one reduction per (particle, face); adjacent4 = runs of adjacent lanes with the same dual cell, cut into groups of four
(segmented_run_sum); match4 / match8 / matchall = all lanes of the warp with the same dual cell (matched_group_sum), groups of 4 / 8 / any size.
tiled_global_reductions: what is left of the match4 reductions for the global volumes once a block adds a chunk's faces up in a
shared-memory tile first (p2g_scatter_kernel / density_scatter_kernel); scheduled_global_reductions: the same for the density scatter's
brick schedule (work items of warps grouped by the cell brick they were sorted into).
"""
import sys

import numpy as np


def dual_keys(p, c, nx, ny):
    """dual cell of component c (0..2: velocity components, transfer_build_linkedlist.comp:21-23; 3: density, offset 0.5 everywhere)"""
    off = np.full(3, 0.5, np.float32)
    if c < 3:
        off[c] = 1.0
    d = (p.astype(np.float32) - off).astype(np.int32)
    return d[:, 0] + nx * (d[:, 1] + ny * d[:, 2])


def reductions_per_particle(p, nx, ny, comps=(0, 1, 2)):
    """p: [n, 3] positions in array order.  Returns {scheme: reductions per particle} summed over `comps` (8 faces per issuing lane)."""
    m = len(p) // 32 * 32
    idx = np.arange(32)[None, :]
    tot = dict(none=0, adjacent4=0, match4=0, match8=0, matchall=0)
    for c in comps:
        k = dual_keys(p[:m], c, nx, ny).reshape(-1, 32)
        start = np.ones_like(k, bool)
        start[:, 1:] = k[:, 1:] != k[:, :-1]
        pos = idx - np.maximum.accumulate(np.where(start, idx, 0), axis=1)           # position inside the adjacent run
        ks = np.sort(k, axis=1)                                                      # rank among ALL equal keys of the warp
        st = np.ones_like(ks, bool)
        st[:, 1:] = ks[:, 1:] != ks[:, :-1]
        r = idx - np.maximum.accumulate(np.where(st, idx, 0), axis=1)
        tot["none"] += k.size
        tot["adjacent4"] += int(((pos & 3) == 0).sum())
        tot["match4"] += int(((r & 3) == 0).sum())
        tot["match8"] += int(((r & 7) == 0).sum())
        tot["matchall"] += int(st.sum())
    return {a: 8.0 * b / m for a, b in tot.items()}


def chunk_windows(cells, cap):
    """The tile window of every chunk, as p2g_scatter_kernel / density_scatter_kernel pick it (scatter_window in transfer_kernels.cu).
    cells: [chunks, ch, 3] primal cells (x, y, z) of the chunk's particles, -1 for slots past the last particle.  The box covers the faces
    [min - 1, max + 1] of the chunk's cells in every dimension; a box larger than `cap` faces is cut, z first, then y (neither below 3), then x,
    around the cell of the chunk's middle particle.  Returns (origin, extent), [chunks, 3] each."""
    valid = cells[:, :, 0] >= 0
    n = valid.sum(axis=1)
    big = np.iinfo(np.int64).max
    mn = np.where(valid[:, :, None], cells, big).min(axis=1)
    mx = np.where(valid[:, :, None], cells, -1).max(axis=1)
    anchor = cells[np.arange(len(cells)), n // 2]
    lo, hi = mn - 1, mx + 1
    e = hi - lo + 1
    ex, ey, ez = e[:, 0].copy(), e[:, 1].copy(), e[:, 2].copy()
    ez = np.minimum(ez, np.maximum(3, cap // (ex * ey)))
    ey = np.minimum(ey, np.maximum(3, cap // (ex * ez)))
    ex = np.minimum(ex, cap // (ey * ez))
    ext = np.stack([ex, ey, ez], axis=1)
    origin = np.clip(anchor - ext // 2, lo, hi - ext + 1)
    return origin, ext


def tiled_global_reductions(p, nx, ny, ch, cap, comps=(0, 1, 2)):
    """Global 64-bit reductions per particle of the tiled scatter: chunks of `ch` consecutive particles share a block-private tile of at most
    `cap` faces (chunk_windows).  A peer-group head (match4) adds a face that lies inside its chunk's window into the tile, any other face
    straight into the global volume; after the chunk every touched tile entry is flushed by one global reduction per word.  Words per face:
    2 for the velocity components (sum w * value, sum w), 1 for the density.  Returns (total, of which flushes, of which outside the window)."""
    m = len(p) // 32 * 32
    nchunk = (m + ch - 1) // ch
    lo = 0.5 if comps == (3,) else 1.0
    q = np.maximum(p[:m].astype(np.float32), np.float32(lo))  # simulated particles never reach the upper clamp plane
    cells = np.full((nchunk * ch, 3), -1, np.int64)
    cells[:m] = q.astype(np.int64)
    origin, ext = chunk_windows(cells.reshape(nchunk, ch, 3), cap)
    return _unit_global_reductions(p, q, nx, ny, np.arange(m) // ch, origin, ext, comps)


# Brick schedule of the scatters (launch_scatter_schedule in transfer_kernels.cu): bricks of BRICK cells, work items of at most
# SCHED_K warps.
BRICK, SCHED_K = (28, 4, 4), 64


def brick_schedule(cell_start, dims, brick=BRICK, k=SCHED_K):
    """Restatement of the schedule build from the cell lists of a re-sort (cell_start: [n + 1], the particles of cell c are the sorted
    indices cell_start[c] .. cell_start[c + 1]).  A warp w (particles 32w .. 32w + 31) belongs to the brick of its first particle's cell;
    brick b = (bz * nby + by) * nbx + bx lists its warps in ascending order, cut into work items of at most k.  Returns the device arrays:
    brick_warps and brick_items ([nbricks + 1], exclusive scans of the per-brick counts), item_start, item_brick, warps."""
    nx, ny, nz = dims
    bx, by, bz = brick
    nbx, nby, nbz = -(-nx // bx), -(-ny // by), -(-nz // bz)
    cs = (np.asarray(cell_start, np.int64) + 31) // 32  # warps whose first particle lies before each cell boundary
    counts, items, item_start, item_brick, warps = [], [], [], [], []
    for b in range(nbx * nby * nbz):
        x0, y0, z0 = b % nbx * bx, b // nbx % nby * by, b // nbx // nby * bz
        ws = []
        for z in range(z0, min(z0 + bz, nz)):
            for y in range(y0, min(y0 + by, ny)):
                c0 = (z * ny + y) * nx + x0
                ws.extend(range(cs[c0], cs[c0 + min(bx, nx - x0)]))
        counts.append(len(ws))
        items.append(-(-len(ws) // k))
        item_start.extend(len(warps) + j for j in range(0, len(ws), k))
        item_brick.extend([b] * items[-1])
        warps.extend(ws)
    scan = lambda a: np.concatenate([[0], np.cumsum(a)]).astype(np.int64)
    return scan(counts), scan(items), np.array(item_start, np.int64), np.array(item_brick, np.int64), np.array(warps, np.int64)


def item_windows(cells, item_brick, dims, cap, brick=BRICK):
    """The tile window of every work item as density_scatter_kernel picks it (item_window): cells [items, L, 3] the primal cells of the item's
    particles NOW (-1 past its last particle).  The faces [min - 1, max + 1] of those cells, cut z first, then y (neither below the brick's
    rows + 2), then x, around the middle of the item's brick."""
    nx, ny, nz = dims
    bx, by, bz = brick
    nbx, nby = -(-nx // bx), -(-ny // by)
    valid = cells[:, :, 0] >= 0
    big = np.iinfo(np.int64).max // 4
    lo = np.where(valid[:, :, None], cells, big).min(axis=1) - 1
    hi = np.where(valid[:, :, None], cells, -big).max(axis=1) + 1
    e = hi - lo + 1
    ex, ey, ez = e[:, 0].copy(), e[:, 1].copy(), e[:, 2].copy()
    ez = np.minimum(ez, np.maximum(bz + 2, cap // (ex * ey)))
    ey = np.minimum(ey, np.maximum(by + 2, cap // (ex * ez)))
    ex = np.minimum(ex, cap // (ey * ez))
    ext = np.stack([ex, ey, ez], axis=1)
    b = np.asarray(item_brick)
    mid = np.stack([b % nbx * bx + bx // 2, b // nbx % nby * by + by // 2, b // nbx // nby * bz + bz // 2], axis=1)
    origin = np.minimum(np.maximum(mid - ext // 2, lo), hi - ext + 1)
    return origin, ext


def scheduled_global_reductions(p, sort_p, nx, ny, nz, cap=2048, comps=(3,)):
    """tiled_global_reductions of the scheduled density scatter: p [n, 3] the positions scattered, sort_p the positions of the same array at
    its last re-sort (sort_by_primal_cell order then).  The work items of brick_schedule share a tile; their windows come from p."""
    m = len(p) // 32 * 32
    cells = sort_p.astype(np.int64)
    lin = cells[:, 0] + nx * (cells[:, 1] + ny * cells[:, 2])
    assert (np.diff(lin) >= 0).all(), "sort_p must be in primal-cell order"
    cell_start = np.searchsorted(lin, np.arange(nx * ny * nz + 1), side="left")
    _, _, item_start, item_brick, warps = brick_schedule(cell_start, (nx, ny, nz))
    item_of_warp = np.repeat(np.arange(len(item_start)), np.diff(np.append(item_start, len(warps))))
    unit = np.empty(len(warps), np.int64)
    unit[warps] = item_of_warp
    unit = unit[np.arange(m) // 32]
    lo = 0.5 if comps == (3,) else 1.0
    q = np.maximum(p[:m].astype(np.float32), np.float32(lo))
    c = q.astype(np.int64)
    order = np.argsort(unit, kind="stable")
    counts = np.bincount(unit, minlength=len(item_start))
    pad = np.full((len(item_start), max(int(counts.max()), 1), 3), -1, np.int64)
    slot = np.arange(m) - np.repeat(np.concatenate([[0], np.cumsum(counts)[:-1]]), counts)
    pad[unit[order], slot] = c[order]
    origin, ext = item_windows(pad, item_brick, (nx, ny, nz), cap)
    return _unit_global_reductions(p, q, nx, ny, unit, origin, ext, comps)


def _unit_global_reductions(p, q, nx, ny, unit, origin, ext, comps):
    """unit[i]: the tile (chunk or work item) of particle i; origin / ext: the windows of the units"""
    nz_max = int(p[:, 2].max()) + 2
    m = len(q)
    chunk = unit
    words = 1 if comps == (3,) else 2
    outside = flushed = 0
    idx = np.arange(32)[None, :]
    for c in comps:
        off = np.full(3, 0.5, np.float32)
        if c < 3:
            off[c] = 1.0
        d = (q - off).astype(np.int64)
        k = (d[:, 0] + nx * (d[:, 1] + ny * d[:, 2])).reshape(-1, 32)
        ks, perm = np.sort(k, axis=1), np.argsort(k, axis=1, kind="stable")
        st = np.ones_like(ks, bool)
        st[:, 1:] = ks[:, 1:] != ks[:, :-1]
        r = idx - np.maximum.accumulate(np.where(st, idx, 0), axis=1)
        head = np.zeros_like(k, bool)
        np.put_along_axis(head, perm, (r & 3) == 0, axis=1)
        h = np.flatnonzero(head.reshape(-1))
        keys = []
        for o in range(8):
            f = d[h] + np.array([o & 1, (o >> 1) & 1, o >> 2])
            rel = f - origin[chunk[h]]
            inside = ((rel >= 0) & (rel < ext[chunk[h]])).all(axis=1)
            outside += int((~inside).sum()) * words
            keys.append((chunk[h][inside] * nz_max + f[inside, 2]) * ny * nx + f[inside, 1] * nx + f[inside, 0])
        flushed += len(np.unique(np.concatenate(keys))) * words
    return (outside + flushed) / m, flushed / m, outside / m


def sort_by_primal_cell(p, order, nx, ny):
    """the stable counting sort of the binning stage: x-fastest cell order, ascending previous index inside a cell"""
    ci = p.astype(np.int32)
    cell = ci[:, 0] + nx * (ci[:, 1] + ny * ci[:, 2])
    return order[np.argsort(cell[order], kind="stable")]


if __name__ == "__main__":
    data, nx, ny = np.load(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    for key in data.files:
        v, d = reductions_per_particle(data[key], nx, ny), reductions_per_particle(data[key], nx, ny, comps=(3,))
        print(key, "P2G", " ".join(f"{a} {b:.2f}" for a, b in v.items()), "| density", " ".join(f"{a} {b:.2f}" for a, b in d.items()))
        # the kernels' chunk and tile sizes (PT, P2G_TILE, DENSITY_TILE in transfer_kernels.cu)
        tv, td = tiled_global_reductions(data[key], nx, ny, 256, 1184), tiled_global_reductions(data[key], nx, ny, 256, 2048, comps=(3,))
        print(key, "tiled global reductions per particle: P2G %.2f (flush %.2f + outside %.2f) | density %.2f (flush %.2f + outside %.2f)" % (tv + td))
