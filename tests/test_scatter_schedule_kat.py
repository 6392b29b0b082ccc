"""The brick schedule of the density scatter (launch_scatter_schedule, transfer_kernels.cu), restated in NumPy (tools/red_stats.py): what the
build produces from the cell lists of a re-sort, and the design argument for it -- on the oracle's dam break the scheduled scatter issues
far fewer global reductions than the 256-particle chunks at every step of a sort window."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools"))
import red_stats as R  # noqa: E402


def _cell_start(cells, dims):
    nx, ny, nz = dims
    lin = cells[:, 0] + nx * (cells[:, 1] + ny * cells[:, 2])
    assert (np.diff(lin) >= 0).all()
    return np.searchsorted(lin, np.arange(nx * ny * nz + 1), side="left")


def test_hand_built_schedule():
    # 8 x 2 x 1 cells, bricks of 4 x 2 x 1 (brick 0: x 0..3, brick 1: x 4..7).  Sorted particles: 0..39 in cell (1, 0), 40..99 in (5, 0),
    # 100..129 in (0, 1).  The first particles of warps 0..4 are 0, 32, 64, 96, 128: cells (1, 0), (1, 0), (5, 0), (5, 0), (0, 1).
    dims = (8, 2, 1)
    cells = np.array([[1, 0, 0]] * 40 + [[5, 0, 0]] * 60 + [[0, 1, 0]] * 30)
    bw, bi, start, brick, warps = R.brick_schedule(_cell_start(cells, dims), dims, brick=(4, 2, 1), k=2)
    assert list(warps) == [0, 1, 4, 2, 3]  # brick 0 row y = 0, then its row y = 1; then brick 1
    assert list(bw) == [0, 3, 5] and list(bi) == [0, 2, 3]
    assert list(start) == [0, 2, 3] and list(brick) == [0, 0, 1]
    bw, bi, start, brick, warps = R.brick_schedule(_cell_start(cells, dims), dims, brick=(4, 2, 1), k=1)
    assert list(start) == [0, 1, 2, 3, 4] and list(brick) == [0, 0, 0, 1, 1]


def _dam_sorted():
    from oracle import oracle as O
    from tests import util

    f = util.oracle_from_scene("dam_small")
    f.set_rebin_frequency(0)
    d = O.load_scene(util.scene_path("dam_small"))["fluid"]["grid_dimension"]
    return f, (d["x"], d["y"], d["z"]), util.DT


def test_schedule_covers_every_warp_once_in_brick_order():
    f, dims, dt = _dam_sorted()
    nx, ny, nz = dims
    for _ in range(12):
        f.step(dt)
    p = f.particles()[:, :3].copy()
    p = p[R.sort_by_primal_cell(p, np.arange(len(p)), nx, ny)]
    cells = p.astype(np.int64)
    bw, bi, start, brick, warps = R.brick_schedule(_cell_start(cells, dims), dims)
    nwarps = (len(p) + 31) // 32
    assert np.array_equal(np.sort(warps), np.arange(nwarps))  # every warp once
    assert bw[-1] == nwarps and bi[-1] == len(start) == len(brick)
    nbx, nby = -(-nx // R.BRICK[0]), -(-ny // R.BRICK[1])
    first = cells[32 * warps]
    own = first[:, 0] // R.BRICK[0] + nbx * (first[:, 1] // R.BRICK[1] + nby * (first[:, 2] // R.BRICK[2]))
    of_brick = np.repeat(np.arange(len(bw) - 1), np.diff(bw))
    assert np.array_equal(own, of_brick)  # a warp belongs to the brick of its first particle's cell
    assert all((np.diff(warps[bw[b]:bw[b + 1]]) > 0).all() for b in range(len(bw) - 1))  # ascending inside a brick
    sizes = np.diff(np.append(start, len(warps)))
    assert sizes.min() >= 1 and sizes.max() <= R.SCHED_K
    assert np.array_equal(np.bincount(brick, minlength=len(bw) - 1), np.diff(bi))
    assert np.array_equal(start[bi[brick] == np.arange(len(start))], bw[brick[bi[brick] == np.arange(len(start))]])  # an item starts its brick's list


def test_schedule_cuts_the_density_reductions_at_every_step_of_a_sort_window():
    """16 steps of the oracle's dam break, re-sorted every 8 (the CUDA path's cadence): the work items' windows, set from the particles' cells
    at the time of the scatter, keep the global reductions of the density scatter at most 55 % of the chunks' (0.34-0.40 against 0.78-0.93
    per particle when this was written)."""
    f, dims, dt = _dam_sorted()
    nx, ny, nz = dims
    order = np.arange(f.num_particles)
    for step in range(16):
        p = f.particles()[:, :3].copy()
        if step % 8 == 0:
            order = R.sort_by_primal_cell(p, order, nx, ny)
            sorted_p = p[order].copy()
        chunks = R.tiled_global_reductions(p[order], nx, ny, 256, 2048, comps=(3,))[0]
        scheduled = R.scheduled_global_reductions(p[order], sorted_p, nx, ny, nz)[0]
        assert scheduled <= 0.55 * chunks, (step, scheduled, chunks)
        f.step(dt)
