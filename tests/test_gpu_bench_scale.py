"""GPU: the workloads bench.py times, stage by stage, against the float64 references of tests/grid_ref.py, at the steps it times.

Each case advances a workload as bench.py does (step(), graph replay, DT_120HZ, default paths and solver; double_dam_box voxelizes its moving
box before every step, bench.SolidStepper's way), then takes one step through step_stages one stage at a time and checks each stage's
downloaded outputs against the reference evaluated on that stage's own downloaded inputs:
  stage 0  the marker on the whole grid exactly; the P2G velocities of the window cores within p2g_bound (scatter form; at dam_256 step 56
           also the gather form, through set_transfer_path(0) for that stage);
  stage 3  the positions: a stable sort by primal cell (clamped to [0, dim - 1]) on a re-sort step; every particle array untouched bit for
           bit otherwise;
  stage 9  the density rhs of the window cores within rhs_bound (scatter form: density_scatter_kernel runs on both paths).
The windows have 32^3-cell cores around the most crowded cell, the brick the schedule cuts into the most work items, the highest-index
FLUID cell, the fluid next to each wall it touches, a sparse free-surface cell and three seeded random FLUID cells.

At these sizes code runs that the small grids never reach, and each case asserts that it did:
  * P2G walks the brick schedule's work items only when there are at least P2G_MIN_ITEM_WAVES x 4 x SMs of them (4224 on 132 SMs): on
    dam_256, tap_256 and basin_512 the items, restated from the cell order the last re-sort left (tools/red_stats.brick_schedule), are at
    least that many, and some item's cell box, restated from the positions the previous step's density scatter saw, is larger than the P2G
    tile (box_window cuts it);
  * a window holds a brick split into two or more items;
  * dam_256 step 56 holds a cell of more than 1024 particles (printed: the maximum per-cell count of each case);
  * the step's solves run both dense tiles and columns (solver_work).
Each case prints the error / bound (median and maximum) of every stage it checks, and for P2G which part of the bound dominates at the
worst face.  On one H100 80GB HBM3 the file takes about 15 minutes.

Not checked here at these sizes (each is checked on small grids only, by tests/test_gpu_step_ref.py, test_gpu_pcg_ref.py and
test_gpu_flow.py): the grid passes and the density correction (stages 1, 4, 5, 11, 12, and their stray-particle regions next to the
moving box of double_dam_box); the pressure solves (stages 2 and 10) iteration by iteration, and the step's solve as the prefix its stop
schedule names; advection and the correction per particle (stages 7 and 13) and the marker after advection; tap_256's flow prologue against
tests/flow_ref.py.  For those, tests/step_ref.py and tests/pcg_ref.py would first need windowed forms, and pcg_ref.check_runs a
streaming form.
Measured there, the most crowded cell held 6355 particles at dam_256 step 56, 4276 at step 57 and 767 at step 230."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (workload, checked step): dam_256 1 (first P2G on items), 56 (the most decayed order of a sort window, whose own stage 3 re-sorts; near the
# crowding peak), 57 (first P2G on the schedule of step 56), 230 (the step whose stages bench.py times); tap_256 with its sources appending
# particles behind the schedule (device-count mode), double_dam_box with its moving box, basin_512 (64.5 M particles, 134 M cells)
CASES = [("dam_256", 1), ("dam_256", 56), ("dam_256", 57), ("dam_256", 230), ("tap_256", 230), ("double_dam_box", 230), ("basin_512", 1)]
RESORT_EVERY = 8      # hybrid_fluid.cu: internal_resort_every_; the scenes also re-bin every 60 steps
P2G_TILE = 1184       # transfer_kernels.cu: faces of the P2G scatter tile
ITEM_WAVES = 8        # transfer_kernels.cu: P2G_MIN_ITEM_WAVES
CORE = 32             # cells per side of a window core
CROWDED_STEP_MIN = 1024
ITEM_PATH = {"dam_256", "tap_256", "basin_512"}  # double_dam_box has too few work items (834 at step 230): its P2G runs the chunks


def _gravity_dt(sc, dt):
    scale = np.float32(sc["fluid"]["grid_to_world_scale"])
    return [float(np.float32(np.float32(np.float32(sc["gravity"][c]) / scale) * np.float32(dt))) for c in "xyz"]


def _resorts(step, rebin):
    return step % rebin == 0 or step % RESORT_EVERY == 0


def _cells(pos, dims, lo):
    """Primal cells (x, y, z) of positions clamped to [lo, dim - 1], as transfer_position / cell_of_position take them."""
    from tests import grid_ref as R

    out = np.empty((len(pos), 3), dtype=np.int64)
    for a in range(0, len(pos), R.CHUNK):
        out[a:a + R.CHUNK] = np.minimum(R.clamp_positions(pos[a:a + R.CHUNK], dims, lo).astype(np.int64), np.asarray(dims) - 1)
    return out


def _lin(c, dims):
    return (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0]


def schedule(sorted_pos, dims):
    """The brick schedule a re-sort builds, restated (tools/red_stats.py, brick_schedule) from the positions the re-sort left: per brick
    its item count, and per item its brick and its particles' [first, last) ranges in the warp list."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import red_stats

    key = _lin(_cells(sorted_pos, dims, 0.0), dims)
    assert (np.diff(key) >= 0).all(), "the re-sort left the particles out of cell order"
    cell_start = np.searchsorted(key, np.arange(int(np.prod(dims)) + 1), side="left")
    brick_warps, brick_items, item_start, item_brick, warps = red_stats.brick_schedule(cell_start, dims)
    return {"brick_items": np.diff(brick_items), "item_start": item_start, "item_brick": item_brick, "warps": warps,
            "np": len(sorted_pos)}


def item_boxes(sched, pos, dims):
    """The cell box of every work item as the density scatter leaves it in item_box (item_window: primal cells clamped to [0.5, dim - 1]
    of the item's particles at the time of that scatter); returns the faces [lo - 1, hi + 1] it spans, [items, 3]."""
    cells = _cells(pos, dims, 0.5)
    warps, starts = sched["warps"], sched["item_start"]
    parts = (32 * warps[:, None] + np.arange(32)[None, :])
    ok = parts < sched["np"]
    seg = np.repeat(np.arange(len(starts)), np.diff(np.append(starts, len(warps))) * 32)[ok.ravel()]
    c = cells[parts[ok]]
    first = np.r_[0, np.flatnonzero(np.diff(seg)) + 1]
    lo, hi = np.minimum.reduceat(c, first, axis=0), np.maximum.reduceat(c, first, axis=0)
    return hi - lo + 3


def brick_centre(b, dims):
    nbx, nby = -(-dims[0] // 28), -(-dims[1] // 4)
    return np.array([b % nbx * 28 + 14, b // nbx % nby * 4 + 2, b // nbx // nby * 4 + 2])


def choose_windows(m, counts, dims, sched, rng):
    """{name: box} of 32^3-cell cores, chosen from the downloaded state."""
    from tests import grid_ref as R

    dims_a = np.asarray(dims)
    zyx = lambda i: np.array(np.unravel_index(i, m.shape))[::-1]
    centres = {"most crowded cell": zyx(int(np.argmax(counts)))}
    fl = np.flatnonzero(m.ravel() == R.FLUID)
    centres["highest FLUID cell"] = zyx(int(fl[-1]))
    b = int(np.argmax(sched["brick_items"]))
    centres[f"brick {b} ({int(sched['brick_items'][b])} items)"] = brick_centre(b, dims)
    for ax, name in enumerate("xyz"):
        for side, plane in (("low", 1), ("high", dims[ax] - 2)):
            sl = [slice(None)] * 3
            sl[2 - ax] = plane
            cand = np.argwhere(m[tuple(sl)] == R.FLUID)
            if len(cand):
                q = np.insert(cand[len(cand) // 2], 2 - ax, plane)[::-1]
                centres[f"{name} {side} wall"] = q
    air = (R._neighbours(m) == R.AIR).any(axis=0) if m.size <= 1 << 25 else None
    sparse = np.flatnonzero((counts.ravel() == 1) & (m.ravel() == R.FLUID) & (air.ravel() if air is not None else True))
    if len(sparse):
        centres["sparse free surface"] = zyx(int(rng.choice(sparse)))
    for k in range(3):
        centres[f"random fluid {k}"] = zyx(int(rng.choice(fl)))
    boxes = {}
    for name, c in centres.items():
        lo = np.clip(np.asarray(c) - CORE // 2, 0, dims_a - CORE)
        boxes[name] = (tuple(int(v) for v in lo), tuple(int(v) for v in lo + CORE))
    return boxes


class Ratios:
    """error / bound of the checked entries, per stage, for the report; and for P2G, which part of the bound dominates at the stage's
    worst face (p2g_bound_terms), so that a ratio near 1 can be told apart as tight by design or a near miss."""

    def __init__(self):
        self.parts, self.worst = {}, {}

    def check(self, stage, got, want, bound, what):
        """Asserts the bound; returns (the largest ratio, its [z, y, x] in these arrays)."""
        from tests import grid_ref as R

        R.check(got, want, bound, what)
        sel = ~np.isnan(want)
        err = np.abs(np.asarray(got, dtype=np.float64)[sel] - want[sel])
        b = bound[sel]
        r = np.where(err > 0, err / np.where(b > 0, b, 1.0), 0.0)
        self.parts.setdefault(stage, []).append(r)
        k = int(np.argmax(r)) if r.size else 0
        return (float(r[k]) if r.size else 0.0), (tuple(np.argwhere(sel)[k]) if r.size else None)

    def note_worst(self, stage, ratio, text):
        if ratio > self.worst.get(stage, (-1.0, ""))[0]:
            self.worst[stage] = (ratio, text)

    def report(self, what):
        for stage, parts in self.parts.items():
            r = np.concatenate(parts)
            print(f"{what} {stage}: {r.size} entries, error / bound: median {np.median(r):.2e}, max {r.max():.2e}")
            if stage in self.worst:
                print(f"{what} {stage}: worst face {self.worst[stage][1]}")


def p2g_windows(f, boxes, pos, rows, m, u, gdt, form, ratios, what):
    from tests import grid_ref as R

    dims = (f.nx, f.ny, f.nz)
    stage = f"stage 0 P2G ({form})"
    for name, box in boxes.items():
        frame = R.grow(box, 1, dims)
        sums = R.p2g_sums(pos, rows, dims, box=frame)
        mf = R.crop(m, frame)
        core = R.inner(frame, box)
        want, bound = R.p2g_velocity(sums, mf, gdt), R.p2g_bound(sums, mf, gdt, form)
        for c in range(3):
            ratio, at = ratios.check(stage, R.crop(u[c], box), want[c][core], bound[c][core], f"{what} {name}: P2G u[{c}] ({form})")
            if at is None or ratio <= ratios.worst.get(stage, (-1.0, ""))[0]:
                continue
            face = tuple(int(sl.start) + int(i) for sl, i in zip(core, at))  # in the frame's arrays
            glob = tuple(int(frame[0][2 - a]) + face[a] for a in range(3))
            terms = {k: float(v[face]) for k, v in R.p2g_bound_terms(sums[c], gdt[c], form).items()}
            total = sum(terms.values())
            parts = ", ".join(f"{k} {v / total:.0%}" for k, v in sorted(terms.items(), key=lambda kv: -kv[1]))
            ratios.note_worst(stage, ratio, f"u[{c}] at [z, y, x] = {glob} ({name}): ratio {ratio:.3f}, bound {float(bound[c][face]):.3e}, "
                                            f"{int(sums[c]['count'][face])} contributions; bound made of {parts}")


def rhs_windows(f, boxes, pos, m, dt, ratios, what):
    from blub_b200 import fluid as F
    from tests import grid_ref as R

    dims = (f.nx, f.ny, f.nz)
    rhs = f.download_grid(F.TAP_RESIDUAL)
    for name, box in boxes.items():
        frame = R.grow(box, 1, dims)
        d = R.density_sums(pos, dims, box=frame)
        mf = R.crop(m, frame)
        core = R.inner(frame, box)
        ratios.check("stage 9 density rhs", R.crop(rhs, box), R.density_rhs(d, mf, dt)[core], R.rhs_bound(d, mf, dt, "scatter")[core],
                     f"{what} {name}: density rhs")


def particles(f):
    from blub_b200 import fluid as F

    return [f.download_particles(t) for t in (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)]


@pytest.mark.gpu
@pytest.mark.parametrize("workload,step", CASES, ids=[f"{w}-step{s}" for w, s in CASES])
def test_benchmarked_step_matches_float64_reference(workload, step):
    import bench
    import blub_b200
    import torch
    from blub_b200 import fluid as F
    from tests import grid_ref as R

    dt = F.DT_120HZ
    sc = json.load(open(bench.scene_path(bench.workload_scene(workload))))
    f = blub_b200.HybridFluid.from_scene(bench.scene_path(bench.workload_scene(workload)))
    dims = (f.nx, f.ny, f.nz)
    gdt = _gravity_dt(sc, dt)
    stepper = bench.SolidStepper(f, sc, bench.SOLID_WORKLOADS[workload]["solid"], 0) if workload in bench.SOLID_WORKLOADS else None
    rebin = int(f.L.blub_fluid_rebinning_frequency(f.h)[0])  # particle_rebinning_step_frequency (the scenes leave it at its default)
    last_resort = max(s for s in range(step) if _resorts(s, rebin))

    def before_step():
        if stepper is not None:  # bench.SolidStepper.step without its fluid.step
            stepper.t += dt
            F.solid_voxelize(stepper.vol.data_ptr(), stepper.dims, stepper.solid, stepper.scale, stepper.origin, stepper.t, dt,
                             cuda_stream=f.stream())

    def whole_step():
        before_step()
        f.step(dt)

    sched, density_pos = None, None
    for k in range(step):
        if k not in (last_resort, step - 1):
            whole_step()
            continue
        before_step()
        f.step_stages(dt, 0, 3)
        if k == last_resort:
            f.step_stages(dt, 3, 4)
            sched = schedule(f.download_particles(), dims)
            f.step_stages(dt, 4, 9)
        else:
            f.step_stages(dt, 3, 9)
        if k == step - 1:
            density_pos = f.download_particles()
        f.step_stages(dt, 9, 14)
    what = f"{workload} step {step}"
    ratios = Ratios()

    # the code paths this case stands for
    items = int(sched["brick_items"].sum())
    threshold = ITEM_WAVES * 4 * torch.cuda.get_device_properties(0).multi_processor_count
    ext = item_boxes(sched, density_pos, dims)
    cut = int((ext.prod(axis=1) > P2G_TILE).sum())
    if workload in ITEM_PATH:
        assert items >= threshold, f"{what}: {items} work items, P2G walks them from {threshold} on"
        assert cut > 0, f"{what}: no item box larger than the P2G tile"
    del density_pos

    # stage 0 (and the gather form on dam_256 step 56: the same stage run first through the gather, then as the step runs it)
    before_step()
    gather = None
    if workload == "dam_256" and step == 56:
        f.set_transfer_path(0)
        f.step_stages(dt, 0, 1)
        gather = ([f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)], f.download_grid(F.TAP_MARKER), f.download_particles())
        f.set_transfer_path(1)
    f.step_stages(dt, 0, 1)
    pos, *rows = particles(f)  # after the flow prologue: what P2G read
    m0 = f.download_grid(F.TAP_MARKER)
    solid = f.download_solid_voxels()[..., 3] != 0 if stepper is not None else None
    assert np.array_equal(m0, R.marker(pos, dims, solid=solid)), f"{what}: marker after P2G"
    counts = np.bincount(_lin(_cells(pos, dims, 1.0), dims), minlength=int(np.prod(dims))).reshape(m0.shape)
    crowd = int(counts.max())
    print(f"{what}: {len(pos)} particles, most crowded cell {crowd} particles, {int((counts > 32).sum())} cells above 32; "
          f"{items} work items (threshold {threshold}), {cut} item boxes cut by box_window, largest brick {int(sched['brick_items'].max())} items")
    if step == 56:
        assert crowd > CROWDED_STEP_MIN, f"{what}: most crowded cell holds {crowd} particles"
    assert sched["brick_items"].max() >= 2  # and a window is centred on that brick
    boxes = choose_windows(m0, counts, dims, sched, np.random.default_rng(step))
    del counts
    p2g_windows(f, boxes, pos, rows, m0, [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)], gdt, "scatter", ratios, what)
    if gather is not None:
        assert np.array_equal(gather[1], m0) and np.array_equal(gather[2].view(np.uint32), pos.view(np.uint32))
        p2g_windows(f, boxes, pos, rows, m0, gather[0], gdt, "gather", ratios, what)
        del gather
    del pos, rows

    # stage 3: the re-sort (or nothing)
    f.step_stages(dt, 1, 3)
    before = particles(f)
    f.step_stages(dt, 3, 4)
    after = particles(f)
    if _resorts(step, rebin):
        order = np.argsort(_lin(_cells(before[0], dims, 0.0), dims), kind="stable")
        assert np.array_equal(before[0][order].view(np.uint32), after[0].view(np.uint32)), f"{what}: the re-sort is not a stable sort by cell"
        # the re-sort moves the positions only (hybrid_fluid.cu, stage 3): the APIC rows stay where they are until advection rewrites them
        for t, (a, b) in enumerate(zip(before[1:], after[1:])):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{what}: the re-sort changed APIC row {t}"
    else:
        for a, b in zip(before, after):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{what}: stage 3 moved particles without a re-sort"
    del before, after

    # stage 9: the density rhs
    f.step_stages(dt, 4, 9)
    pos9 = f.download_particles()
    m9 = f.download_grid(F.TAP_MARKER)
    f.step_stages(dt, 9, 10)
    rhs_windows(f, boxes, pos9, m9, dt, ratios, what)
    del pos9
    f.step_stages(dt, 10, 14)
    work = f.solver_work()
    assert work["tiles"] > 0 and work["columns"] > 0, f"{what}: solver work {work}"
    ratios.report(what)
    f.close()
    import resource

    print(f"{what}: peak host memory of the process so far {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20:.1f} GiB")
