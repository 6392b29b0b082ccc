"""GPU: particle tags (DESIGN.md §8, "Particle tags").  Tags change no result of a step, follow their particles through the binning, the
drain compaction, the source emission, checkpoints and z-slab migration, and the paint and census kernels agree bit for bit with NumPy
restatements.  Tags include bit patterns that are NaN, infinity and denormal as floats: a path that put them through float arithmetic would
change them."""
import ctypes as C
import json

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import flow_ref, util
from tests.test_gpu_state import snapshot
from tests.test_tags_kat import census_fixed
from tests.util import DT

pytestmark = pytest.mark.gpu

TAPS = (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)
# NaN (quiet and signalling, both signs), infinity, denormals, negative zero
SPECIAL = np.array([0xFFFFFFFF, 0x7F800001, 0x00000001, 0x7F800000, 0x7FC00001, 0x807FFFFF, 0xFF800001, 0x80000000], dtype=np.uint32)
INT32_MAX, INT32_MIN = 2 ** 31 - 1, -(2 ** 31)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def set_tags(f, tags):
    """Writes the tags through the fourth word of the position tap (blub_fluid_upload)."""
    pos = f.download_particles()
    pos[:, 3] = np.asarray(tags, dtype=np.uint32).view(np.float32)
    assert f.L.blub_fluid_upload(f.h, F.TAP_POS, pos.ctypes.data_as(C.c_void_p), pos.nbytes) == 0


def random_tags(n, seed):
    t = np.random.default_rng(seed).integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    t[: len(SPECIAL) * 64] = np.tile(SPECIAL, 64)
    return t


def assert_same_physics(a, b, stats=True):
    """Everything of two snapshots bit for bit, except the tag column of the positions.  stats=False leaves out the solver statistics
    history: over many graph-replayed steps its asynchronous read-back ring may drop samples depending on host timing."""
    assert np.array_equal(bits(a["particles_position"][:, :3]), bits(b["particles_position"][:, :3]))
    for name in ("particles_velocity_x", "particles_velocity_y", "particles_velocity_z", "grid_velocity_x", "grid_velocity_y", "grid_velocity_z",
                 "pressure_from_velocity", "pressure_from_density"):
        assert a[name].shape == b[name].shape and np.array_equal(bits(a[name]), bits(b[name])), name
    assert np.array_equal(a["marker"], b["marker"])
    for name in ("last_solve", "stats", "step_count") if stats else ("last_solve", "step_count"):
        assert a[name] == b[name], name


def assert_bits_identical(a, b):
    assert_same_physics(a, b)
    assert np.array_equal(bits(a["particles_position"]), bits(b["particles_position"]))


# ---- 1. tags do not change the physics -----------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
@pytest.mark.parametrize("scene", ["tap_small", "dam_halfhalf"])
def test_tags_do_not_change_the_physics(scene, path, graph):
    """70 steps: re-sorts every 8th step, rebinning at 0 and 60; tap_small also drains and emits."""
    runs = []
    for tagged in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        set_tags(f, random_tags(f.num_particles, 1) if tagged else np.zeros(f.num_particles, np.uint32))
        for _ in range(70):
            f.step(DT)
        runs.append((f, snapshot(f)))
    assert_same_physics(runs[0][1], runs[1][1], stats=False)
    assert not runs[0][0].particle_tags().any()
    assert runs[1][0].particle_tags().any()


# ---- 2. tags follow their particles through the binning -----------------------------------------------------------------
def _keyed(pos):
    """Rows sorted by their xyz bytes: (keys, tags)."""
    k = bits(pos[:, :3])
    order = np.lexsort((k[:, 2], k[:, 1], k[:, 0]))
    return k[order], bits(pos[:, 3])[order]


@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_tags_follow_their_particles_through_rebinning_and_resort(path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_halfhalf"))
    f.set_transfer_path(path)
    set_tags(f, random_tags(f.num_particles, 2))
    for step in (0, 8):  # the rebinning of step 0, the internal re-sort of step 8
        while f.step_count < step:
            f.step(DT)
        f.step_stages(DT, 0, 3)
        before = f.download_particles()
        kb, tb = _keyed(before)
        assert np.all(np.any(kb[1:] != kb[:-1], axis=1)), "xyz keys are not unique"
        f.step_stages(DT, 3, 4)
        after = f.download_particles()
        assert not np.array_equal(bits(before), bits(after)), "the binning did not move the particles"
        ka, ta = _keyed(after)
        assert np.array_equal(kb, ka) and np.array_equal(tb, ta)
        f.step_stages(DT, 4, 14)


# ---- 3. tags form a permutation ------------------------------------------------------------------------------------------
def test_index_tags_stay_a_permutation():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_halfhalf"))
    n = f.num_particles
    set_tags(f, np.arange(n, dtype=np.uint32))
    for _ in range(70):
        f.step(DT)
    assert np.array_equal(np.sort(f.particle_tags()), np.arange(n, dtype=np.uint32))


# ---- 4. sources and drains -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_prologue_keeps_survivor_tags_and_tags_emitted_particles(path):
    """test_gpu_flow's prologue case with tags: survivors keep theirs in order, drained tags vanish, appended particles carry their source's."""
    rng = np.random.default_rng(11)
    dims, cap = (32, 32, 32), 9000
    pos = np.concatenate([rng.uniform(1.001, 30.999, (5000, 4)), rng.uniform(1.0, 6.0, (1500, 4)),
                          np.c_[rng.uniform(12, 15, (40, 3)), np.zeros(40)]]).astype(np.float32)
    tags = np.arange(1000, 1000 + len(pos), dtype=np.uint32)
    tags[:len(SPECIAL) - 1] = SPECIAL[SPECIAL != 0x00000001]
    pos[:, 3] = tags.view(np.float32)
    rows = [rng.standard_normal((len(pos), 4)).astype(np.float32) for _ in range(3)]
    sources = [((12, 12, 12), (16, 14, 15), (0.0, -30.0, 4.0), 0xDEADBEEF), ((20, 20, 20), (24, 22, 23), (7.0, 0.0, 0.0), 0x00000001)]
    drains = [((1, 1, 1), (5, 4, 6)), ((26, 2, 2), (30, 5, 8))]
    f = blub_b200.HybridFluid(*dims, cap)
    f.set_transfer_path(path)
    f.set_particles(pos, *rows)
    f.set_flow(sources, drains)
    f.step_stages(DT, 0, 1)
    flow = flow_ref.make_flow(dims, [s[:3] for s in sources], drains)
    want_pos, want_rows, (emitted, drained, _) = flow_ref.prologue(pos, rows, 0, dims, cap, flow)
    survivors = len(want_pos) - emitted
    c = flow_ref.cells_of(want_pos[survivors:], dims)
    for (lo, hi, _), (_, _, _, tag) in zip(flow["sources"], sources):
        inside = np.ones(emitted, dtype=bool)
        for k in range(3):
            inside &= (c[k] >= lo[k]) & (c[k] < hi[k])
        want_pos[survivors:, 3][inside] = np.uint32(tag).view(np.float32)
    got = [f.download_particles(t) for t in TAPS]
    for g, w in zip(got, [want_pos] + want_rows):
        assert np.array_equal(bits(g), bits(w))
    got_tags = bits(got[0][:, 3])
    assert emitted > 0 and drained > 0
    assert np.array_equal(got_tags[:survivors], bits(pos[:, 3])[np.isin(bits(pos[:, 3]), got_tags[:survivors])])  # survivors in order
    assert set(got_tags[survivors:].tolist()) == {0xDEADBEEF, 0x00000001}
    gone = np.setdiff1d(tags, got_tags[:survivors])
    assert len(gone) == drained and not np.isin(gone, got_tags).any()


# ---- 5. painting ---------------------------------------------------------------------------------------------------------
def painted(pos, dims, mn, mx, tag):
    """NumPy restatement: clamp the box as add_cube does, take the drains' cell of every particle, set the tag inside."""
    lo = [flow_ref.clamp_to_grid(dims[k], mn[k]) for k in range(3)]
    hi = [flow_ref.clamp_to_grid(dims[k], mx[k]) for k in range(3)]
    c = flow_ref.cells_of(pos, dims)
    inside = np.ones(len(pos), dtype=bool)
    for k in range(3):
        inside &= (c[k] >= lo[k]) & (c[k] < hi[k])
    out = bits(pos[:, 3]).copy()
    out[inside] = tag
    return out, int(inside.sum())


def face_particles(rng):
    """Random particles in the whole grid, border cells included, plus particles exactly on and next to the faces of box (4..9, 5..11, 6..13)."""
    pos = rng.uniform(0.0, 32.0, (6000, 4)).astype(np.float32)
    faces = []
    for v in (4.0, 9.0, np.nextafter(np.float32(9.0), np.float32(0)), np.nextafter(np.float32(4.0), np.float32(0))):
        for axis in range(3):
            p = rng.uniform(4.0, 9.0, (50, 4)).astype(np.float32)
            p[:, axis] = v
            faces.append(p)
    pos = np.concatenate([pos] + faces).astype(np.float32)
    pos[:, 3] = random_tags(len(pos), 5).view(np.float32)
    return pos


@pytest.mark.parametrize("device_count", [False, True])
def test_paint_matches_the_restatement(device_count):
    rng = np.random.default_rng(4)
    dims = (32, 32, 32)
    pos = face_particles(rng)
    rows = [rng.standard_normal((len(pos), 4)).astype(np.float32) for _ in range(3)]
    f = blub_b200.HybridFluid(*dims, 8000)
    f.set_particles(pos, *rows)
    if device_count:
        f.set_flow(drains=[((28, 28, 28), (31, 31, 31))])  # flow set active: the paint kernel reads the device count
        assert f.has_flow
    cur = pos.copy()
    for mn, mx, tag in [((4.0, 5.0, 6.0), (9.0, 11.0, 13.0), 0x7F800001), ((4.0, 4.0, 4.0), (9.0, 9.0, 9.0), 3),
                        ((-5.0, -5.0, -5.0), (100.0, 100.0, 100.0), 0xFFFFFFFF), ((0.0, 0.0, 0.0), (2.9, 40.0, 40.0), 0x00000001)]:
        f.paint_tags(mn, mx, tag)
        want, hits = painted(cur, dims, mn, mx, tag)
        assert hits > 0
        got = f.download_particles()
        assert np.array_equal(bits(got[:, 3]), want)
        assert np.array_equal(bits(got[:, :3]), bits(pos[:, :3]))
        cur = got
    for t, r in zip(TAPS[1:], rows):
        assert np.array_equal(bits(f.download_particles(t)), bits(r))
    # the whole-grid box stops at the border cells
    c = flow_ref.cells_of(cur, dims)
    border = np.zeros(len(cur), dtype=bool)
    for k in range(3):
        border |= (c[k] == 0) | (c[k] == dims[k] - 1)
    assert border.any() and not (bits(cur[:, 3])[~border] == 0x7F800001).any()


def test_paint_refusals_change_nothing():
    f = blub_b200.HybridFluid(32, 32, 32, 4000)
    f.add_fluid_cube((2, 2, 2), (10, 10, 10), tag=9)
    before = f.particle_tags().copy()
    for mn, mx in [((4, 4, 4), (8, float("nan"), 8)), ((float("inf"), 4, 4), (8, 8, 8)), ((5, 5, 5), (5, 9, 9)), ((40, 40, 40), (50, 50, 50))]:
        with pytest.raises(blub_b200.BlubError):
            f.paint_tags(mn, mx, 1)
    f.step_stages(DT, 0, 3)
    with pytest.raises(blub_b200.BlubError):
        f.paint_tags((2, 2, 2), (10, 10, 10), 1)
    assert b"inside a step" in F.lib().blub_last_error()
    f.step_stages(DT, 3, 14)
    assert np.array_equal(f.particle_tags(), before) and np.all(before == 9)
    f.paint_tags((0, 0, 0), (40, 40, 40), 1)  # the whole interior: every simulated particle lies in [1.001, dim - 1.001]
    assert np.all(f.particle_tags() == 1)
    slab = blub_b200.HybridFluid.create_slab(32, 32, 16, 1000, 0, 2)
    with pytest.raises(blub_b200.BlubError):
        slab.paint_tags((2, 2, 2), (10, 10, 10), 1)
    assert b"z-slab" in F.lib().blub_last_error()


# ---- 6. census -----------------------------------------------------------------------------------------------------------
def numpy_census(pos, rows, dims, first, count):
    """Exact int64 sums per tag of the downloaded particles (sorted by tag, then reduceat)."""
    tags = bits(pos[:, 3]).astype(np.int64) - first
    keep = (tags >= 0) & (tags < count)
    tags = tags[keep]
    order = np.argsort(tags, kind="stable")
    tags = tags[order]
    fx = [census_fixed(pos[keep, k])[order] for k in range(3)] + [census_fixed(r[keep, 3])[order] for r in rows]
    cells = [c[keep][order] for c in flow_ref.cells_of(pos, dims)]
    out = {"count": np.zeros(count, np.uint64), "position_sum_fx": np.zeros((count, 3), np.int64), "velocity_sum_fx": np.zeros((count, 3), np.int64),
           "cell_min": np.full((count, 3), INT32_MAX, np.int32), "cell_max": np.full((count, 3), INT32_MIN, np.int32)}
    if len(tags) == 0:
        return out
    present, starts = np.unique(tags, return_index=True)
    out["count"][present] = np.diff(np.append(starts, len(tags)))
    for k in range(3):
        out["position_sum_fx"][present, k] = np.add.reduceat(fx[k], starts)
        out["velocity_sum_fx"][present, k] = np.add.reduceat(fx[3 + k], starts)
        out["cell_min"][present, k] = np.minimum.reduceat(cells[k], starts)
        out["cell_max"][present, k] = np.maximum.reduceat(cells[k], starts)
    return out


def assert_census(got, want):
    for name in ("count", "position_sum_fx", "velocity_sum_fx", "cell_min", "cell_max"):
        assert np.array_equal(got[name], want[name]), name


@pytest.mark.parametrize("sort", [False, True])
def test_census_matches_exact_numpy_sums(sort):
    """Tags 0..299 with 50 absent, census of [10, 266): out-of-range tags skipped, empty tags report the sentinels.  Sorted by tag, whole
    warps share one tag (the register-reduced path); unsorted, they do not."""
    rng = np.random.default_rng(6)
    dims, n = (32, 32, 32), 20000
    pos = rng.uniform(0.0, 32.0, (n, 4)).astype(np.float32)
    tags = rng.integers(0, 300, n).astype(np.uint32)
    tags[tags == 50] = 51
    if sort:
        tags = np.sort(tags)
    pos[:, 3] = tags.view(np.float32)
    rows = [(rng.standard_normal((n, 4)) * 300).astype(np.float32) for _ in range(3)]
    f = blub_b200.HybridFluid(*dims, n)
    f.set_particles(pos, *rows)
    got = f.tag_census(10, 256)
    assert_census(got, numpy_census(pos, rows, dims, 10, 256))
    assert got["count"][40] == 0 and tuple(got["cell_min"][40]) == (INT32_MAX,) * 3 and tuple(got["cell_max"][40]) == (INT32_MIN,) * 3
    assert int(got["count"].sum()) == int(((tags >= 10) & (tags < 266)).sum())
    one = f.tag_census(7, 1)
    assert_census(one, numpy_census(pos, rows, dims, 7, 1))
    np.testing.assert_allclose(one["centroid"][0], pos[tags == 7, :3].astype(np.float64).mean(axis=0), rtol=1e-6)
    # the top of the tag range and the refusals
    top = np.uint32(0xFFFFFFFF) - (tags % 7)
    pos[:, 3] = top.view(np.float32)
    f.set_particles(pos, *rows)
    assert_census(f.tag_census(2 ** 32 - 256, 256), numpy_census(pos, rows, dims, 2 ** 32 - 256, 256))
    L = F.lib()
    buf = (F.TagCensus * 257)()
    for first, count in [(0, 0), (0, 257), (2 ** 32 - 255, 256), (0xFFFFFFFF, 2)]:
        assert L.blub_fluid_tag_census(f.h, first, count, buf) == 1, (first, count)


def test_census_on_the_device_count_and_at_16_million_particles():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    n = f.num_particles
    assert n > 16_000_000
    set_tags(f, (np.arange(n, dtype=np.uint32) // 1000) % 300)
    for _ in range(3):
        f.step(DT)
    pos = f.download_particles()
    rows = [f.download_particles(t) for t in TAPS[1:]]
    dims = f.grid_dimension()
    assert_census(f.tag_census(0, 256), numpy_census(pos, rows, dims, 0, 256))
    assert_census(f.tag_census(299, 1), numpy_census(pos, rows, dims, 299, 1))
    # device-count mode: a far drain makes the count live on the device
    f.set_flow(drains=[((250, 250, 250), (255, 255, 255))])
    assert_census(f.tag_census(44, 256), numpy_census(pos, rows, dims, 44, 256))


# ---- 7. checkpoints ------------------------------------------------------------------------------------------------------
def test_tagged_fluid_with_tagged_sources_resumes_bit_for_bit(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_tagged_small"))
    set_tags(f, random_tags(f.num_particles, 8))
    for _ in range(7):
        f.step(DT)
    path = str(tmp_path / "tagged.blub")
    f.save_state(path)
    assert blub_b200.state_info(path).format_version == 4
    g = blub_b200.HybridFluid.from_state(path)
    assert np.array_equal(bits(g.download_particles()), bits(f.download_particles()))
    for _ in range(3):  # emission and the re-sort at step 8 after the load
        f.step(DT)
        g.step(DT)
    assert_bits_identical(snapshot(f), snapshot(g))
    assert g.flow_counters == f.flow_counters and g.flow_counters["emitted"] > 0
    assert {100, 0x7F800001} <= set(g.particle_tags().tolist())
    # tags written after the load: add_fluid_cube appends tagged particles
    n = g.num_particles
    g.add_fluid_cube((20, 20, 20), (22, 22, 22), tag=0x00000001)
    t = g.particle_tags()
    assert len(t) == n + 64 and np.all(t[n:] == 1)


@pytest.mark.parametrize("scene,version", [("dam_small", 1), ("tap_small", 2)])
def test_particle_tags_alone_keep_the_file_version(tmp_path, scene, version):
    f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    f.step(DT)
    set_tags(f, random_tags(f.num_particles, 9))
    f.step(DT)
    path = str(tmp_path / "p.blub")
    f.save_state(path)
    assert blub_b200.state_info(path).format_version == version
    g = blub_b200.HybridFluid.from_state(path)
    for _ in range(7):  # crosses the re-sort at step 8
        f.step(DT)
        g.step(DT)
    assert_bits_identical(snapshot(f), snapshot(g))


# ---- 8. scene keys -------------------------------------------------------------------------------------------------------
def test_tagged_scene_tags_cubes_and_sources():
    scene = util.scene_path("tap_tagged_small")
    sc = json.load(open(scene))
    cube_tags = [c["tag"] for c in sc["fluid"]["fluid_cubes"]]
    source_tags = [s["tag"] for s in sc["fluid"]["sources"]]
    f = blub_b200.HybridFluid.from_scene(scene)
    t0 = f.particle_tags()
    scale = np.float32(sc["fluid"]["grid_to_world_scale"])
    want = []
    for c in sc["fluid"]["fluid_cubes"]:  # corners world / scale in float32, clamped as add_cube clamps them
        ext = [flow_ref.clamp_to_grid(32, np.float32(c["max"][a]) / scale) - flow_ref.clamp_to_grid(32, np.float32(c["min"][a]) / scale) for a in "xyz"]
        want.append(int(np.prod(ext)) * 8)
    assert [int((t0 == t).sum()) for t in cube_tags] == want == [15 * 5 * 30 * 8] * 2
    for _ in range(10):
        f.step(DT)
    t = f.particle_tags()
    assert set(t.tolist()) <= set(cube_tags + source_tags) and set(source_tags) <= set(t.tolist())
    for tag in cube_tags + source_tags:
        assert int(f.tag_census(tag, 1)["count"][0]) == int((t == tag).sum())


# ---- 9. slab migration ---------------------------------------------------------------------------------------------------
def test_index_tags_survive_sharded_steps_as_a_permutation():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from tests.test_gpu_multi import make_slabs
    nx, ny, nz_owned, world = 64, 64, 32, 2
    cap = 8 * 31 * 40 * 62 + 1000
    slabs = make_slabs(world, nx, ny, nz_owned)
    for s in slabs:
        s.close()
    slabs = [blub_b200.HybridFluid.create_slab(nx, ny, nz_owned, cap, rank=k, world=world, device=k) for k in range(world)]
    windows = [s.slab_window()[0] for s in slabs]
    for s in slabs:
        s.attach_slab_peers(windows)
    base = 0
    for s in slabs:
        s.add_fluid_cube([0.0, 0.0, 0.0], [32.0, 41.0, float(world * nz_owned)])
        s.set_gravity_grid([0.0, -981.0, 0.0])
        n = s.num_particles
        set_tags(s, np.arange(base, base + n, dtype=np.uint32))
        base += n
    for _ in range(20):
        for s in slabs:
            s.step(DT)
        for s in slabs:
            s.synchronize()
    assert all(s.slab_error() == 0 for s in slabs)
    tags = np.concatenate([s.particle_tags() for s in slabs])
    assert np.array_equal(np.sort(tags), np.arange(base, dtype=np.uint32))
    # the census of a rank covers that rank's particles
    for s in slabs:
        t = s.particle_tags()
        assert int(s.tag_census(0, 256)["count"].sum()) == int((t < 256).sum())
