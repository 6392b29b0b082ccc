"""GPU: sources and drains (flow_kernels.cu).  The prologue agrees bit for bit with the NumPy restatement in tests/flow_ref.py, steps with a
flow set are reproducible on both transfer paths and in graph and eager launches, device-count mode alone changes no result, and a fluid with
a flow set saves and resumes bit for bit."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from tests import flow_ref, util
from tests.test_gpu_state import assert_identical, snapshot
from tests.util import DT

pytestmark = pytest.mark.gpu

TAPS = (blub_b200.fluid.TAP_POS, blub_b200.fluid.TAP_VX, blub_b200.fluid.TAP_VY, blub_b200.fluid.TAP_VZ)


def tap_flow(dims=(32, 32, 32)):
    """The flow set of tests/golden/scenes/tap_small.json in grid units (what blub_scene_load applies)."""
    return {"sources": [((12.0, 25.5, 12.0), (18.5, 28.5, 18.5), (0.0, -100.0, 0.0))], "drains": [((0.5, 0.5, 0.5), (5.5, 3.5, 5.5))]}


@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_prologue_matches_the_restatement_bit_for_bit(path):
    rng = np.random.default_rng(11)
    dims, cap = (32, 32, 32), 9000
    pos = np.concatenate([rng.uniform(1.001, 30.999, (5000, 4)), rng.uniform(1.0, 6.0, (1500, 4)),  # many in the drain, across chunks
                          np.c_[rng.uniform(12, 15, (40, 3)), np.zeros(40)]]).astype(np.float32)  # partly filled source cells
    pos[:, 3] = 0.0
    rows = [rng.standard_normal((len(pos), 4)).astype(np.float32) for _ in range(3)]
    sources = [((12, 12, 12), (16, 14, 15), (0.0, -30.0, 4.0)), ((20, 20, 20), (24, 22, 23), (7.0, 0.0, 0.0))]
    drains = [((1, 1, 1), (5, 4, 6)), ((26, 2, 2), (30, 5, 8))]
    f = blub_b200.HybridFluid(*dims, cap)
    f.set_transfer_path(path)
    f.set_particles(pos, *rows)
    f.set_flow(sources, drains)
    f.step_stages(DT, 0, 1)
    want_pos, want_rows, want_counts = flow_ref.prologue(pos, rows, 0, dims, cap, flow_ref.make_flow(dims, sources, drains))
    assert f.num_particles == len(want_pos)
    got = [f.download_particles(t) for t in TAPS]
    for g, w in zip(got, [want_pos] + want_rows):
        np.testing.assert_array_equal(g, w)
    assert f.flow_counters == dict(zip(("emitted", "drained", "refused"), want_counts))
    assert want_counts[0] > 0 and want_counts[1] > 0


def test_trajectory_follows_the_oracle():
    """DESIGN §5's N-step tolerance on tap_small with converged solves: 99.9 % of the positions within 1e-2 cells; equal counts every step."""
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    o = util.oracle_from_scene("tap_small")  # the oracle's scene loader seeds the cubes only: the prologue comes from tests/flow_ref.py
    util.tight_solver(f, o)
    flow = flow_ref.make_flow((32, 32, 32), tap_flow()["sources"], tap_flow()["drains"])
    counters = [0, 0, 0]
    for k in range(6):
        f.step(DT)
        flow_ref.step_with_flow(o, flow, counters, dt=DT)
        assert f.num_particles == o.num_particles, k
    # particle orders differ (the library re-sorts every 8th step, the oracle rebins every 60th): pair every particle with the nearest oracle
    # particle in the max norm, as a sort by coordinates would mis-pair particles whose x differ by less than the rounding differences
    from scipy.spatial import cKDTree
    dist, _ = cKDTree(o.particles()[:, :3].astype(np.float64)).query(f.download_particles()[:, :3].astype(np.float64), p=np.inf)
    assert np.mean(dist < 1e-2) >= 0.999
    assert f.flow_counters == dict(zip(("emitted", "drained", "refused"), counters)) and counters[0] > 0


def _run(path, graph, steps=20, scene="tap_small", setup=None):
    f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    f.set_transfer_path(path)
    f.set_graph_replay(graph)
    if setup:
        setup(f)
    for _ in range(steps):
        f.step(DT)
    return f, snapshot(f)


@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_runs_are_reproducible_and_graph_replay_equals_eager_launches(path):
    f1, a = _run(path, True)
    f2, b = _run(path, True)
    f3, c = _run(path, False)
    assert_identical(a, b)
    assert_identical(a, c)
    assert f1.flow_counters == f2.flow_counters == f3.flow_counters
    assert f1.flow_counters["emitted"] > 0


@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_device_count_mode_alone_changes_nothing(path):
    far_drain = lambda f: f.set_flow(drains=[((28, 28, 28), (31, 31, 31))])  # the top far corner: no particle of dam_small gets there in 20 steps
    f1, a = _run(path, True, scene="dam_small")
    f2, b = _run(path, True, scene="dam_small", setup=far_drain)
    assert f2.flow_counters == {"emitted": 0, "drained": 0, "refused": 0}
    assert_identical(a, b)


def test_save_and_resume_with_the_flow_active(tmp_path):
    # saved after step 7, resumed for 3 steps: emission steps and the re-sort at step 8 after the load
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    for _ in range(7):
        f.step(DT)
    path = str(tmp_path / "flow.blub")
    f.save_state(path)
    info = blub_b200.state_info(path)
    assert info.format_version == 2 and info.num_particles == f.num_particles and info.step_count == 7
    g = blub_b200.HybridFluid.from_state(path)
    assert g.flow_counters == f.flow_counters and g.num_particles == f.num_particles
    emitted_at_save = g.flow_counters["emitted"]
    for _ in range(3):
        f.step(DT)
        g.step(DT)
    assert_identical(snapshot(f), snapshot(g))
    assert g.flow_counters == f.flow_counters
    assert g.flow_counters["emitted"] > emitted_at_save  # the resumed steps emit
    plain = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    plain.step(DT)
    plain.save_state(str(tmp_path / "plain.blub"))
    assert blub_b200.state_info(str(tmp_path / "plain.blub")).format_version == 1


def test_solid_source_cells_do_not_emit():
    torch = pytest.importorskip("torch")
    dims, cap = (32, 32, 32), 4000
    solid = np.zeros(dims[::-1], dtype=bool)
    solid[12, 12:14, 12:15] = True  # (z, y, x): 6 cells of the source box
    vox = np.zeros(dims[::-1] + (4,), dtype=np.float16)
    vox[..., 3] = solid
    dev = torch.from_numpy(vox).cuda()
    rng = np.random.default_rng(5)
    pos = np.c_[rng.uniform(2, 8, (300, 3)), np.zeros(300)].astype(np.float32)
    rows = [rng.standard_normal((300, 4)).astype(np.float32) for _ in range(3)]
    sources = [((12, 12, 12), (16, 15, 14), (0.0, -20.0, 0.0))]
    f = blub_b200.HybridFluid(*dims, cap)
    f.set_solid_voxels(dev.data_ptr())
    f.set_particles(pos, *rows)
    f.set_flow(sources)
    f.step_stages(DT, 0, 1)
    want_pos, want_rows, want_counts = flow_ref.prologue(pos, rows, 0, dims, cap, flow_ref.make_flow(dims, sources), solid)
    assert want_counts[0] == (4 * 3 * 2 - 6) * 8
    for t, w in zip(TAPS, [want_pos] + want_rows):
        np.testing.assert_array_equal(f.download_particles(t), w)
    del f
    torch.cuda.synchronize()


def test_runner_reports_the_counters_of_a_library_run(tmp_path):
    runner = os.path.join(os.path.dirname(blub_b200.fluid.lib_path()), "blub_run")
    stats = str(tmp_path / "stats.json")
    res = subprocess.run([runner, util.scene_path("tap_small"), "--steps", "20", "--stats", stats], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    for _ in range(20):
        f.step(DT)
    assert json.load(open(stats))["flow"] == f.flow_counters and f.flow_counters["emitted"] > 0
    assert f"progress 16/20, " in res.stdout and f"progress 20/20, {f.num_particles} particles)" in res.stdout
    plain = str(tmp_path / "plain.json")
    res = subprocess.run([runner, util.scene_path("dam_small"), "--steps", "2", "--stats", plain], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "flow" not in json.load(open(plain)) and "(progress 2/2)\n" in res.stdout


def test_capacity_holds_and_the_refused_counter_grows():
    f = blub_b200.HybridFluid(32, 32, 32, 3000)
    f.add_fluid_cube((1, 1, 1), (10, 4, 10))  # 81 cells x 3 rows = 1944 particles
    f.set_flow(sources=[((12, 20, 12), (20, 24, 20), (0, -50, 0))])  # 256 cells, 2048 particles at once
    refused = []
    for _ in range(3):
        f.step(DT)
        assert f.num_particles == 3000
        refused.append(f.flow_counters["refused"])
    assert refused[0] == 1944 + 2048 - 3000 and refused[2] > refused[1] > refused[0]


def test_refusals():
    f = blub_b200.HybridFluid(32, 32, 32, 1000)
    src = [((4, 4, 4), (8, 8, 8), (0, 0, 0))]
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(sources=src + [((6, 6, 6), (10, 10, 10), (0, 0, 0))])  # overlapping sources
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(sources=src, drains=[((7, 7, 7), (9, 9, 9))])  # source overlaps a drain
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(drains=[((k + 1, 1, 1), (k + 2, 2, 2)) for k in range(17)])
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(sources=[((4, 4, 4), (8, 8, 8), (0, float("nan"), 0))])
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(drains=[((5, 5, 5), (5, 9, 9))])  # empty
    f.step_stages(DT, 0, 3)
    with pytest.raises(blub_b200.BlubError):
        f.set_flow(sources=src)
    f.step_stages(DT, 3, 14)
    f.set_flow(sources=src)
    f.set_flow()
    slab = blub_b200.HybridFluid.create_slab(32, 32, 16, 1000, 0, 2)
    with pytest.raises(blub_b200.BlubError):
        slab.set_flow(sources=src)
