"""CFL-limited substeps on the GPU: the exact largest particle velocity against NumPy, the planning rule on the measurement, advance() without
hidden effects, varying step lengths against the oracle, refusals and the runner's --cfl (DESIGN.md §8 "CFL-limited substeps")."""
import json
import os
import subprocess
import zlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from tests import util

pytestmark = pytest.mark.gpu

INTERVAL_NS = 8_333_333  # blub_simulation_delta_ns(120)
G = (0.0, -981.0, 0.0)
RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
GRID_TAPS = (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_MARKER, F.TAP_P_VEL, F.TAP_P_DEN)
PARTICLE_TAPS = (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)


def secs(dt_ns):
    return float(F.lib().blub_duration_as_secs_f32(int(dt_ns)))


def expected_bits(rows, n):
    """max |row[:, 3]| per row as float32 bits: the sign bit cleared, an unsigned max (0 for no particles)."""
    return [int((r[:n, 3].view(np.uint32) & np.uint32(0x7FFFFFFF)).max()) if n else 0 for r in rows]


def measured_bits(f):
    return [int(np.float32(v).view(np.uint32)) for v in f.max_particle_velocity()]


def random_particles(n, rng, dims=(32, 32, 32)):
    pos = np.zeros((n, 4), dtype=np.float32)
    for k in range(3):
        pos[:, k] = rng.uniform(1.5, dims[k] - 1.5, n)
    pos[:, 3] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)  # tags, any bits: never read
    rows = [(rng.standard_normal((n, 4)) * 50.0).astype(np.float32) for _ in range(3)]
    for r in rows:
        r[:, :3] = np.float32(3e38)  # the C columns are not read either
    return pos, rows


def case_rows(case, rng):
    if case.startswith("count_"):
        n = int(case.split("_")[1])
        return random_particles(n, rng)
    pos, rows = random_particles(1000, rng)
    w = [r[:, 3] for r in rows]
    if case == "signed_zeros":
        for x in w:
            x[:] = np.where(rng.random(1000) < 0.5, np.float32(0.0), np.float32(-0.0))
    elif case == "denormals":
        for x in w:
            x[:] = (rng.integers(1, 2 ** 23, 1000).astype(np.uint32) | (rng.integers(0, 2, 1000).astype(np.uint32) << 31)).view(np.float32)
        w[1][:] = -np.float32(1.4e-45)
    elif case == "largest_finite":
        w[0][500] = -np.finfo(np.float32).max
        w[2][7] = np.finfo(np.float32).max
    elif case == "max_first":
        for c, x in enumerate(w):
            x[0] = -1e6 * (c + 1)
    elif case == "max_last":
        for c, x in enumerate(w):
            x[-1] = 1e6 * (c + 1) * (-1) ** c
    return pos, rows


@pytest.mark.parametrize("case", ["signed_zeros", "denormals", "largest_finite", "max_first", "max_last", "count_0", "count_1", "count_31", "count_33",
                                  "count_1000", "count_123457"])
def test_max_velocity_is_exact_on_uploaded_particles(case):
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    pos, rows = case_rows(case, rng)
    f = blub_b200.HybridFluid(32, 32, 32, 200_000)
    if len(pos):
        f.set_particles(pos, *rows)
    assert f.num_particles == len(pos)
    got = measured_bits(f)
    assert got == expected_bits(rows, len(pos)), (case, got)
    if case == "signed_zeros" or case == "count_0":
        assert got == [0, 0, 0]  # +0
    if case == "largest_finite":
        assert got[0] == got[2] == int(np.finfo(np.float32).max.view(np.uint32))


def test_max_velocity_of_all_dam_256_particles():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_256"))
    for _ in range(12):
        f.step()
    f.synchronize()
    n = f.num_particles
    assert n > 16_000_000
    rows = [f.download_particles(t) for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]
    got = measured_bits(f)
    assert got == expected_bits(rows, n)
    assert np.array(got, dtype=np.uint32).view(np.float32)[1] > 10.0  # the column is falling


def test_max_velocity_in_device_count_mode_ignores_stale_particles():
    """After a drain the device count is below the arrays' old length: the compaction leaves the drained particles' rows behind it.  The
    drained particles are the last ones and carry huge velocities, so a kernel that read past the live count would see them."""
    rng = np.random.default_rng(3)
    pos, rows = random_particles(20_000, rng)
    k = 500
    pos[-k:, :3] = rng.uniform(26.2, 29.8, (k, 3))
    for c, r in enumerate(rows):
        r[-k:, 3] = np.float32(1e30) * (c + 1)
    f = blub_b200.HybridFluid(32, 32, 32, 40_000)
    f.set_rebin_frequency(0)
    f.set_gravity_grid(G)
    f.set_particles(pos, *rows)
    f.set_flow(drains=[((26, 26, 26), (30, 30, 30))])
    assert measured_bits(f) == expected_bits(rows, len(pos))  # before the drain they are live
    f.step()
    n = f.num_particles
    assert n <= len(pos) - k and f.flow_counters["drained"] >= k
    live = [f.download_particles(t) for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]
    got = measured_bits(f)
    assert got == expected_bits(live, n)
    assert np.array(got, dtype=np.uint32).view(np.float32).max() < 1e6


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_non_finite_velocities_come_out_as_themselves_and_are_unstable(bad):
    rng = np.random.default_rng(9)
    pos, rows = random_particles(5000, rng)
    rows[1][1234, 3] = bad
    f = blub_b200.HybridFluid(32, 32, 32, 10_000)
    f.set_particles(pos, *rows)
    got = measured_bits(f)
    assert got == expected_bits(rows, 5000)
    v = f.max_particle_velocity()
    assert np.isinf(v[1]) if np.isinf(bad) else np.isnan(v[1])
    with pytest.raises(F.BlubError, match="error 6.*not finite"):
        f.plan_substep(INTERVAL_NS)
    assert f.step_count == 0
    with pytest.raises(F.BlubError, match="error 6"):
        f.advance(INTERVAL_NS)
    assert f.step_count == 0


def test_plan_equals_the_rule_on_the_measurement():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    f.set_gravity_grid(G)
    for _ in range(6):
        f.step()
    for remaining in (1, 1_000_000, 3_000_001, INTERVAL_NS, 10 ** 9):
        for cfl in (0.25, 1.0, 3.0):
            dt, v = f.plan_substep(remaining, cfl, remaining, 1)
            assert v == f.max_particle_velocity()
            assert dt == F.cfl_substep_ns(remaining, v, G, cfl, remaining, 1)
    assert max(v) > 10.0
    d_ns = F.cfl_substep_ns(10 ** 9, v, G, 1.0, 10 ** 9, 1)
    with pytest.raises(F.BlubError, match="error 6.*min_dt_ns"):  # the same measurement refused by the same rule
        f.plan_substep(10 ** 9, 1.0, 10 ** 9, d_ns + 1)
    assert f.plan_substep(10 ** 9, 1.0, 10 ** 9, d_ns)[0] == d_ns
    launches = blub_b200.kernel_launch_count()
    f.plan_substep(INTERVAL_NS)
    assert blub_b200.kernel_launch_count() - launches == 1  # one kernel per plan


def snapshot(f):
    f.synchronize()
    out = [f.download_particles(t) for t in PARTICLE_TAPS] + [f.download_grid(t) for t in GRID_TAPS]
    out.append(np.array([f.step_count, f.num_particles], dtype=np.int64))
    return out


def assert_identical(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), k


def scene_fluid(graph=True, flow=False, bodies=False):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    f.set_graph_replay(graph)
    f.set_gravity_grid(G)
    if flow:
        f.set_flow(sources=[((20, 20, 4), (24, 24, 8), (0.0, -40.0, 60.0))], drains=[((26, 1, 24), (31, 5, 31))])
    if bodies:
        f.set_bodies([{"shape": "box", "half_extent": (3.0, 2.0, 3.0), "relative_density": 0.6, "centre": (22.0, 12.0, 16.0)},
                      {"shape": "sphere", "half_extent": 3.0, "relative_density": 2.0, "centre": (8.0, 26.0, 20.0)}])
    return f


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("extras", ["plain", "flow_and_bodies"])
def test_advance_has_no_hidden_effects(graph, extras):
    """A fresh fluid stepped by hand with advance's dts computes the same bits; two advance runs are identical."""
    kw = dict(graph=graph, flow=extras != "plain", bodies=extras != "plain")
    a = scene_fluid(**kw)
    plans = []
    for _ in range(4):
        plans += a.advance(INTERVAL_NS, cfl=0.5)
    dts = [dt for dt, _ in plans]
    assert sum(dts) == 4 * INTERVAL_NS and len(set(dts)) > 1 and len(dts) > 4
    b = scene_fluid(**kw)
    for dt in dts:
        b.step(secs(dt))
    sa, sb = snapshot(a), snapshot(b)
    assert_identical(sa, sb)
    if kw["bodies"]:
        for i in range(2):
            ha, hb = a.body_history(i), b.body_history(i)
            for key in ("force_fx", "torque_fx", "centre", "velocity"):
                assert np.array_equal(ha[key], hb[key]), key
        # dam_small is seeded at its capacity: the source asks for particles in every step and is refused for capacity
        assert a.flow_counters == b.flow_counters and a.flow_counters["emitted"] + a.flow_counters["refused"] > 0
    c = scene_fluid(**kw)
    again = []
    for _ in range(4):
        again += c.advance(INTERVAL_NS, cfl=0.5)
    assert again == plans
    assert_identical(snapshot(c), sa)


def test_state_saved_inside_an_interval_continues_bit_for_bit(tmp_path):
    a = scene_fluid(flow=True)
    a.advance(INTERVAL_NS, cfl=0.25)
    dt, _ = a.plan_substep(INTERVAL_NS, 0.25, INTERVAL_NS, INTERVAL_NS // 256)  # one substep into the second interval
    a.step(secs(dt))
    remaining = INTERVAL_NS - dt
    assert 0 < remaining < INTERVAL_NS
    path = str(tmp_path / "mid.blub")
    a.save_state(path)
    b = blub_b200.HybridFluid.from_state(path)
    runs = []
    for f in (a, b):
        plans, left = [], remaining
        while left:
            dt, v = f.plan_substep(left, 0.25, INTERVAL_NS, INTERVAL_NS // 256)
            f.step(secs(dt))
            left -= dt
            plans.append((dt, v))
        plans += f.advance(INTERVAL_NS, cfl=0.25)
        runs.append((plans, snapshot(f)))
    assert runs[0][0] == runs[1][0]
    assert_identical(runs[0][1], runs[1][1])


def test_varying_step_lengths_match_the_oracle():
    """dam_small over two intervals at C = 0.25: the planned substeps differ in length, and the oracle stepping the same dts agrees at the
    tolerances of the fixed-step scene parity test."""
    orc = util.oracle_from_scene("dam_small")
    gpu = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    for f in (orc, gpu):
        f.set_rebin_frequency(0)
        f.set_gravity_grid(G)
        f.set_solver_config(0, 1e-4, 128, 4)
        f.set_solver_config(1, 1e-4, 128, 4)
    dts = []
    for _ in range(2):
        for dt, _ in gpu.advance(INTERVAL_NS, cfl=0.25):
            orc.step(secs(dt))
            dts.append(dt)
    assert sum(dts) == 2 * INTERVAL_NS and len(set(dts)) >= 3, dts
    p_o, p_g = orc.particles()[:, :3], gpu.download_particles()[:, :3]
    d = np.abs(p_o - p_g).max(axis=1)
    assert np.isfinite(p_g).all()
    assert np.quantile(d, 0.999) <= 1e-2, (np.quantile(d, 0.999), d.max())
    v_o = np.c_[orc.particles(O.ARR_ROWX)[:, 3], orc.particles(O.ARR_ROWY)[:, 3], orc.particles(O.ARR_ROWZ)[:, 3]].astype(np.float64)
    v_g = np.c_[gpu.download_particles(F.TAP_VX)[:, 3], gpu.download_particles(F.TAP_VY)[:, 3], gpu.download_particles(F.TAP_VZ)[:, 3]].astype(np.float64)
    ke_o, ke_g = (v_o ** 2).sum(), (v_g ** 2).sum()
    assert abs(ke_o - ke_g) <= 1e-3 * ke_o
    assert np.abs(v_o.sum(0) - v_g.sum(0)).max() <= 1e-3 * np.abs(v_o).sum(0).max()


def test_refusals():
    f = scene_fluid()
    f.step()
    for args in [dict(cfl=0.0), dict(cfl=17.0), dict(cfl=float("nan")), dict(max_dt_ns=10, min_dt_ns=11), dict(min_dt_ns=0)]:
        with pytest.raises(F.BlubError, match="error 1"):
            f.plan_substep(INTERVAL_NS, **args)
    with pytest.raises(F.BlubError, match="error 1"):
        f.plan_substep(0)
    launches = blub_b200.kernel_launch_count()
    with pytest.raises(F.BlubError, match="error 1"):
        f.plan_substep(INTERVAL_NS, cfl=-1.0)
    assert blub_b200.kernel_launch_count() == launches  # refused before anything is launched
    with pytest.raises(F.BlubError, match="error 6.*min_dt_ns"):  # a step below min_dt_ns: nothing is stepped
        f.advance(INTERVAL_NS, cfl=1e-6)
    assert f.step_count == 1
    f.step_stages(F.DT_120HZ, 0, 5)
    for call in (lambda: f.max_particle_velocity(), lambda: f.plan_substep(INTERVAL_NS)):
        with pytest.raises(F.BlubError, match="error 1.*inside a step"):
            call()
    f.step_stages(F.DT_120HZ, 5, 14)
    f.plan_substep(INTERVAL_NS)
    slab = blub_b200.HybridFluid.create_slab(32, 32, 16, 1000, 0, 2)
    for call in (lambda: slab.max_particle_velocity(), lambda: slab.plan_substep(INTERVAL_NS)):
        with pytest.raises(F.BlubError, match="error 1.*z-slab"):
            call()


def test_runner_cfl_matches_python_advance(tmp_path):
    assert os.path.exists(RUNNER), "blub_run is built by python -m blub_b200.build"
    stats, dump = str(tmp_path / "stats.json"), str(tmp_path / "p.f32")
    res = subprocess.run([RUNNER, util.scene_path("dam_small"), "--steps", "5", "--batch", "2", "--cfl", "0.5", "--stats", stats, "--dump", dump],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    ts = json.load(open(stats))["time_stepping"]
    assert abs(ts["cfl"] - 0.5) < 1e-9 and ts["interval_ns"] == INTERVAL_NS and ts["min_dt_ns"] == INTERVAL_NS // 256
    assert len(ts["intervals"]) == 5
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    for rec in ts["intervals"]:
        assert sum(rec["dt_ns"]) == INTERVAL_NS and len(rec["max_velocity"]) == len(rec["dt_ns"])
        plans = f.advance(INTERVAL_NS, cfl=0.5)
        assert [dt for dt, _ in plans] == rec["dt_ns"]
        assert np.array_equal(np.float32([v for _, v in plans]), np.float32(rec["max_velocity"]))
    assert sum(len(r["dt_ns"]) for r in ts["intervals"]) > 5
    got = np.fromfile(dump, dtype=np.float32).reshape(-1, 4)
    assert np.array_equal(got.view(np.uint32), f.download_particles().view(np.uint32))
