"""CFL substep rule (blub_cfl_substep_ns, host only) against its Python restatement in tests/cfl_ref.py.  No GPU needed."""
import ctypes as C
import math

import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import cfl_ref

INVALID, UNSTABLE = 1, F.BLUB_ERR_UNSTABLE
G = (0.0, -981.0, 0.0)  # 9.81 m/s^2 at 1 cm cells


def lib_substep(remaining_ns, v, g, cfl, max_dt_ns, min_dt_ns, reserved=0):
    """(return code, dt_ns, last error) of the library's rule."""
    ts = F.TimeStepping(float(cfl), int(reserved), int(max_dt_ns), int(min_dt_ns))
    out = C.c_uint64(12345)
    rc = F.lib().blub_cfl_substep_ns(int(remaining_ns), F._f3(v), F._f3(g), C.byref(ts), C.byref(out))
    return rc, int(out.value), F.lib().blub_last_error().decode()


def ref_substep(remaining_ns, v, g, cfl, max_dt_ns, min_dt_ns, reserved=0):
    try:
        return 0, cfl_ref.substep_ns(remaining_ns, v, g, cfl, max_dt_ns, min_dt_ns, reserved)
    except ValueError:
        return INVALID, None
    except cfl_ref.Unstable:
        return UNSTABLE, None


def agree(*args, **kw):
    rc, dt, err = lib_substep(*args, **kw)
    rrc, rdt = ref_substep(*args, **kw)
    assert rc == rrc, (args, rc, rrc, err)
    if rc == 0:
        assert dt == rdt, (args, dt, rdt)
    return rc, dt, err


def test_no_speed_takes_the_whole_remaining_time_up_to_max_dt():
    # s = 0 (no velocity, no gravity): d = +inf, so d_ns is max_dt_ns
    assert agree(1000, (0, 0, 0), (0, 0, 0), 1.0, 1000, 1)[1] == 1000
    assert agree(999, (0, 0, 0), (0, 0, 0), 1.0, 1000, 1)[1] == 999
    assert agree(1000, (0, 0, 0), (0, 0, 0), 1.0, 400, 1)[1] == 400  # R >= 2 d
    assert agree(700, (0, 0, 0), (0, 0, 0), 1.0, 400, 1)[1] == 350  # d < R < 2 d
    assert agree(701, (-0.0, 0, 0), (0, 0, 0), 1.0, 400, 1)[1] == 351  # odd R: R - R // 2


def test_gravity_margin_alone():
    # u = 0: s = sqrt(5 |g|) = sqrt(4905) cells/s; C = 1 gives d = 14.278... ms
    d_ns = math.floor(1.0 / math.sqrt(5.0 * 981.0) * 1e9)
    assert cfl_ref.cfl_step_ns((0, 0, 0), G, 1.0, 10 ** 12) == d_ns
    assert agree(10 ** 9, (0, 0, 0), G, 1.0, 10 ** 12, 1)[1] == d_ns
    # the norm of the gravity, not one component
    g3 = (300.0, -400.0, 1200.0)  # |g| = 1300
    assert agree(10 ** 9, (0, 0, 0), g3, 1.0, 10 ** 12, 1)[1] == math.floor(1e9 / math.sqrt(6500.0))


@pytest.mark.parametrize("remaining", [1, 2, 999_999, 1_000_000, 1_000_001, 1_500_000, 1_999_999, 2_000_000, 2_000_001, 8_333_333])
def test_remaining_time_cases(remaining):
    # u = 1000 cells/s, no gravity, C = 1: d = 1 ms exactly
    v = (1000.0, -20.0, 3.0)
    rc, dt, _ = agree(remaining, v, (0, 0, 0), 1.0, 10 ** 9, 1)
    assert rc == 0
    d = 1_000_000
    if remaining <= d:
        assert dt == remaining
    elif remaining < 2 * d:
        assert dt == remaining - remaining // 2 and dt <= d and remaining - dt <= d
    else:
        assert dt == d


def test_largest_axis_sets_the_step():
    for axis in range(3):
        v = [1.0, 1.0, 1.0]
        v[axis] = -250.0  # |v| per axis
        assert agree(10 ** 9, v, (0, 0, 0), 0.5, 10 ** 9, 1)[1] == 2_000_000


def test_saturation_at_huge_steps():
    tiny = float(np.float32(1e-45))  # the smallest denormal: d = 7e44 s, far beyond 2^64 ns
    assert agree(2 ** 64 - 1, (tiny, 0, 0), (0, 0, 0), 16.0, 2 ** 64 - 1, 1)[1] == 2 ** 64 - 1
    assert agree(2 ** 64 - 1, (0, 0, 0), (0, 0, 0), 1.0, 2 ** 64 - 1, 2 ** 64 - 1)[1] == 2 ** 64 - 1
    assert agree(5, (tiny, 0, 0), (0, 0, 0), 1.0, 2 ** 63, 1)[1] == 5
    # just below 2^64 ns: floor, then the max_dt_ns clamp
    v = 1.0 / 1.8e10  # d = 1.8e10 s = 1.8e19 ns < 2^64
    assert 1.7e19 < cfl_ref.cfl_step_ns((v, 0, 0), (0, 0, 0), 1.0, 2 ** 64 - 1) < 2 ** 64 - 1
    assert agree(10 ** 19, (v, 0, 0), (0, 0, 0), 1.0, 2 ** 64 - 1, 1)[1] == 10 ** 19
    assert agree(2 ** 64 - 1, (v, 0, 0), (0, 0, 0), 1.0, 2 ** 64 - 1, 1)[1] == 2 ** 63  # d < R < 2 d without overflowing 2 d


def test_min_dt_refusal_names_the_case_and_the_velocity():
    v = (1000.0, 0.0, 0.0)  # d = 1 ms
    assert agree(10 ** 9, v, (0, 0, 0), 1.0, 10 ** 9, 1_000_000)[1] == 1_000_000  # d_ns == min_dt_ns is allowed
    rc, _, err = agree(10 ** 9, v, (0, 0, 0), 1.0, 10 ** 9, 1_000_001)
    assert rc == UNSTABLE and "min_dt_ns" in err and "1000" in err
    with pytest.raises(F.BlubError, match="error 6"):
        F.cfl_substep_ns(10 ** 9, v, (0, 0, 0), 1.0, 10 ** 9, 1_000_001)


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_non_finite_velocity_is_unstable(bad):
    for axis in range(3):
        v = [1.0, 2.0, 3.0]
        v[axis] = bad
        rc, _, err = agree(1000, v, G, 1.0, 1000, 1)
        assert rc == UNSTABLE and "not finite" in err and ("inf" in err or "nan" in err)


@pytest.mark.parametrize("config", [
    dict(cfl=0.0), dict(cfl=-1.0), dict(cfl=16.0001), dict(cfl=float("nan")), dict(cfl=float("inf")), dict(reserved=1),
    dict(min_dt_ns=0), dict(min_dt_ns=11, max_dt_ns=10), dict(max_dt_ns=0, min_dt_ns=0), dict(remaining=0), dict(g=(0.0, float("nan"), 0.0)),
    dict(g=(float("inf"), 0.0, 0.0)),
])
def test_bad_configs_are_refused(config):
    args = dict(remaining=1000, v=(1.0, 2.0, 3.0), g=G, cfl=1.0, max_dt_ns=1000, min_dt_ns=1, reserved=0)
    args.update(config)
    rc, dt, _ = agree(args["remaining"], args["v"], args["g"], args["cfl"], args["max_dt_ns"], args["min_dt_ns"], reserved=args["reserved"])
    assert rc == INVALID and dt == 12345  # the output is left alone


def test_config_edges_are_accepted():
    assert agree(1000, (0, 0, 0), (0, 0, 0), 16.0, 1000, 1000)[0] == 0
    assert agree(1000, (0, 0, 0), (0, 0, 0), float(np.float32(1e-30)), 1000, 1)[0] == 0


def test_null_arguments_are_refused():
    ts = F.TimeStepping(1.0, 0, 1000, 1)
    out = C.c_uint64(0)
    L = F.lib()
    assert L.blub_cfl_substep_ns(1000, None, F._f3(G), C.byref(ts), C.byref(out)) == INVALID
    assert L.blub_cfl_substep_ns(1000, F._f3((0, 0, 0)), None, C.byref(ts), C.byref(out)) == INVALID
    assert L.blub_cfl_substep_ns(1000, F._f3((0, 0, 0)), F._f3(G), None, C.byref(out)) == INVALID
    assert L.blub_cfl_substep_ns(1000, F._f3((0, 0, 0)), F._f3(G), C.byref(ts), None) == INVALID
    assert L.blub_fluid_plan_substep(None, 1000, C.byref(ts), C.byref(out), None) == INVALID
    assert L.blub_fluid_max_particle_velocity(None, F._f3((0, 0, 0))) == INVALID


def test_substeps_cover_random_intervals_exactly():
    """With a fixed velocity the loop of advance covers any interval exactly, and no substep is longer than d_ns."""
    rng = np.random.default_rng(7)
    for _ in range(400):
        v = rng.uniform(0, 2000, 3).astype(np.float32) * np.float32(rng.choice([0, 1]))
        g = rng.normal(0, 600, 3).astype(np.float32)
        cfl = float(np.float32(rng.uniform(0.05, 4.0)))
        interval = int(rng.integers(1, 10 ** 8))
        max_dt = int(rng.integers(1, 2 * interval + 2))
        min_dt = max(1, interval // 256)
        d_ns = cfl_ref.cfl_step_ns(v, g, cfl, max_dt)
        done, dts = 0, []
        while done < interval:
            rc, dt, err = agree(interval - done, v, g, cfl, max_dt, min(min_dt, max_dt))
            if rc == UNSTABLE:
                assert d_ns < min(min_dt, max_dt) and not dts
                break
            assert rc == 0 and 1 <= dt <= d_ns, (dt, d_ns)
            dts.append(dt)
            done += dt
        else:
            assert sum(dts) == interval
            # a sliver never ends an interval: only the last two substeps may be shorter than d_ns
            assert all(dt == d_ns for dt in dts[:-2]), dts
            assert len(dts) <= math.ceil(interval / d_ns) + 1


def test_random_arguments_agree_with_the_restatement():
    rng = np.random.default_rng(11)
    for _ in range(3000):
        v = (rng.standard_normal(3) * 10.0 ** rng.uniform(-3, 6, 3)).astype(np.float32)
        g = (rng.standard_normal(3) * 10.0 ** rng.uniform(-2, 4)).astype(np.float32) * np.float32(rng.choice([0, 1]))
        cfl = float(np.float32(rng.uniform(0.01, 16.0)))
        remaining = int(rng.integers(1, 2 ** 40))
        max_dt = int(rng.integers(1, 2 ** 40))
        min_dt = int(rng.integers(1, max_dt + 1)) if rng.random() < 0.3 else 1
        agree(remaining, v, g, cfl, max_dt, min_dt)


@pytest.mark.parametrize("args", [["--cfl", "0"], ["--cfl", "16.5"], ["--cfl", "nan"], ["--cfl", "1", "--load-state", "missing.blub"]])
def test_runner_refuses_bad_cfl_options_before_any_device_work(args):
    import os
    import subprocess

    from tests import util
    runner = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
    res = subprocess.run([runner, util.scene_path("dam_small")] + args, capture_output=True, text=True, timeout=60)
    assert res.returncode == 2, res.stdout + res.stderr
    assert "--cfl" in res.stderr


def test_python_wrapper_defaults():
    # max_dt_ns defaults to the remaining time, min_dt_ns to 1
    assert F.cfl_substep_ns(8_333_333, (0, 0, 0), (0, 0, 0)) == 8_333_333
    assert F.cfl_substep_ns(8_333_333, (500.0, 0, 0), (0, 0, 0), cfl=1.0) == 2_000_000
