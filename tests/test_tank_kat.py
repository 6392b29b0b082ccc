"""Moving tanks on the host (no GPU): the closed-form frame of a prescribed motion against an independent evaluation, the step constants
against NumPy float64, the refusals, the scene key and the CFL bound under a frame."""
import json
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from blub_b200 import fluid as F
from tests import tank_ref as T
from tests import util

MOTION = {"pivot": (16.0, 12.5, 15.0),
          "translations": [{"direction": (1.0, 0.0, 0.0), "amplitude": 3.0, "frequency": 0.7, "phase": 0.3},
                           {"direction": (0.0, 0.6, 0.8), "amplitude": 1.5, "frequency": 1.9, "phase": -1.1}],
          "rotation": {"axis": (0.0, 0.0, 1.0), "amplitude": 0.35, "frequency": 0.45, "phase": 0.2, "rate": 0.25}}
OBLIQUE = dict(MOTION, rotation={"axis": tuple(np.array([1.0, 2.0, -2.0]) / 3.0), "amplitude": 0.5, "frequency": 1.3, "phase": 0.9, "rate": -0.4})
GRAVITY = np.array([0.0, -981.0, 0.0], dtype=np.float32)


def _translation(m, t):
    x = np.zeros(3)
    for tr in m["translations"]:
        x += tr["amplitude"] * np.asarray(tr["direction"]) * math.sin(2 * math.pi * tr["frequency"] * t + tr["phase"])
    return x


def _rotation(m, t):
    r = m["rotation"]
    theta = r["amplitude"] * math.sin(2 * math.pi * r["frequency"] * t + r["phase"]) + r["rate"] * t
    return Rotation.from_rotvec(theta * np.asarray(r["axis"])).as_matrix()


def _d1(f, t, h):
    """Five-point central first derivative."""
    return (-f(t + 2 * h) + 8 * f(t + h) - 8 * f(t - h) + f(t - 2 * h)) / (12 * h)


def _d2(f, t, h):
    """Five-point central second derivative."""
    return (-f(t + 2 * h) + 16 * f(t + h) - 30 * f(t) + 16 * f(t - h) - f(t - 2 * h)) / (12 * h * h)


def _omega(m, t):
    """omega in tank axes from the skew part of R' R^T (world axes), rotated back: omega_tank = R^T omega_world."""
    R = _rotation(m, t)
    W = _d1(lambda s: _rotation(m, s), t, 1e-3) @ R.T
    return R.T @ np.array([W[2, 1] - W[1, 2], W[0, 2] - W[2, 0], W[1, 0] - W[0, 1]]) / 2


def _close(a, b, rel=1e-6):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.abs(a - b).max() <= rel * max(np.abs(b).max(), 1.0), (a, b)


@pytest.mark.parametrize("motion", [MOTION, OBLIQUE], ids=["z_axis", "oblique"])
@pytest.mark.parametrize("t", [0.0, 0.37, 2.5, 11.0])
def test_frame_at_matches_independent_evaluation(motion, t):
    f = F.tank_frame_at(motion, t)
    _close(f["rotation"], _rotation(motion, t))
    _close(f["angular_velocity"], _omega(motion, t))
    _close(f["angular_acceleration"], _d1(lambda s: _omega(motion, s), t, 1e-3))
    _close(f["acceleration"], _d2(lambda s: _translation(motion, s), t, 1e-3))
    assert np.array_equal(f["pivot"], np.asarray(motion["pivot"]))


@pytest.mark.parametrize("motion", [MOTION, OBLIQUE], ids=["z_axis", "oblique"])
@pytest.mark.parametrize("dt", [F.DT_120HZ, 1e-3, 0.05])
def test_step_constants_within_one_ulp_of_float64(motion, dt):
    for t in (0.0, 0.8, 3.3):
        frame = F.tank_frame_at(motion, t)
        got = F.tank_step_constants(frame, GRAVITY, dt)
        ref = T.step_constants(frame, GRAVITY, dt)
        for name in ("gravity", "coriolis", "force", "pivot"):
            r = np.asarray(ref[name], dtype=np.float64)
            ulp = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64)
            assert (np.abs(got[name].astype(np.float64) - r) <= ulp).all(), name
        assert got["rotating"]
        assert np.allclose(got["coriolis"].astype(np.float64) @ got["coriolis"].T.astype(np.float64), np.eye(3), atol=1e-6)


def test_identity_frame_is_exact():
    g = np.array([0.25, -981.0, 3.0e-3], dtype=np.float32)
    c = F.tank_step_constants({"pivot": (3.0, 4.0, 5.0)}, g, F.DT_120HZ)
    assert np.array_equal(c["gravity"].view(np.uint32), g.view(np.uint32))
    assert np.array_equal(c["coriolis"], np.eye(3, dtype=np.float32)) and not c["force"].any() and not c["rotating"]


def test_translation_only_frame_does_not_rotate():
    R = Rotation.from_euler("xyz", [0.1, -0.2, 0.3]).as_matrix()
    c = F.tank_step_constants({"rotation": R, "acceleration": (5.0, -2.0, 1.0)}, GRAVITY, F.DT_120HZ)
    assert not c["rotating"] and np.array_equal(c["coriolis"], np.eye(3, dtype=np.float32)) and not c["force"].any()
    ref = R.T @ (GRAVITY.astype(np.float64) - np.array([5.0, -2.0, 1.0]))
    assert np.array_equal(c["gravity"], ref.astype(np.float32))


def _refused(fn, *args):
    with pytest.raises(F.BlubError) as e:
        fn(*args)
    assert e.value.code == 1
    return e


BAD_FRAMES = [
    {"rotation": np.diag([1.0, 1.0, -1.0])},                 # det -1
    {"rotation": np.diag([1.0, 1.0, 1.00001])},              # not orthonormal
    {"rotation": np.eye(3) * 0.5},
    {"acceleration": (math.nan, 0, 0)},
    {"angular_velocity": (0, math.inf, 0)},
    {"angular_acceleration": (0, 0, -math.inf)},
    {"pivot": (math.nan, 0, 0)},
    {"rotation": np.where(np.eye(3) > 0, math.inf, 0.0)},
]


@pytest.mark.parametrize("k", range(len(BAD_FRAMES)))
def test_malformed_frames_are_refused(k):
    _refused(F.tank_step_constants, BAD_FRAMES[k], GRAVITY, F.DT_120HZ)
    _refused(F.tank_cfl_substep_ns, 8333333, (1, 1, 1), GRAVITY, BAD_FRAMES[k], (32, 32, 32))


def test_bad_gravity_and_dt_are_refused():
    for g, dt in (((math.nan, 0, 0), F.DT_120HZ), ((0, math.inf, 0), F.DT_120HZ), (GRAVITY, 0.0), (GRAVITY, -1.0), (GRAVITY, math.inf)):
        _refused(F.tank_step_constants, {}, g, dt)


def _motion(**changes):
    m = json.loads(json.dumps(MOTION))
    for key, value in changes.items():
        if key.startswith("tr_"):
            m["translations"][0][key[3:]] = value
        elif key.startswith("rot_"):
            m["rotation"][key[4:]] = value
        else:
            m[key] = value
    return m


BAD_MOTIONS = [
    _motion(pivot=(math.nan, 0, 0)), _motion(tr_direction=(1.0, 1.0, 0.0)), _motion(tr_direction=(0.0, 0.0, 0.0)),
    _motion(tr_amplitude=math.inf), _motion(tr_frequency=-1.0), _motion(tr_phase=math.nan), _motion(rot_axis=(0.0, 0.0, 2.0)),
    _motion(rot_amplitude=math.nan), _motion(rot_frequency=-0.5), _motion(rot_phase=math.inf), _motion(rot_rate=math.nan),
    _motion(translations=MOTION["translations"] * 3),
]


@pytest.mark.parametrize("k", range(len(BAD_MOTIONS)))
def test_malformed_motions_are_refused(k):
    _refused(F.tank_frame_at, BAD_MOTIONS[k], 0.5)


def test_reserved_time_and_nulls_are_refused():
    m = F.TankMotion.from_dict(MOTION)
    m.reserved = 1
    _refused(F.tank_frame_at, m, 0.0)
    _refused(F.tank_frame_at, MOTION, math.nan)
    L = F.lib()
    import ctypes as C
    fr, k, ts = F.TankFrame.from_dict({}), F.TankStepConstants(), F.time_stepping(1.0, 10, 1)
    out, mot = C.c_uint64(), F.TankMotion.from_dict(MOTION)
    d = (C.c_uint32 * 3)(32, 32, 32)
    assert L.blub_tank_frame_at(None, 0.0, C.byref(fr)) == 1 and L.blub_tank_frame_at(C.byref(mot), 0.0, None) == 1
    assert L.blub_tank_step_constants(None, F._f3(GRAVITY), 0.01, C.byref(k)) == 1
    assert L.blub_tank_step_constants(C.byref(fr), None, 0.01, C.byref(k)) == 1
    assert L.blub_tank_step_constants(C.byref(fr), F._f3(GRAVITY), 0.01, None) == 1
    v = F._f3((1, 1, 1))
    assert L.blub_tank_cfl_substep_ns(10, None, F._f3(GRAVITY), C.byref(fr), d, C.byref(ts), C.byref(out)) == 1
    assert L.blub_tank_cfl_substep_ns(10, v, None, C.byref(fr), d, C.byref(ts), C.byref(out)) == 1
    assert L.blub_tank_cfl_substep_ns(10, v, F._f3(GRAVITY), C.byref(fr), None, C.byref(ts), C.byref(out)) == 1
    assert L.blub_tank_cfl_substep_ns(10, v, F._f3(GRAVITY), C.byref(fr), d, None, C.byref(out)) == 1
    assert L.blub_tank_cfl_substep_ns(10, v, F._f3(GRAVITY), C.byref(fr), d, C.byref(ts), None) == 1
    assert L.blub_fluid_set_tank_frame(None, C.byref(fr)) == 1
    assert L.blub_fluid_tank_frame(None, C.byref(fr)) == 0
    has = C.c_int32()
    path = util.scene_path("dam_small").encode()
    assert L.blub_scene_tank_motion(None, C.byref(mot), C.byref(has)) == 1
    assert L.blub_scene_tank_motion(path, None, C.byref(has)) == 1 and L.blub_scene_tank_motion(path, C.byref(mot), None) == 1


# --- the scene key -------------------------------------------------------------------------------------------------------------------

SCENE_MOTION = {"pivot": {"x": 0.16, "y": 0.1, "z": 0.16},
                "translations": [{"direction": {"x": 2.0, "y": 0.0, "z": 0.0}, "amplitude": 0.02, "frequency": 0.8, "phase": 0.5},
                                 {"direction": {"x": 0.0, "y": 1.0, "z": 1.0}, "amplitude": 0.01, "frequency": 2.0}],
                "rotation": {"axis": {"x": 0.0, "y": 0.0, "z": 3.0}, "amplitude": 0.2, "frequency": 0.5, "rate": 0.1}}


def _scene(tmp_path, motion, name="tank.json"):
    with open(util.scene_path("dam_small")) as fh:
        s = json.load(fh)
    if motion is not None:
        s["fluid"]["tank_motion"] = motion
    p = tmp_path / name
    p.write_text(json.dumps(s))
    return str(p)


def test_scene_tank_motion_in_grid_units(tmp_path):
    assert F.scene_tank_motion(util.scene_path("dam_small")) is None
    m = F.scene_tank_motion(_scene(tmp_path, SCENE_MOTION))
    f32 = np.float32
    assert m["pivot"] == tuple(float(f32(v) / f32(0.01)) for v in (0.16, 0.1, 0.16))
    t0, t1 = m["translations"]
    assert t0["direction"] == (1.0, 0.0, 0.0) and t0["amplitude"] == float(f32(0.02) / f32(0.01))
    assert t0["frequency"] == float(f32(0.8)) and t0["phase"] == float(f32(0.5))
    assert np.allclose(t1["direction"], (0.0, 2 ** -0.5, 2 ** -0.5), rtol=0, atol=1e-15) and t1["phase"] == 0.0
    r = m["rotation"]
    assert r["axis"] == (0.0, 0.0, 1.0) and r["amplitude"] == float(f32(0.2)) and r["phase"] == 0.0 and r["rate"] == float(f32(0.1))
    m = F.scene_tank_motion(_scene(tmp_path, {"pivot": {"x": 0.1, "y": 0.1, "z": 0.1}}))
    assert m["translations"] == [] and m["rotation"]["rate"] == 0.0 and m["rotation"]["amplitude"] == 0.0
    assert F.tank_step_constants(F.tank_frame_at(m, 3.0), GRAVITY, F.DT_120HZ)["rotating"] is False


def _bad(**kw):
    m = json.loads(json.dumps(SCENE_MOTION))
    for k, v in kw.items():
        if k == "tr":
            m["translations"][0].update(v)
        elif k == "rot":
            m["rotation"].update(v)
        else:
            m[k] = v
    return m


BAD_SCENES = [
    "not an object", {"translations": []}, _bad(pivot={"x": 1.0, "y": 1.0}), _bad(pivot={"x": 1e39, "y": 0, "z": 0}),
    _bad(translations={}), _bad(translations=SCENE_MOTION["translations"] * 3), _bad(translations=[1.0]),
    _bad(tr={"direction": {"x": 0.0, "y": 0.0, "z": 0.0}}), _bad(tr={"amplitude": "big"}), _bad(tr={"frequency": -1.0}),
    _bad(tr={"amplitude": 1e39}), _bad(rot={"axis": {"x": 0.0, "y": 0.0, "z": 0.0}}), _bad(rot={"rate": 1e39}),
    _bad(rot={"frequency": -2.0}), _bad(rotation=[0.0]),
]


@pytest.mark.parametrize("k", range(len(BAD_SCENES)))
def test_malformed_scene_values_are_refused(tmp_path, k):
    path = _scene(tmp_path, BAD_SCENES[k])
    for fn in (F.scene_tank_motion, F.scene_info):
        with pytest.raises(F.BlubError) as e:
            fn(path)
        assert e.value.code == 5


# --- the CFL bound ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("v", [(0.0, 0.0, 0.0), (12.5, -3.0, 40.0), (1e-3, 2e-3, 0.0)])
def test_cfl_without_a_frame_is_the_rule(v):
    for cfl in (0.5, 1.0, 3.0):
        assert F.tank_cfl_substep_ns(8333333, v, GRAVITY, None, (64, 32, 48), cfl) == F.cfl_substep_ns(8333333, v, GRAVITY, cfl)


@pytest.mark.parametrize("motion", [MOTION, OBLIQUE, {"pivot": (3.0, 4.0, 5.0), "translations": MOTION["translations"]}],
                         ids=["z_axis", "oblique", "translation"])
@pytest.mark.parametrize("v", [(0.0, 0.0, 0.0), (12.5, -3.0, 40.0)])
def test_cfl_under_a_frame_uses_the_bound(motion, v):
    for t in (0.0, 1.7):
        frame = F.tank_frame_at(motion, t)
        vv, gg = T.cfl_inputs(v, GRAVITY, frame, (64, 32, 48))
        for cfl in (0.5, 2.0):
            got = F.tank_cfl_substep_ns(8333333, v, GRAVITY, frame, (64, 32, 48), cfl)
            assert got == F.cfl_substep_ns(8333333, vv, gg, cfl)
            assert got <= F.cfl_substep_ns(8333333, v, GRAVITY, cfl)


def test_cfl_under_a_frame_refuses_as_the_rule():
    frame = F.tank_frame_at(MOTION, 0.3)
    with pytest.raises(F.BlubError) as e:
        F.tank_cfl_substep_ns(8333333, (math.nan, 0, 0), GRAVITY, frame, (32, 32, 32))
    assert e.value.code == F.BLUB_ERR_UNSTABLE
    with pytest.raises(F.BlubError) as e:
        F.tank_cfl_substep_ns(8333333, (1e9, 0, 0), GRAVITY, frame, (32, 32, 32), min_dt_ns=1000)
    assert e.value.code == F.BLUB_ERR_UNSTABLE
    _refused(F.tank_cfl_substep_ns, 0, (1, 1, 1), GRAVITY, frame, (32, 32, 32))
    _refused(F.tank_cfl_substep_ns, 100, (1, 1, 1), GRAVITY, frame, (32, 32, 32), 0.0)


def test_kernel_restatement_applies_the_frame():
    """A particle of a world at rest in a spinning tank moves on its circle, and the force term of a spin-up adds -alpha x r dt."""
    frame = {"angular_velocity": (0.0, 0.0, 2.0), "pivot": (16.0, 16.0, 16.0)}
    c = F.tank_step_constants(frame, (0, 0, 0), F.DT_120HZ)
    pos = np.array([[20.0, 16.0, 16.0, 0.0]], dtype=np.float32)
    rows = np.zeros((3, 1, 4), dtype=np.float32)
    rows[1, 0, 3] = -8.0  # -omega x r at r = (4, 0, 0)
    out = T.apply_frame_kernel(pos, rows, c["coriolis"], c["force"], c["pivot"])
    # world at rest: Coriolis and centrifugal forces add up to the centripetal acceleration v^2 / r = 16 towards the pivot, speed kept
    assert abs(np.hypot(out[0, 0, 3], out[1, 0, 3]) - 8.0) < 1e-2 and abs(out[0, 0, 3] + 16.0 * F.DT_120HZ) < 1e-3
    c = F.tank_step_constants({"angular_acceleration": (0.0, 0.0, 3.0), "pivot": (16.0, 16.0, 16.0)}, (0, 0, 0), F.DT_120HZ)
    out = T.apply_frame_kernel(pos, np.zeros((3, 1, 4), dtype=np.float32), c["coriolis"], c["force"], c["pivot"])
    assert np.allclose(out[:, 0, 3], [0.0, -3.0 * 4.0 * F.DT_120HZ, 0.0], atol=1e-7)
