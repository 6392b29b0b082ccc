"""GPU: whitewater (DESIGN.md §8 "Whitewater").  The liquid does not see it; the pass equals tests/whitewater_ref.py bit for bit on a dam
break past the first wave, with a moving solid and with sources; runs are reproducible and graph replay equals eager launches; a version-1024
file resumes bit for bit; the capacity holds; off launches nothing and refusals change nothing; the physics is sane."""
import struct

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import whitewater_ref as W
from tests import util
from tests.test_gpu_bodies import DOUBLE_DAM_BODIES
from tests.test_gpu_loads import BOX, Solid
from tests.test_gpu_state import assert_identical, snapshot
from tests.util import DT

pytestmark = pytest.mark.gpu
f32 = np.float32
# generous rates, so that the small scenes make plenty of all three kinds
HIGH = {"trapped_air_rate": 600.0, "wave_crest_rate": 600.0, "trapped_air_range": (2.0, 10.0), "energy_range": (1.0, 100.0)}


def gravity_of(scene):
    info = F.scene_info(scene)
    return np.array([f32(info.gravity[k]) / f32(info.grid_to_world_scale) for k in range(3)], dtype=f32)


def make(scene, graph=True, bodies=False):
    f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    f.set_graph_replay(graph)
    if bodies:
        f.set_bodies(DOUBLE_DAM_BODIES)
    return f


def ww_state(f):
    pos, vel = f.whitewater_raw()
    c = f.whitewater_counters
    return {"pos": pos, "vel": vel, "counters": [c["emitted"], c["removed"], c["refused"]]}


def state_sections(path):
    """A state file's header with the fields that differ between runs of the same liquid masked (format_version, num_stats, num_sections,
    header_crc) and its section payloads by id (a payload's CRC follows from it)."""
    data = open(path, "rb").read()
    header = bytearray(data[:144])
    header[8:12] = bytes(4)
    header[128:144] = bytes(16)
    out, at = {}, 144
    while at < len(data):
        sid, _, length = struct.unpack_from("<IIQ", data, at)
        assert sid not in out
        out[sid] = data[at + 16:at + 16 + length]
        at += 16 + length + 4
    return bytes(header), out


def assert_same_liquid_sections(a, b):
    """Everything but the statistics histories (sections 12 and 13: read back without blocking, so they depend on how far the host ran
    ahead) and the whitewater (section 22)."""
    ha, sa = state_sections(a)
    hb, sb = state_sections(b)
    assert ha == hb
    liquid = lambda s: {k: v for k, v in s.items() if k not in (12, 13, 22)}
    assert liquid(sa).keys() == liquid(sb).keys()
    for k in liquid(sa):
        x, y = sa[k], sb[k]
        if k == 14 and len(x) != len(y):  # 992 bytes in a version-2 file, 1056 with the source tags (all 0 here) in every later one
            x, y = sorted((x, y), key=len)
            assert len(x) == 992 and y[992:] == bytes(64)
            y = y[:992]
        assert x == y, k


CASES = [("dam_small", False, False), ("tap_small", False, False), ("dam_small", True, False), ("double_dam", False, True)]


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("scene, moving, bodies", CASES)
def test_the_liquid_does_not_see_the_whitewater(tmp_path, scene, moving, bodies, graph):
    runs = []
    for on in (False, True):
        f = make(scene, graph, bodies)
        if on:
            f.set_whitewater(100000, **HIGH)
        solid = Solid(f, BOX) if moving else None
        for _ in range(64):  # past the re-sorts every 8 steps and the rebinning at step 60
            if solid:
                solid.voxelize()
            f.step(DT)
        f.save_state(str(tmp_path / f"{on}.blub"))
        runs.append((snapshot(f), f))
    # the solver statistics history is read back without blocking and may drop samples while the host runs ahead: it is not liquid state
    for run in runs:
        run[0].pop("stats")
    assert_identical(dict(runs[0][0], stats=None), dict(runs[1][0], stats=None))
    assert runs[1][1].whitewater_counters["emitted"] > 0
    assert F.state_info(str(tmp_path / "True.blub")).format_version == 1024
    assert 22 in state_sections(str(tmp_path / "True.blub"))[1]
    assert_same_liquid_sections(str(tmp_path / "False.blub"), str(tmp_path / "True.blub"))


def check_pass(f, steps, vox=False):
    """steps consecutive steps, each split at the end of stage 5, the pass against the restatement."""
    s = f.whitewater()
    g = gravity_of(f._scene)
    kinds, removed = set(), 0
    for _ in range(steps):
        before = ww_state(f)
        step = f.step_count
        if getattr(f, "_solid", None):
            f._solid.voxelize()
        f.step_stages(DT, 0, 6)
        u = [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)]
        marker = f.download_grid(F.TAP_MARKER)
        vox_w = f.download_solid_voxels()[..., 3].astype(f32) if vox else None
        want = W.whitewater_pass(before, u, marker, vox_w, f32(DT), step, g, s)
        got = ww_state(f)
        assert got["counters"] == want["counters"], step
        assert got["pos"].tobytes() == want["pos"].tobytes(), step
        assert got["vel"].tobytes() == want["vel"].tobytes(), step
        kinds |= set(got["vel"][:, 3].view(np.uint32).tolist())
        removed = got["counters"][1]
        f.step_stages(DT, 6, 14)
    return kinds, removed


@pytest.mark.parametrize("scene, moving", [("dam_small", False), ("dam_small", True), ("tap_small", False)])
def test_the_pass_equals_the_restatement_bit_for_bit(scene, moving):
    f = make(scene)
    f._scene = util.scene_path(scene)
    f.set_whitewater(100000, **HIGH)
    f._solid = Solid(f, BOX) if moving else None
    for _ in range(70):  # the front has hit the far wall
        if f._solid:
            f._solid.voxelize()
        f.step(DT)
    kinds, removed = check_pass(f, 4, vox=moving)
    assert kinds == {W.SPRAY, W.FOAM, W.BUBBLE} and removed > 0, (kinds, removed)


def test_runs_are_reproducible_and_graph_replay_equals_eager():
    out = []
    for graph in (True, True, False):
        f = make("dam_small", graph)
        f.set_whitewater(100000, **HIGH)
        for _ in range(40):
            f.step(DT)
        st = ww_state(f)
        out.append((st["pos"].tobytes(), st["vel"].tobytes(), st["counters"]))
    assert out[0] == out[1] == out[2]


def test_a_version_1024_file_resumes_bit_for_bit(tmp_path):
    ref = make("dam_small")
    ref.set_whitewater(100000, **HIGH)
    for _ in range(50):
        ref.step(DT)
    a = make("dam_small")
    a.set_whitewater(100000, **HIGH)
    for _ in range(40):
        a.step(DT)
    a.save_state(str(tmp_path / "s.blub"))
    assert F.state_info(str(tmp_path / "s.blub")).format_version == 1024
    b = blub_b200.HybridFluid.from_state(str(tmp_path / "s.blub"))
    assert b.whitewater() == ref.whitewater()
    for _ in range(10):
        b.step(DT)
    want, got = snapshot(ref), snapshot(b)
    want.pop("stats"), got.pop("stats")  # read back without blocking: not liquid state (see above)
    assert_identical(dict(want, stats=None), dict(got, stats=None))
    sr, sb = ww_state(ref), ww_state(b)
    assert sr["pos"].tobytes() == sb["pos"].tobytes() and sr["vel"].tobytes() == sb["vel"].tobytes() and sr["counters"] == sb["counters"]


def test_turning_whitewater_off_saves_the_old_bytes(tmp_path):
    files = []
    for on in (False, True):
        f = make("dam_small")
        if on:
            f.set_whitewater(100000, **HIGH)
        for _ in range(20):
            f.step(DT)
        if on:
            f.set_whitewater(0)
        path = tmp_path / f"s{on}.blub"
        f.save_state(str(path))
        files.append(str(path))
    assert F.state_info(files[0]).format_version == F.state_info(files[1]).format_version
    assert 22 not in state_sections(files[1])[1]
    assert_same_liquid_sections(files[0], files[1])


def test_the_capacity_holds_and_the_refused_count_grows():
    f = make("dam_small")
    f.set_whitewater(300, **HIGH)
    for k in range(80):
        f.step(DT)
        if k % 10 == 9:
            c = f.whitewater_counters
            assert c["live"] <= 300
    c = f.whitewater_counters
    assert c["refused"] > 0 and c["live"] <= 300
    assert c["emitted"] - c["removed"] == c["live"]


def launches_of_a_step(f):
    f.synchronize()
    before = blub_b200.kernel_launch_count()
    f.step(DT)
    f.synchronize()
    return blub_b200.kernel_launch_count() - before


@pytest.mark.parametrize("graph", [True, False])
def test_off_launches_nothing_and_refusals_change_nothing(graph):
    never, again = make("dam_small", graph), make("dam_small", graph)
    again.set_whitewater(1000)
    again.step(DT)
    again.set_whitewater(0)
    never.step(DT)
    assert again.whitewater_counters == {"live": 0, "emitted": 0, "removed": 0, "refused": 0}
    # off is stored as an all-zero setting, whatever the other fields of a capacity-0 setting held
    off = F.Whitewater.from_dict(dict(F.WHITEWATER_DEFAULTS, max_num_particles=0, drag=float("nan"), buoyancy=float("inf")))
    F._check(again.L.blub_fluid_set_whitewater(again.h, F.C.byref(off)))
    assert bytes(F.Whitewater.from_dict(again.whitewater())) == bytes(F.Whitewater())
    for _ in range(2):
        assert launches_of_a_step(never) == launches_of_a_step(again)
    f = make("dam_small", graph)
    f.set_whitewater(1000)
    want = f.whitewater()
    bad = [{"drag": 1.5}, {"drag": float("nan")}, {"energy_range": (5.0, 5.0)}, {"trapped_air_rate": -1.0}, {"spray_below": 21},
           {"bubble_from": 28, "spray_below": 6}, {"lifetime_lo": 3.0, "lifetime_hi": 1.0}, {"max_per_cell": 17}]
    for change in bad:
        with pytest.raises(F.BlubError):
            f.set_whitewater(1000, **change)
        assert f.whitewater() == want
    with pytest.raises(F.BlubError):
        f.set_whitewater(F.WHITEWATER_MAX_PARTICLES + 1)
    f.step_stages(DT, 0, 6)
    with pytest.raises(F.BlubError):
        f.set_whitewater(500)
    assert f.whitewater() == want
    f.step_stages(DT, 6, 14)
    slab = blub_b200.HybridFluid.create_slab(32, 32, 32, 1000, 0, 2)
    with pytest.raises(F.BlubError):
        slab.set_whitewater(1000)
    assert slab.whitewater()["max_num_particles"] == 0


def test_physical_sanity_on_the_dam_break():
    f = make("dam_small")
    f.set_whitewater(200000, **HIGH)
    for _ in range(90):
        f.step(DT)
    p = f.whitewater_particles()
    marker = f.download_grid(F.TAP_MARKER)
    cell = lambda x: marker[x[:, 2].astype(int), x[:, 1].astype(int), x[:, 0].astype(int)]
    spray, foam, bubble = (p["kind"] == k for k in (W.SPRAY, W.FOAM, W.BUBBLE))
    assert spray.sum() > 0 and bubble.sum() > 0 and foam.sum() > 0, {k: int(v.sum()) for k, v in (("s", spray), ("f", foam), ("b", bubble))}
    # the marker after the step against where the particles are classified from: most spray is in AIR cells, most bubbles in FLUID ones
    assert (cell(p["position"][spray]) == W.AIR).mean() > 0.5
    assert (cell(p["position"][bubble]) == W.FLUID).mean() > 0.5
    assert np.median(p["position"][spray][:, 1]) > np.median(p["position"][bubble][:, 1])
    # foam moves with the liquid: split the next step after the pass, where u is still the projected grid velocity (stage 11 reuses it)
    f.step_stages(DT, 0, 6)
    u = [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)]
    p = f.whitewater_particles()
    foam = p["kind"] == W.FOAM
    fv = p["velocity"][foam]
    off = np.linalg.norm(fv - W.sample_u(u, p["position"][foam]), axis=1)
    assert np.median(off) < 0.2 * np.median(np.linalg.norm(fv, axis=1))
    f.step_stages(DT, 6, 14)


def test_a_still_basin_emits_nothing():
    f = make("filled_basin")
    f.set_whitewater(10000)
    for _ in range(100):
        f.step(DT)
    assert f.whitewater_counters["emitted"] == 0


def test_the_runner_equals_a_ctypes_run(tmp_path):
    import json
    import os
    import subprocess
    runner = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
    scene, stats, prefix = util.scene_path("dam_whitewater_small"), str(tmp_path / "stats.json"), str(tmp_path / "frame")
    res = subprocess.run([runner, scene, "--steps", "40", "--stats", stats, "--record", "60", prefix], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    assert f.whitewater() == F.scene_whitewater(scene)
    frames = sorted(p for p in os.listdir(tmp_path) if p.endswith(".whitewater.f32"))
    assert len(frames) == 20  # two steps per frame at 60 frames per second
    for _ in range(40):
        f.step(DT)
    assert json.load(open(stats))["whitewater"] == f.whitewater_counters
    pos, vel = f.whitewater_raw()
    got = np.fromfile(str(tmp_path / frames[-1]), dtype=np.float32).reshape(-1, 8)
    assert got.tobytes() == np.concatenate([pos, vel], axis=1).tobytes()
    assert f.whitewater_counters["emitted"] > 0
    # the renderer hand-off: the runner's --dump of the liquid after 64 steps is the same file with and without whitewater
    dumps = []
    for name in ("dam_small", "dam_whitewater_small"):
        dump = str(tmp_path / f"{name}.f32")
        res = subprocess.run([runner, util.scene_path(name), "--steps", "64", "--dump", dump], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        dumps.append(open(dump, "rb").read())
    assert len(dumps[0]) > 0 and dumps[0] == dumps[1]
