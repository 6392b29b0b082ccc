"""CPU: the whitewater rules (DESIGN.md §8 "Whitewater") on synthetic grids through the NumPy restatement, the scene key through the host-only
blub_scene_whitewater, and state files with section 22 through blub_state_info.  No GPU needed."""
import json
import struct

import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import whitewater_ref as W
from tests.flow_ref import Xoshiro
from tests.test_state_file import section
from tests.test_state_layout_kat import ACCEPTED, BASES, PAYLOADS, SUBSETS, accepted, info_rc, relabel, bases  # noqa: F401
from tests.util import DT, scene_path

f32 = np.float32
S = dict(F.WHITEWATER_DEFAULTS, max_num_particles=1000)
BLUB_ERR_PARSE = 5


def grid(shape=(24, 24, 24), level=12):
    """A tank (SOLID border) filled with FLUID below y = level and AIR above; zero velocity."""
    nz, ny, nx = shape
    m = np.full(shape, W.AIR, dtype=np.int8)
    m[:, :level, :] = W.FLUID
    m[0, :, :] = m[-1, :, :] = m[:, 0, :] = m[:, -1, :] = m[:, :, 0] = m[:, :, -1] = W.SOLID
    return m, [np.zeros(shape, dtype=f32) for _ in range(3)]


def emitted(u, m, s=S, step=7):
    _, count, _ = W.emit_counts(u, m, DT, step, s)
    return int(count.sum())


def test_a_liquid_at_rest_emits_nothing():
    m, u = grid()
    assert len(W.band(m)[0]) > 0
    assert emitted(u, m) == 0


def test_a_flat_surface_moving_along_itself_emits_nothing():
    m, u = grid()
    u[0][:] = f32(30.0)  # a uniform stream along x: no curl, and u . n = 0 on the flat surface
    lin, i_ta, i_wc, i_k = W.potentials(u, m, S)
    inner = i_k > 0
    assert inner.any() and not i_ta[inner].any() and not i_wc[inner].any()
    assert emitted(u, m) == 0


def test_an_outward_moving_crest_emits():
    m, u = grid()
    u[1][:] = f32(30.0)  # the surface moves up, along its outward normal
    lin, i_ta, i_wc, i_k = W.potentials(u, m, S)
    assert (i_wc > 0).any() and not i_ta[i_k > 0].any()
    assert emitted(u, m) > 0


def test_a_vortex_in_the_band_emits_by_trapped_air():
    m, u = grid()
    nz, ny, nx = m.shape
    z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    w = f32(4.0)  # rigid rotation about the z axis through (12, 12): curl 2w
    u[0][:] = (-w * (y + f32(0.5) - f32(12))).astype(f32)
    u[1][:] = (w * (x + f32(1.0) - f32(12))).astype(f32)
    lin, i_ta, i_wc, i_k = W.potentials(u, m, dict(S, wave_crest_rate=0.0))
    assert (i_ta > 0).any()
    assert emitted(u, m, dict(S, wave_crest_rate=0.0)) > 0


def test_the_ramps_are_zero_at_lo_and_one_at_hi():
    assert W.ramp(f32(5), 5, 20) == 0 and W.ramp(f32(20), 5, 20) == 1
    assert W.ramp(f32(4), 5, 20) == 0 and W.ramp(f32(21), 5, 20) == 1 and W.ramp(f32(12.5), 5, 20) == f32(0.5)


def test_the_classification_thresholds():
    m, _ = grid()
    s = dict(S, spray_below=6, bubble_from=20)
    nz, ny, nx = m.shape
    # a cell deep inside: 27 FLUID cells -> bubble; the level below the surface: 18 -> foam; the first AIR level: 9 -> foam; above: 0 -> spray
    pts = np.array([[12.5, 5.5, 12.5], [12.5, 11.5, 12.5], [12.5, 12.5, 12.5], [12.5, 13.5, 12.5]], dtype=f32)
    assert W.classify(m, pts, s).tolist() == [W.BUBBLE, W.FOAM, W.FOAM, W.SPRAY]
    assert W.fluid_count(m, *[np.array([int(v)]) for v in (12, 11, 12)]).tolist() == [18]
    # exactly at the thresholds: a = spray_below is not spray, a = bubble_from is a bubble
    assert W.classify(m, pts[2:3], dict(s, spray_below=9, bubble_from=9)).tolist() == [W.FOAM]
    assert W.classify(m, pts[2:3], dict(s, spray_below=10, bubble_from=10)).tolist() == [W.SPRAY]
    assert W.classify(m, pts[1:2], dict(s, spray_below=6, bubble_from=18)).tolist() == [W.BUBBLE]
    assert W.classify(m, pts[1:2], dict(s, spray_below=6, bubble_from=19)).tolist() == [W.FOAM]


def particle(x, v=(0, 0, 0), life=1.0, kind=W.SPRAY):
    return (np.array([[*x, life]], dtype=f32), np.array([[*v, np.array([kind], dtype=np.uint32).view(f32)[0]]], dtype=f32))


@pytest.mark.parametrize("case", ["lifetime", "low", "high", "solid cell", "solid volume", "survives"])
def test_every_removal_rule(case):
    m, u = grid()
    g = (0.0, -100.0, 0.0)
    vox = np.zeros(m.shape, dtype=f32)
    x, v, life = (12.5, 5.5, 12.5), (0, 0, 0), 1.0
    if case == "lifetime":  # foam ages by dt
        x, life = (12.5, 11.5, 12.5), DT / 2
    elif case == "low":  # spray falls below y = 1
        x, v = (12.5, 1.05, 12.5), (0, -30, 0)
        m[:, :, :] = W.AIR
    elif case == "high":
        x, v = (12.5, 22.9, 12.5), (0, 50, 0)
    elif case == "solid cell":
        m[12, 5, 13] = W.SOLID
        x, v = (12.9, 5.5, 12.5), (30, 0, 0)
    elif case == "solid volume":
        vox[12, 5, 12] = 1.0
    p, q = particle(x, v, life, W.FOAM if case == "lifetime" else W.SPRAY)
    pos, vel, removed = W.update(p, q, u, m, vox, DT, g, S)
    assert removed == (0 if case == "survives" else 1), case


def test_survivors_keep_their_order_and_only_foam_ages():
    m, u = grid()
    pts = np.array([[12.5, 5.5, 12.5, 2.0], [12.5, 11.5, 12.5, 2.0], [12.5, 20.5, 12.5, 2.0], [3.5, 3.5, 3.5, 2.0]], dtype=f32)
    vel = np.zeros((4, 4), dtype=f32)
    pos, v, removed = W.update(pts, vel, u, m, None, DT, (0, -10, 0), S)
    assert removed == 0 and np.array_equal(pos[:, 0], pts[:, 0])
    kinds = v[:, 3].view(np.uint32)
    assert kinds.tolist() == [W.BUBBLE, W.FOAM, W.SPRAY, W.BUBBLE]
    assert pos[1, 3] == f32(2.0) - f32(DT) and pos[0, 3] == pos[2, 3] == f32(2.0)


def test_the_seeds_are_not_the_flow_prologues():
    cells = np.arange(0, 1 << 20, 997, dtype=np.uint64)
    for step in (0, 1, 4096, 0xFFFFFFFF):
        ww = W.seeds(step, cells)
        assert np.all((ww & np.uint64(0x80000000)) != 0)  # a flow seed's low half is a cell index below 2^31
    # and the draws differ from the prologue's for the same (step, cell)
    a = Xoshiro(W.seeds(3, cells)).next_f32()
    b = Xoshiro((np.uint64(3) << np.uint64(32)) | cells).next_f32()
    assert not np.array_equal(a, b)


def test_emission_is_capped_per_cell_and_appended_in_cell_order():
    m, u = grid()
    u[1][:] = f32(30.0)
    s = dict(S, wave_crest_rate=1e6, max_per_cell=3)
    lin, count, _ = W.emit_counts(u, m, DT, 1, s)
    assert count.max() == 3
    pos, vel, total = W.emit(u, m, DT, 1, s, room=10)
    assert total == int(count.sum()) and len(pos) == 10
    cells = ((pos[:, 2].astype(int) * m.shape[1] + pos[:, 1].astype(int)) * m.shape[2] + pos[:, 0].astype(int))
    assert np.all(np.diff(cells) >= 0)
    assert np.all((pos[:, 3] >= f32(S["lifetime_lo"])) & (pos[:, 3] < f32(S["lifetime_hi"])))


# ---- the scene key ----
WW_KEY = {"max_num_particles": 5000, "trapped_air_rate": 100.0, "wave_crest_rate": 50.0, "trapped_air_range": [5.0, 20.0],
          "wave_crest_range": [6.0, 18.0], "energy_range": [0.04, 4.0], "lifetime": [1.0, 3.0], "buoyancy": 2.0, "drag": 0.5,
          "spray_below": 6, "bubble_from": 20, "max_per_cell": 4}


def scene_with(tmp_path, key):
    with open(scene_path("dam_small")) as f:
        scene = json.load(f)
    scene["fluid"]["whitewater"] = key
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(scene))
    return str(path), scene["fluid"]["grid_to_world_scale"]


def test_the_scene_key_is_converted_to_grid_units(tmp_path):
    path, scale = scene_with(tmp_path, WW_KEY)
    w = F.scene_whitewater(path)
    s2 = f32(scale) * f32(scale)
    assert w["energy_range"] == (float(f32(0.04) / s2), float(f32(4.0) / s2))
    assert w["trapped_air_range"] == (5.0, 20.0) and w["wave_crest_range"] == (6.0, 18.0)
    assert (w["max_num_particles"], w["lifetime_lo"], w["lifetime_hi"], w["max_per_cell"]) == (5000, 1.0, 3.0, 4)
    assert F.scene_whitewater(scene_path("dam_small")) is None
    assert F.scene_whitewater(scene_path("dam_whitewater_small"))["max_num_particles"] > 0


@pytest.mark.parametrize("change", [{"drag": 1.5}, {"energy_range": [4.0, 0.04]}, {"trapped_air_rate": -1.0}, {"bubble_from": 28},
                                    {"spray_below": 21}, {"lifetime": [2.0]}, {"max_num_particles": -1}, {"max_per_cell": 17},
                                    {"max_num_particles": (1 << 26) + 1}, {"trapped_air_range": "x"}, None])
def test_malformed_scene_keys_are_refused(tmp_path, change):
    key = dict(WW_KEY, **change) if change else {k: v for k, v in WW_KEY.items() if k != "drag"}
    path, _ = scene_with(tmp_path, key)
    with pytest.raises(F.BlubError) as e:
        F.scene_whitewater(path)
    assert e.value.code == BLUB_ERR_PARSE


# ---- section 22 of the state file ----
def ww_payload(count=2, capacity=100, settings=None, counters=(5, 3, 0)):
    s = dict(S, max_num_particles=capacity) if settings is None else settings
    head = bytes(F.Whitewater.from_dict(s)) + struct.pack("<3QI", *counters, count)
    rng = np.random.default_rng(count)
    parts = np.zeros((count, 8), dtype=f32)
    parts[:, :3] = rng.uniform(2, 10, (count, 3))
    parts[:, 3] = 1.0
    return head + parts.tobytes()


@pytest.mark.parametrize("base", list(BASES))
def test_version_1024_files_are_accepted_exactly_when_they_append_section_22_to_an_allowed_layout(tmp_path, bases, base):  # noqa: F811
    nb, tagged, _ = BASES[base]
    path = str(tmp_path / "state.blub")
    n = 0
    for extra in SUBSETS:
        # the layout without section 22 must follow the rule at its own version; from version 4 on section 14 is 1056 bytes long
        own = max([1] + [2, 8, 16][:max(0, nb - 13)] + [{17: 32, 18: 64, 19: 128, 20: 256, 21: 512}[i] for i in extra])
        own = 4 if own == 2 and tagged else own
        ok = (nb < 14 or tagged) and accepted(own, nb, tagged, extra)
        data = relabel(bases[base], 1024, nb + len(extra) + 1) + b"".join(section(i, PAYLOADS[i]) for i in extra) + section(22, ww_payload())
        rc, msg = info_rc(path, data)
        assert (rc == 0) == ok, (extra, msg)
        n += ok
        # without section 22 no version-1024 file is accepted
        rc, _ = info_rc(path, relabel(bases[base], 1024, nb + len(extra)) + b"".join(section(i, PAYLOADS[i]) for i in extra))
        assert rc == BLUB_ERR_PARSE
    assert n > 0 or (nb >= 14 and not tagged)  # a 992-byte section 14 belongs to version 2 only
    assert ACCEPTED[1024] == 0


@pytest.mark.parametrize("case", ["out of order", "repeated", "truncated", "overlong", "count above capacity", "length disagrees",
                                  "capacity 0", "bad setting", "at version 512"])
def test_malformed_section_22_is_refused(tmp_path, bases, case):  # noqa: F811
    base = bases["13"]
    version, secs = 1024, [section(22, ww_payload())]
    if case == "out of order":
        secs = [section(22, ww_payload()), section(21, PAYLOADS[21])]
    elif case == "repeated":
        secs = [section(22, ww_payload()), section(22, ww_payload())]
    elif case == "truncated":
        secs = [section(22, ww_payload())[:-10]]
    elif case == "overlong":
        secs = [section(22, ww_payload() + bytes(32))]
    elif case == "count above capacity":
        secs = [section(22, ww_payload(count=3, capacity=2))]
    elif case == "length disagrees":
        p = bytearray(ww_payload(count=2))
        p[88:92] = struct.pack("<I", 3)
        secs = [section(22, bytes(p))]
    elif case == "capacity 0":
        secs = [section(22, ww_payload(count=0, capacity=0))]
    elif case == "bad setting":
        secs = [section(22, ww_payload(settings=dict(S, max_num_particles=100, drag=2.0)))]
    elif case == "at version 512":
        version = 512
    rc, msg = info_rc(str(tmp_path / "state.blub"), relabel(base, version, 13 + len(secs)) + b"".join(secs))
    assert rc == BLUB_ERR_PARSE, (case, msg)
    rc, msg = info_rc(str(tmp_path / "state.blub"), relabel(base, 1024, 14) + section(22, ww_payload()))
    assert rc == 0, msg
