"""CPU: known answers of the floating bodies (DESIGN.md §8, "Floating bodies"): the NumPy restatement (tests/body_ref.py) in free fall against
the closed form of semi-implicit Euler, the tank clamp, the quaternion normalisation, the cell rule and the composite voxel values, state files of
format version 8 written from the documented layout, and bad scene `bodies` values.  No GPU needed."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import body_ref, util
from tests.test_state_file import GRID, HEADER_BYTES, header, payloads, section, write

BLUB_ERR_PARSE = 5
DT = np.float32(1.0 / 120.0)
G = (0.0, -981.0, 0.0)


# ---- integrator -----------------------------------------------------------------------------------------------------------
def test_free_fall_follows_the_closed_form_of_semi_implicit_euler():
    """No load: v_n = v_0 + n dt g, c_n = c_0 + n dt v_0 + dt^2 g n (n + 1) / 2 (float64), to float32 rounding."""
    dims = (64, 256, 64)
    b = body_ref.body(centre=(32, 200, 32), velocity=(3, 0, -2), half_extent=(4, 4, 4))
    c0, v0 = np.array(b["centre"]), np.array(b["velocity"])
    g, dt = np.array(G), float(DT)
    for n in range(1, 61):
        b = body_ref.integrate(b, (0, 0, 0), (0, 0, 0), DT, G, dims)
        assert np.allclose(b["velocity"], v0 + n * dt * g, rtol=1e-5, atol=1e-3)
        assert np.allclose(b["centre"], c0 + n * dt * v0 + dt * dt * g * n * (n + 1) / 2, rtol=1e-5, atol=1e-3)
        assert b["rotation"] == (1.0, 0.0, 0.0, 0.0) and b["angular_velocity"] == (0.0, 0.0, 0.0)


def test_the_clamp_keeps_the_bounding_box_in_the_tank_and_zeroes_outward_velocity():
    dims = (32, 32, 32)
    b = body_ref.body(centre=(16, 5.2, 29), velocity=(1, -100, 50), half_extent=(2, 4, 2))
    b = body_ref.integrate(b, (0, 0, 0), (0, 0, 0), DT, G, dims)
    assert b["centre"][1] - 4.0 == 1.0 and b["velocity"][1] == 0.0        # floor: shifted up, downward velocity gone
    assert b["centre"][2] + 2.0 == 31.0 and b["velocity"][2] == 0.0       # +z wall
    assert b["velocity"][0] == 1.0 and b["centre"][0] == float(np.float32(16) + DT * np.float32(1))
    # at rest on the floor: gravity is added and clamped away in every step
    for _ in range(5):
        b = body_ref.integrate(b, (0, 0, 0), (0, 0, 0), DT, G, dims)
        assert b["centre"][1] == 5.0 and b["velocity"][1] == 0.0
    # a rotated box: the bounding box, not the centre, is clamped
    s = np.float32(np.sqrt(0.5))
    t = body_ref.body(centre=(16, 3, 16), rotation=(s, 0, 0, s), half_extent=(4, 1, 1))
    t = body_ref.integrate(t, (0, 0, 0), (0, 0, 0), DT, G, dims)
    e = body_ref.bounding_extents(t)
    assert np.float32(t["centre"][1]) - e[1] >= np.float32(1) - np.float32(1e-5) and e[1] > 3.9


def test_quaternion_normalisation_and_a_spin_keep_unit_norm():
    q = body_ref.normalised((1.0005, 0.0, 0.0, 0.0))
    assert q == (1.0, 0.0, 0.0, 0.0)
    b = body_ref.body(centre=(16, 16, 16), angular_velocity=(0.0, 3.0, 1.0), half_extent=(3, 2, 1))
    for _ in range(300):
        b = body_ref.integrate(b, (0, 0, 0), (0, 0, 0), DT, (0, 0, 0), (32, 32, 32))
        assert abs(np.linalg.norm(np.float64(b["rotation"])) - 1.0) < 1e-6
    # torque-free: the angular velocity does not change (no gyroscopic term)
    assert b["angular_velocity"] == (0.0, 3.0, 1.0)


def test_a_torque_turns_the_body_about_the_world_axis():
    b = body_ref.body(centre=(16, 16, 16), half_extent=(2, 2, 2), relative_density=1.0)
    m, inertia = body_ref.mass_and_inertia(b)
    assert m == 64.0 and inertia[0] == np.float32(64.0 * 8 / 3)
    b = body_ref.integrate(b, (0, 0, 0), (0, 0, 100 << 8), DT, (0, 0, 0), (32, 32, 32))
    assert b["angular_velocity"][2] == float(DT * (np.float32(100) / inertia[2])) and b["angular_velocity"][:2] == (0.0, 0.0)


# ---- cell rule and composite volume -----------------------------------------------------------------------------------------
def test_cell_rule_and_composite_values():
    dims = (16, 16, 16)
    box = body_ref.body(centre=(8, 8, 8), half_extent=(2, 3, 1), velocity=(1, 2, 3), angular_velocity=(0, 0, 1))
    mask, _ = body_ref.covered(dims, box)
    assert mask.sum() == 4 * 6 * 2 and mask[7:9, 5:11, 6:10].all()
    sphere = body_ref.body("sphere", 2.0, centre=(8, 8, 8))
    assert body_ref.covered(dims, sphere)[0].sum() == 32  # cell centres within 2 of (8, 8, 8): offsets (+-0.5, +-0.5, +-0.5) and +-1.5 on one axis
    vox = body_ref.composite(dims, None, [box])
    # cell (9, 8, 8): d = (1.5, 0.5, 0.5), v + w x d = (1 - 0.5, 2 + 1.5, 3)
    assert vox[8, 8, 9].tolist() == [0.5, 3.5, 3.0, 1.0] and vox[0, 0, 0].tolist() == [0.0] * 4
    # a later body wins where bodies overlap
    both = body_ref.composite(dims, None, [box, dict(sphere, velocity=(-7.0, 0.0, 0.0))])
    assert both[8, 8, 8].tolist() == [-7.0, 0.0, 0.0, 1.0]


# ---- state file version 8 ---------------------------------------------------------------------------------------------------
BODY_SLOT = struct.Struct("<i3ff3f4f3f3f")
assert BODY_SLOT.size == 72


def v8_bytes(bodies, num_bodies=None, flow=None, corrupt_crc=False, body_section_pad=b""):
    data = bytearray(header(version=8))
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", 15)  # num_sections
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    out = bytes(data)
    for sid, p in enumerate(payloads(), start=1):
        out += section(sid, p)
    fl = flow if flow is not None else bytes(1056)  # an empty flow set: counts 0, boxes 0, counters 0, tags 0
    out += section(14, fl)
    slots = b"".join(BODY_SLOT.pack(0 if b["shape"] == "box" else 1, *b["half_extent"], b["relative_density"], *b["centre"], *b["rotation"],
                                    *b["velocity"], *b["angular_velocity"]) for b in bodies)
    payload = struct.pack("<I", len(bodies) if num_bodies is None else num_bodies) + slots + bytes(72 * (16 - len(bodies))) + body_section_pad
    sec = section(15, payload)
    if corrupt_crc:
        sec = sec[:-4] + struct.pack("<I", zlib.crc32(payload) ^ 1)
    return out + sec


BODIES = [body_ref.body(centre=(16, 16, 20), half_extent=(3, 2, 4)), body_ref.body("sphere", 2.5, centre=(8, 8, 8), relative_density=2.0)]


def test_version_8_written_from_the_documented_layout_is_accepted(tmp_path):
    info = blub_b200.state_info(write(tmp_path, v8_bytes(BODIES)))
    assert info.format_version == 8 and tuple(info.grid_dimension) == GRID


@pytest.mark.parametrize("case, make, needle", [
    ("count above 16", lambda: v8_bytes(BODIES, num_bodies=17), "more than 16 bodies"),
    ("bad CRC", lambda: v8_bytes(BODIES, corrupt_crc=True), "checksum mismatch in section 15"),
    ("section 15 too long", lambda: v8_bytes(BODIES, body_section_pad=b"\0\0\0\0"), "its header describes"),
    ("bad body", lambda: v8_bytes([dict(BODIES[0], relative_density=0.0)]), "relative_density"),
    ("outside the tank", lambda: v8_bytes([dict(BODIES[0], centre=(2.0, 16.0, 16.0))]), "bounding box"),
])
def test_malformed_version_8_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    assert rc == BLUB_ERR_PARSE, case
    assert needle in L.blub_last_error().decode(), (case, L.blub_last_error().decode())


# ---- scene key --------------------------------------------------------------------------------------------------------------
def v3(x, y, z):
    return {"x": x, "y": y, "z": z}


def scene_with(tmp_path, bodies, name="s.json"):
    sc = json.load(open(util.scene_path("dam_small")))  # 32^3 cells of 0.01 m
    sc["fluid"]["bodies"] = bodies
    path = str(tmp_path / name)
    with open(path, "w") as f:
        json.dump(sc, f)
    return path


GOOD = {"shape": "box", "position": v3(0.16, 0.2, 0.16), "half_extent": v3(0.04, 0.02, 0.03), "relative_density": 0.5}


def test_scene_bodies_convert_to_grid_units(tmp_path):
    path = scene_with(tmp_path, [dict(GOOD, rotation_angles_deg=v3(0.0, 90.0, 0.0), velocity=v3(0.1, 0.0, 0.0), angular_velocity=v3(0.0, 1.0, 0.0)),
                                 {"shape": "sphere", "position": v3(0.1, 0.1, 0.1), "half_extent": 0.03, "relative_density": 2.0}])
    got = F.scene_bodies(path)
    scale = np.float32(0.01)
    assert got[0]["centre"] == tuple(float(np.float32(v) / scale) for v in (0.16, 0.2, 0.16))
    assert got[0]["half_extent"] == tuple(float(np.float32(v) / scale) for v in (0.04, 0.02, 0.03))
    assert got[0]["velocity"] == (float(np.float32(0.1) / scale), 0.0, 0.0) and got[0]["angular_velocity"] == (0.0, 1.0, 0.0)
    assert np.allclose(got[0]["rotation"], (np.sqrt(0.5), 0.0, np.sqrt(0.5), 0.0), atol=1e-6)
    assert got[1]["shape"] == "sphere" and got[1]["half_extent"][0] == float(np.float32(0.03) / scale) and got[1]["relative_density"] == 2.0
    F.scene_info(path)


@pytest.mark.parametrize("what, bodies", [
    ("not an array", {"shape": "box"}),
    ("bad shape", [dict(GOOD, shape="cone")]),
    ("missing density", [{k: v for k, v in GOOD.items() if k != "relative_density"}]),
    ("zero density", [dict(GOOD, relative_density=0.0)]),
    ("negative density", [dict(GOOD, relative_density=-1.0)]),
    ("below one cell", [dict(GOOD, half_extent=v3(0.005, 0.02, 0.02))]),
    ("out of the float range", [dict(GOOD, velocity=v3(1e39, 0.0, 0.0))]),
    ("outside the tank", [dict(GOOD, position=v3(0.02, 0.2, 0.16))]),
    ("seventeen", [GOOD] * 17),
])
def test_bad_scene_bodies_are_parse_errors(tmp_path, what, bodies):
    path = scene_with(tmp_path, bodies)
    assert F.lib().blub_scene_info(os.fsencode(path), F.SceneInfo()) == BLUB_ERR_PARSE, what
    with pytest.raises(F.BlubError):
        F.scene_bodies(path)
