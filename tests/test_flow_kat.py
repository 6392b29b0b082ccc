"""CPU: known answers of the flow prologue (sources and drains, DESIGN.md §8) on the NumPy restatement the GPU tests compare against, the
scene keys as blub_scene_info parses them, and the version-2 state file as blub_state_info reads it.  No GPU needed."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import flow_ref, test_state_file as SF, util

DIMS = (16, 16, 16)
BLUB_ERR_PARSE = 5


def _cell_particles(cells_and_counts, rng):
    """Particles at random points of the given cells, cells in the given order: [((x, y, z), count)]."""
    pos = []
    for (x, y, z), k in cells_and_counts:
        for _ in range(k):
            pos.append([x + rng.uniform(0.05, 0.95), y + rng.uniform(0.05, 0.95), z + rng.uniform(0.05, 0.95), 0.0])
    return np.asarray(pos, dtype=np.float32).reshape(-1, 4)


def _rows(n, rng):
    return [rng.standard_normal((n, 4)).astype(np.float32) for _ in range(3)]


def test_drain_removes_exactly_the_particles_in_the_box_and_keeps_the_order():
    rng = np.random.default_rng(1)
    pos = rng.uniform(1.0, 15.0, (500, 4)).astype(np.float32)
    rows = _rows(500, rng)
    flow = flow_ref.make_flow(DIMS, drains=[((3, 3, 3), (8, 6, 9))])
    out, out_rows, (emitted, drained, refused) = flow_ref.prologue(pos, rows, 0, DIMS, 1000, flow)
    inside = (pos[:, 0] >= 3) & (pos[:, 0] < 8) & (pos[:, 1] >= 3) & (pos[:, 1] < 6) & (pos[:, 2] >= 3) & (pos[:, 2] < 9)
    assert drained == int(inside.sum()) > 0 and emitted == refused == 0
    np.testing.assert_array_equal(out, pos[~inside])  # survivors in their order
    for a in range(3):
        np.testing.assert_array_equal(out_rows[a], rows[a][~inside])


def test_source_fills_an_empty_box_with_8_particles_per_cell_in_their_octants():
    flow = flow_ref.make_flow(DIMS, sources=[((4, 5, 6), (6, 7, 8), (1.0, -2.0, 3.0))])
    pos, rows, (emitted, drained, refused) = flow_ref.prologue(np.zeros((0, 4), np.float32), _rows(0, np.random.default_rng(0)), 5, DIMS, 1000, flow)
    assert (emitted, drained, refused) == (2 * 2 * 2 * 8, 0, 0)
    order = [(x, y, z) for z in (6, 7) for y in (5, 6) for x in (4, 5)]  # cell x fastest, then the 8 slots
    for j, cell in enumerate(order):
        for slot in range(8):
            p = pos[8 * j + slot, :3]
            strat = np.array([slot % 2, slot // 2 % 2, slot // 4 % 2])
            lo = np.array(cell) + 0.5 * strat
            assert np.all(p >= lo) and np.all(p < lo + 0.5), (cell, slot, p)
    for a, v in enumerate((1.0, -2.0, 3.0)):
        np.testing.assert_array_equal(rows[a], np.tile(np.float32([0, 0, 0, v]), (64, 1)))


def test_emission_jitter_is_a_function_of_step_cell_and_slot():
    flow = flow_ref.make_flow(DIMS, sources=[((4, 4, 4), (5, 5, 5), (0, 0, 0))])
    empty = np.zeros((0, 4), np.float32)
    rows0 = _rows(0, np.random.default_rng(0))
    a, _, _ = flow_ref.prologue(empty, rows0, 7, DIMS, 100, flow)
    b, _, _ = flow_ref.prologue(empty, rows0, 7, DIMS, 100, flow)
    c, _, _ = flow_ref.prologue(empty, rows0, 8, DIMS, 100, flow)
    np.testing.assert_array_equal(a, b)
    assert not np.array_equal(a, c)
    # the same draws as add_cube's generator: seed step << 32 | cell, 8 slots x 3 floats in slot order
    rng = flow_ref.Xoshiro(np.array([(7 << 32) | ((4 * 16 + 4) * 16 + 4)], dtype=np.uint64))
    r = np.array([[rng.next_f32()[0] for _ in range(3)] for _ in range(8)], dtype=np.float32)
    strat = np.array([[s % 2, s // 2 % 2, s // 4 % 2] for s in range(8)], dtype=np.float32)
    np.testing.assert_array_equal(a[:, :3], np.float32(4) + (strat * np.float32(0.5) + r * np.float32(0.5)))


def test_top_up_fills_cells_below_4_to_8_and_leaves_the_rest():
    rng = np.random.default_rng(2)
    flow = flow_ref.make_flow(DIMS, sources=[((4, 4, 4), (6, 5, 5), (0, 5, 0))])
    pos = _cell_particles([((4, 4, 4), 3), ((5, 4, 4), 4)], rng)
    rows = _rows(len(pos), rng)
    out, out_rows, (emitted, drained, refused) = flow_ref.prologue(pos, rows, 1, DIMS, 100, flow)
    assert (emitted, drained, refused) == (5, 0, 0)
    np.testing.assert_array_equal(out[:7], pos)
    c = flow_ref.cells_of(out[7:], DIMS)
    assert np.all(c[0] == 4) and np.all(c[1] == 4) and np.all(c[2] == 4)
    for slot, p in zip(range(3, 8), out[7:, :3]):  # slots count..7
        lo = np.array([4, 4, 4]) + 0.5 * np.array([slot % 2, slot // 2 % 2, slot // 4 % 2])
        assert np.all(p >= lo) and np.all(p < lo + 0.5)
    for a in range(3):  # every particle in a source cell, old and new, leaves with the nozzle velocity
        np.testing.assert_array_equal(out_rows[a], np.tile(np.float32([0, 0, 0, 5.0 if a == 1 else 0.0]), (12, 1)))


def test_capacity_truncates_in_emission_order_and_counts_the_refused():
    flow = flow_ref.make_flow(DIMS, sources=[((2, 2, 2), (4, 3, 3), (0, 0, 0)), ((8, 8, 8), (9, 9, 9), (0, 0, 0))])
    rng = np.random.default_rng(3)
    pos = rng.uniform(10.0, 14.0, (10, 4)).astype(np.float32)
    full, _, _ = flow_ref.prologue(pos, _rows(10, rng), 3, DIMS, 1000, flow)
    out, _, (emitted, drained, refused) = flow_ref.prologue(pos, _rows(10, rng), 3, DIMS, 10 + 13, flow)
    assert (emitted, drained, refused) == (13, 0, 24 - 13)
    np.testing.assert_array_equal(out, full[:23])  # source 0 cell (2,2,2), then (3,2,2) up to slot 4; source 1 refused


def test_solid_and_border_cells_do_not_emit():
    solid = np.zeros(DIMS[::-1], dtype=bool)
    solid[5, 5, 5] = True  # (z, y, x)
    flow = flow_ref.make_flow(DIMS, sources=[((4, 5, 5), (7, 6, 6), (0, 0, 0))])
    out, _, (emitted, _, _) = flow_ref.prologue(np.zeros((0, 4), np.float32), _rows(0, np.random.default_rng(0)), 0, DIMS, 100, flow, solid)
    assert emitted == 16
    assert set(flow_ref.cells_of(out, DIMS)[0].tolist()) == {4, 6}
    # a box reaching the far wall is clamped to dim - 1 (exclusive): the border cells never emit
    flow = flow_ref.make_flow(DIMS, sources=[((14, 14, 14), (40, 40, 40), (0, 0, 0))])
    assert flow["sources"][0][:2] == ((14, 14, 14), (15, 15, 15))


# ---- scene keys -------------------------------------------------------------------------------------------------------
def test_scene_info_accepts_the_tap_scene():
    info = blub_b200.scene_info(util.scene_path("tap_small"))
    assert tuple(info.grid_dimension) == (32, 32, 32) and info.num_fluid_cubes == 1


@pytest.mark.parametrize("key,value", [
    ("sources", {"min": {"x": 0.1, "y": 0.1, "z": 0.1}, "max": {"x": 0.2, "y": 0.2, "z": 0.2}}),  # no velocity
    ("sources", [{"min": {"x": 0.1, "y": 0.1, "z": 0.1}, "max": {"x": 0.2, "y": 0.2, "z": 0.2}}]),
    ("sources", [{"min": {"x": 0.1, "y": 0.1}, "max": {"x": 0.2, "y": 0.2, "z": 0.2}, "velocity": {"x": 0, "y": 0, "z": 0}}]),
    ("drains", [{"min": {"x": 0.1, "y": 0.1, "z": 0.1}, "max": {"x": "a", "y": 0.2, "z": 0.2}}]),
    ("drains", 3),
])
def test_malformed_flow_keys_are_parse_errors(tmp_path, key, value):
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"][key] = value
    path = tmp_path / "bad.json"
    path.write_text(json.dumps(sc))
    out = F.SceneInfo()
    assert F.lib().blub_scene_info(os.fsencode(str(path)), out) == BLUB_ERR_PARSE


# ---- state file, format version 2 -------------------------------------------------------------------------------------
def flow_payload(num_sources=1, num_drains=1, counters=(1000, 24, 0)):
    src = np.zeros((16, 6), np.int32)
    vel = np.zeros((16, 3), np.float32)
    drn = np.zeros((16, 6), np.int32)
    src[:num_sources] = [4, 20, 4, 8, 24, 8]
    vel[:num_sources] = [0.0, -100.0, 0.0]
    drn[:num_drains] = [1, 1, 1, 5, 3, 5]
    return struct.pack("<2I", num_sources, num_drains) + src.tobytes() + vel.tobytes() + drn.tobytes() + struct.pack("<3Q", *counters)


def state_v2(payload14=None):
    h = bytearray(SF.header(version=2))
    struct.pack_into("<I", h, SF.HEADER_BYTES - 8, 14)  # num_sections
    struct.pack_into("<I", h, SF.HEADER_BYTES - 4, zlib.crc32(bytes(h[:SF.HEADER_BYTES - 4])))
    out = bytes(h)
    for sid, p in enumerate(SF.payloads(), start=1):
        out += SF.section(sid, p)
    return out + SF.section(14, flow_payload() if payload14 is None else payload14)


def test_an_unsupported_format_version_is_a_parse_error(tmp_path):
    rc, msg, _ = SF.info_rc(SF.write(tmp_path, SF.header(version=3) + state_v2()[SF.HEADER_BYTES:]))
    assert rc == BLUB_ERR_PARSE and "version 3 is not supported" in msg, msg


def test_a_version_2_file_from_the_documented_layout_is_accepted(tmp_path):
    data = state_v2()
    assert len(flow_payload()) == 992
    info = blub_b200.state_info(SF.write(tmp_path, data))
    assert (info.num_particles, info.format_version) == (SF.NUM_PARTICLES, 2)


@pytest.mark.parametrize("case,make,needle", [
    ("corrupted section 14", lambda: state_v2()[:-8] + bytes([state_v2()[-8] ^ 1]) + state_v2()[-7:], "checksum"),
    ("overlapping source and drain", lambda: state_v2(flow_payload().replace(struct.pack("<6i", 4, 20, 4, 8, 24, 8), struct.pack("<6i", 2, 2, 2, 8, 24, 8))),
     "overlaps"),
    ("corner outside the grid", lambda: state_v2(flow_payload().replace(struct.pack("<6i", 1, 1, 1, 5, 3, 5), struct.pack("<6i", 0, 1, 1, 5, 3, 5))),
     "outside"),
    ("section 14 missing", lambda: state_v2()[:-(16 + 992 + 4)], "bytes"),
])
def test_malformed_version_2_files_are_parse_errors(tmp_path, case, make, needle):
    rc, msg, _ = SF.info_rc(SF.write(tmp_path, make()))
    assert rc == BLUB_ERR_PARSE and needle in msg, (case, rc, msg)
