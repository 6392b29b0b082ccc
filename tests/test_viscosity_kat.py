"""CPU: known answers of the viscosity rule (DESIGN.md §8 "Viscous liquids") through its float64 restatement tests/visc_ref.py, the version-32
state file as the host-only reader sees it, and the scene key.  No GPU needed."""
import json
import os
import struct
import zlib

import numpy as np
import pytest
import scipy.sparse.linalg as spl

import blub_b200
from blub_b200 import fluid as F
from tests import util, visc_ref as V
from tests.test_bodies_kat import BODIES, v8_bytes
from tests.test_mesh_bodies_kat import v16_bytes
from tests.test_state_file import HEADER_BYTES, section, state_bytes, write

BLUB_ERR_PARSE = 5


def salt_and_pepper(shape=(12, 10, 14), seed=3):
    """Every marker value next to every other one, inside SOLID border cells; about a third FLUID."""
    rng = np.random.default_rng(seed)
    m = rng.integers(-1, 2, shape).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def random_vox(shape, seed=5):
    rng = np.random.default_rng(seed)
    vox = rng.uniform(-2, 2, shape + (4,))
    vox[..., 3] = 1.0
    return vox


@pytest.mark.parametrize("k", [0.05, 1.0, 20.0])
def test_matrix_is_symmetric_with_dirichlet_row_sums_and_eigenvalues_of_at_least_one(k):
    m = salt_and_pepper()
    classes = set()
    for c in range(3):
        s = V.System(m, c, k, np.zeros(m.shape), 0.0, random_vox(m.shape))
        assert s.n > 100
        assert abs(s.A - s.A.T).max() == 0.0
        assert np.allclose(np.asarray(s.A.sum(axis=1)).ravel(), 1.0 + k * s.num_dirichlet, rtol=1e-13)
        assert spl.eigsh(s.A, k=1, which="SA", return_eigenvectors=False)[0] >= 1.0 - 1e-9
        for (coupled, dirichlet, _) in V.neighbours(m, c):
            classes |= {(bool(a), bool(b)) for a, b in zip(coupled[s.live], dirichlet[s.live])}
    assert classes == {(True, False), (False, True), (False, False)}  # every neighbour class occurs


def test_sine_products_are_eigenvectors_of_the_all_fluid_box():
    N, k = 12, 0.7
    m = np.zeros((N, N, N), dtype=np.int8)
    m[1:-1, 1:-1, 1:-1] = V.FLUID
    for c in range(3):
        s = V.System(m, c, k, np.zeros(m.shape), 0.0)
        # live rows per axis: along the component's own axis the faces between cells 1 .. N - 2 (N - 3 of them), across it the cells 1 .. N - 2
        rows = [N - 3 if d == c else N - 2 for d in range(3)]
        assert s.n == rows[0] * rows[1] * rows[2]
        modes = (2, 1, 3)
        lam = [2.0 - 2.0 * np.cos(np.pi * modes[d] / (rows[d] + 1)) for d in range(3)]
        z, y, x = np.meshgrid(*[np.arange(N)] * 3, indexing="ij")
        vec = np.ones(m.shape)
        for d, coord in enumerate((x, y, z)):
            vec *= np.sin(np.pi * modes[d] * coord / (rows[d] + 1))  # the first live row sits at coordinate 1
        u_star = np.where(s.live, vec, 0.0)
        s = V.System(m, c, k, u_star, 0.0)
        x_direct = s.solve()
        assert np.allclose(x_direct, u_star[s.live] / (1.0 + k * sum(lam)), rtol=1e-12, atol=1e-14)


def test_a_shell_moving_with_the_liquid_is_a_fixed_point():
    N, vel = 12, (0.75, -1.5, 2.25)
    m = np.zeros((N, N, N), dtype=np.int8)
    m[3:9, 3:9, 3:9] = V.FLUID  # the block's shell: SOLID cells that all carry the velocity
    vox = np.zeros(m.shape + (4,))
    vox[...] = (*vel, 1.0)
    for c in range(3):
        s = V.System(m, c, 5.0, np.full(m.shape, vel[c]), 0.0, vox)
        assert s.num_dirichlet.max() >= 2
        assert np.abs(s.residual(np.full(m.shape, vel[c]))).max() < 1e-12
        assert np.allclose(s.solve(), vel[c], rtol=1e-12)


def test_free_surface_faces_contribute_nothing():
    N, k = 12, 2.0
    def layer(above):
        m = np.zeros((N, N, N), dtype=np.int8)
        m[1:-1, 1:5, 1:-1] = V.FLUID  # [z, y, x]: a layer of four cells on the floor
        m[1:-1, 5:-1, 1:-1] = above
        return m
    air = layer(V.AIR)
    s = V.System(air, 0, k, np.zeros(air.shape), 0.0)
    top = s.index[5, 4, 5]  # an x face of the top fluid row, away from the walls
    assert s.A[top, top] == 1.0 + 5 * k and s.A[top].nnz == 6 and s.num_dirichlet[top] == 0
    assert s.index[5, 5, 5] == -1  # the face above lies between two AIR cells: not an unknown
    # the vertical faces between the top fluid row and the air are live and see only the face below
    t = V.System(air, 1, k, np.zeros(air.shape), 0.0)
    up = t.index[5, 4, 5]
    assert up >= 0 and t.A[up, up] == 1.0 + 5 * k and t.index[5, 5, 5] == -1
    assert np.allclose(np.asarray(s.A.sum(axis=1)).ravel(), 1.0 + k * s.num_dirichlet)


def test_rest_gives_zero_and_gravity_is_added_back():
    m = salt_and_pepper()
    gdt = -0.08175
    s = V.System(m, 1, 3.0, np.full(m.shape, gdt), gdt)
    assert np.abs(s.b).max() == 0.0 and np.abs(s.solve()).max() == 0.0
    rng = np.random.default_rng(1)
    u_star = rng.standard_normal(m.shape)
    s, s0 = V.System(m, 1, 3.0, u_star + gdt, gdt), V.System(m, 1, 3.0, u_star, 0.0)
    assert np.allclose(s.solve(), s0.solve(), rtol=1e-12, atol=1e-14)
    result = np.zeros(m.shape)
    result[s.live] = s.solve() + gdt
    assert np.abs(s.residual(result)).max() < 1e-12


# ---- state file version 32 --------------------------------------------------------------------------------------------------
def viscosity_payload(nu=0.5, tolerance=1e-4, max_it=200, reserved=0):
    return struct.pack("<ffiI", nu, tolerance, max_it, reserved)


def promote(base, num_sections, payload=None, version=32, tail=b"", corrupt_crc=False):
    """A file of an older version with its header rewritten to `version` and `num_sections`, and section 17 behind it."""
    data = bytearray(base)
    data[8:12] = struct.pack("<I", version)
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", num_sections)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    payload = viscosity_payload() if payload is None else payload
    sec = section(17, payload)
    if corrupt_crc:
        sec = sec[:-4] + struct.pack("<I", zlib.crc32(payload) ^ 1)
    return bytes(data) + sec + tail


BASES = {
    "13 sections": (lambda: state_bytes(), 14),
    "flow section": (lambda: state_bytes() + section(14, bytes(1056)), 15),  # 1056 bytes, here an empty set as version 8 allows
    "bodies": (lambda: v8_bytes(BODIES), 16),
    "mesh body": (lambda: v16_bytes(), 17),
}


@pytest.mark.parametrize("base", sorted(BASES))
def test_version_32_written_from_the_documented_layout_is_accepted(tmp_path, base):
    make, ns = BASES[base]
    info = F.state_info(write(tmp_path, promote(make(), ns)))
    assert info.format_version == 32


@pytest.mark.parametrize("case, make, needle", [
    ("viscosity 0", lambda: promote(state_bytes(), 14, viscosity_payload(nu=0.0)), "above 0"),
    ("viscosity NaN", lambda: promote(state_bytes(), 14, viscosity_payload(nu=float("nan"))), "kinematic_viscosity"),
    ("viscosity negative", lambda: promote(v8_bytes(BODIES), 16, viscosity_payload(nu=-1.0)), "kinematic_viscosity"),
    ("tolerance 0", lambda: promote(state_bytes(), 14, viscosity_payload(tolerance=0.0)), "error_tolerance"),
    ("cap 0", lambda: promote(state_bytes(), 14, viscosity_payload(max_it=0)), "max_num_iterations"),
    ("reserved", lambda: promote(state_bytes(), 14, viscosity_payload(reserved=1)), "reserved"),
    ("section 17 too long", lambda: promote(state_bytes(), 14, viscosity_payload() + bytes(4)), "its header describes"),
    ("section 17 too short", lambda: promote(state_bytes(), 14, viscosity_payload()[:12]), "its header describes"),
    ("num_sections names another layout", lambda: promote(state_bytes(), 15), "its header describes"),
    ("num_sections names no layout", lambda: promote(state_bytes(), 13), "14 to 17"),
    ("trailing bytes", lambda: promote(state_bytes(), 14, tail=bytes(4)), "its header describes"),
    ("trailing bytes behind a mesh body", lambda: promote(v16_bytes(), 17, tail=bytes(4)), "section"),
    ("bad CRC", lambda: promote(state_bytes(), 14, corrupt_crc=True), "checksum mismatch in section 17"),
    ("flow section at its version-2 length", lambda: promote(state_bytes() + section(14, bytes(992)), 15), "its header describes"),
] + [(f"version {v}", (lambda v=v: promote(state_bytes(), 14, version=v)), "version") for v in list(range(17, 32)) + [33]])
def test_malformed_version_32_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    assert rc == BLUB_ERR_PARSE, (case, rc)
    assert needle in L.blub_last_error().decode(), (case, L.blub_last_error().decode())


# ---- scene key --------------------------------------------------------------------------------------------------------------
def scene_with(tmp_path, value, scale=0.02):
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"]["grid_to_world_scale"] = scale
    if value is not None:
        sc["fluid"]["viscosity"] = value
    p = tmp_path / "viscous.json"
    p.write_text(json.dumps(sc))
    return str(p)


def test_scene_viscosity_is_converted_to_cells():
    assert F.scene_viscosity(util.scene_path("dam_small")) == 0.0
    path = util.scene_path("dam_viscous")
    sc = json.load(open(path))
    scale = np.float32(sc["fluid"]["grid_to_world_scale"])
    assert F.scene_viscosity(path) == float(np.float32(sc["fluid"]["viscosity"]) / (scale * scale)) > 0.0


def test_scene_viscosity_by_scale(tmp_path):
    assert F.scene_viscosity(scene_with(tmp_path, 1e-3, 0.02)) == float(np.float32(1e-3) / (np.float32(0.02) * np.float32(0.02)))
    assert F.scene_viscosity(scene_with(tmp_path, None)) == 0.0
    assert blub_b200.scene_info(scene_with(tmp_path, 0)).max_num_particles > 0


@pytest.mark.parametrize("value", [-1e-3, "thick", [1.0], {"x": 1}, 1e39, True, None])
def test_scene_viscosity_refuses_bad_values(tmp_path, value):
    sc = json.load(open(util.scene_path("dam_small")))
    sc["fluid"]["viscosity"] = value
    p = tmp_path / "bad.json"
    p.write_text(json.dumps(sc))
    L = F.lib()
    assert L.blub_scene_info(os.fsencode(str(p)), F.SceneInfo()) == BLUB_ERR_PARSE
    assert L.blub_scene_viscosity(os.fsencode(str(p)), F.C.c_float()) == BLUB_ERR_PARSE
