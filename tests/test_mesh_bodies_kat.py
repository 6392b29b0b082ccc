"""CPU: triangle-mesh bodies (DESIGN.md §8, "Mesh bodies") against the library's host entry points and tests/mesh_body_ref.py: mass
properties against closed forms and a NumPy float64 restatement, the principal frame's rules, the refusals, the crossing-parity cell rule
against a float64 winding-number inside test, its tie rule, and the asymmetric tank clamp."""
import numpy as np
import pytest

from blub_b200 import fluid as F
from tests import body_ref, mesh_body_ref as M

f32 = np.float32
TILT = (float(f32(np.cos(0.3))), float(f32(np.sin(0.3) * 0.6)), 0.0, float(f32(np.sin(0.3) * 0.8)))
TILT2 = tuple(float(f32(v)) for v in np.array([0.8, -0.2, 0.5, 0.25]) / np.linalg.norm([0.8, -0.2, 0.5, 0.25]))


def assert_frame(p):
    R = M.quat_to_matrix(p["principal_rotation"])
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and abs(np.linalg.det(R) - 1) < 1e-12
    return R


# ---- mass properties ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inward", [False, True])
def test_box_mesh_closed_form(inward):
    v, t = M.box_mesh((0, 0, 0), (4, 6, 8))
    if inward:
        t = t[:, ::-1].copy()
    p = F.mesh_body_properties(v, t, 0.5)
    a, b, c = 2.0, 3.0, 4.0
    V = a * b * c
    assert p["volume"] == pytest.approx(V, rel=1e-14)
    assert np.allclose(p["centroid"], (2, 3, 4), atol=1e-13)
    assert np.allclose(p["principal_moments"], [V * (b * b + c * c) / 12, V * (a * a + c * c) / 12, V * (a * a + b * b) / 12], rtol=1e-13)
    assert p["principal_rotation"] == (1.0, 0.0, 0.0, 0.0)
    assert p["bounds_lo"] == (-1.0, -1.5, -2.0) and p["bounds_hi"] == (1.0, 1.5, 2.0)
    assert p["mass"] == f32(V) and p["moments"] == tuple(float(f32(x)) for x in p["principal_moments"])


def test_tetrahedron_closed_form():
    v = np.array([[0, 0, 0], [3, 0, 0], [0, 3, 0], [0, 0, 3]], dtype=np.float32)
    t = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], dtype=np.uint32)
    p = F.mesh_body_properties(v, t, 1.0)
    assert p["volume"] == pytest.approx(4.5, rel=1e-14)
    assert np.allclose(p["centroid"], (0.75, 0.75, 0.75), atol=1e-14)
    # the corner tetrahedron of side a: about its centroid, the moments are 3 a^5 / 200 ... in closed form through the covariance
    a = 3.0
    C = a ** 5 / 120 * (np.ones((3, 3)) + np.eye(3)) - 4.5 * np.outer([0.75] * 3, [0.75] * 3)
    I = np.trace(C) * np.eye(3) - C
    assert np.allclose(p["inertia"], I, rtol=1e-12)
    assert np.allclose(sorted(p["principal_moments"]), np.linalg.eigvalsh(I), rtol=1e-12)
    assert_frame(p)


def test_l_block_closed_form_and_restatement():
    v, t = M.l_block()
    p = F.mesh_body_properties(v, t, 2.0)
    # five unit cubes scaled by 2: V = 40, centroid (model units) = mean of the cube centres
    centres = np.array([(0.5, 0.5, 0.5), (1.5, 0.5, 0.5), (2.5, 0.5, 0.5), (0.5, 1.5, 0.5), (0.5, 2.5, 0.5)])
    assert p["volume"] == pytest.approx(40.0, rel=1e-13)
    assert np.allclose(p["centroid"], centres.mean(0), atol=1e-13)
    # inertia about the centre of mass: each cube (side 2, mass 8) about its own centre plus the parallel axis term
    com = 2 * centres.mean(0)
    I = np.zeros((3, 3))
    for c in 2 * centres:
        r = c - com
        I += 8 * (2 * 4 / 12) * np.eye(3) + 8 * (r @ r * np.eye(3) - np.outer(r, r))
    assert np.allclose(p["inertia"], I, rtol=1e-12)
    assert abs(p["inertia"][0, 1]) > 1.0  # non-diagonal
    V, c, Iref = M.mass_properties(v, t, 2.0)
    assert np.allclose(p["inertia"], Iref, rtol=1e-12) and np.allclose(p["centroid"], c, atol=1e-13)
    R = assert_frame(p)
    assert np.allclose(R.T @ p["inertia"] @ R, np.diag(p["principal_moments"]), atol=1e-9)
    assert list(p["principal_moments"]) == sorted(p["principal_moments"])  # ascending
    for j in range(3 - 1):  # the largest component of the first two axes is positive
        assert R[np.argmax(abs(R[:, j])), j] > 0
    q = F.mesh_body_properties(v, t[:, ::-1].copy(), 2.0)
    assert np.allclose(q["inertia"], p["inertia"], rtol=1e-13) and np.allclose(q["principal_rotation"], p["principal_rotation"], atol=1e-12)


@pytest.mark.parametrize("mesh", ["icosphere", "torus"])
def test_symmetric_meshes_keep_the_model_frame(mesh):
    v, t = M.icosphere(3, 1.0) if mesh == "icosphere" else M.torus(2.0, 0.7, 32, 16)
    p = F.mesh_body_properties(v, t, 6.0)
    assert p["principal_rotation"] == (1.0, 0.0, 0.0, 0.0)
    V, c, I = M.mass_properties(v, t, 6.0)
    assert p["volume"] == pytest.approx(V, rel=1e-12) and np.allclose(p["inertia"], I, rtol=1e-10, atol=1e-9 * np.trace(I))


# ---- refusals ------------------------------------------------------------------------------------------------------------------
def test_refusals():
    v, t = M.icosphere(1, 1.0)
    F.mesh_body_properties(v, t, 4.0)
    flipped = np.concatenate([t[:1, ::-1], t[1:]])
    thin_v, thin_t = M.box_mesh((0, 0, 0), (10, 10, 0.5))
    flat_v = v.copy()
    flat_v[:, 2] = 0
    bad = [(v, t[1:], 4.0, "open"), (v, flipped, 4.0, "flipped"), (v, t, 0.0, "scale 0"), (v, t, -1.0, "negative"), (v, t, float("nan"), "nan"),
           (v, t, float("inf"), "inf"), (thin_v, thin_t, 1.0, "thin"), (flat_v, t, 4.0, "zero volume"), (v, t[:0], 4.0, "empty"),
           (v, np.array([[0, 0, 1]]), 4.0, "repeated vertex"), (v, np.array([[0, 1, 500]]), 4.0, "index out of range")]
    for pos, tri, scale, why in bad:
        with pytest.raises(F.BlubError):
            F.mesh_body_properties(pos, tri, scale)
            pytest.fail(why)


def test_vertex_limit():
    """More than 2^18 vertices: a closed voxel-union mesh is cheap to make that large (a 1 x 1 x k column has 4k + 4 vertices)."""
    k = (262144 // 4) + 1
    x = np.arange(k + 1, dtype=np.float32)
    # a long square tube along x, closed by two end caps: 4 (k + 1) vertices
    ring = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], dtype=np.float32)
    v = np.concatenate([np.stack([np.full(4, xi), ring[:, 0], ring[:, 1]], -1) for xi in x])
    tris = []
    for i in range(k):
        for j in range(4):
            a, b, c, d = 4 * i + j, 4 * i + (j + 1) % 4, 4 * (i + 1) + (j + 1) % 4, 4 * (i + 1) + j
            tris += [(a, b, c), (a, c, d)]
    last = 4 * k
    tris += [(0, 2, 1), (0, 3, 2), (last, last + 1, last + 2), (last, last + 2, last + 3)]
    t = np.array(tris, dtype=np.uint32)
    assert len(v) > 262144
    with pytest.raises(F.BlubError, match="262144"):
        F.mesh_body_properties(v, t, 2.0)
    F.mesh_body_properties(v[:4 * 1001], np.array(tris[:8 * 1000] + [(0, 2, 1), (0, 3, 2), (4000, 4001, 4002), (4000, 4002, 4003)], dtype=np.uint32), 2.0)


# ---- the cell rule ---------------------------------------------------------------------------------------------------------------
def check_against_winding_number(pos, tri, scale, b, dims=(48, 48, 48)):
    vb = F.mesh_body_vertices(pos, tri, scale)
    p = F.mesh_body_properties(pos, tri, scale)
    mid, half = M.mid_and_half(p)
    body = dict(b, shape="mesh", half_extent=tuple(float(h) for h in half))
    cube = M.cube_side([body], [mid])
    mask, _ = M.covered(dims, body, (mid, vb, tri), cube)
    vg = M.grid_vertices(body, vb)
    lo = np.floor(vg.min(0)).astype(int) - 1
    hi = np.ceil(vg.max(0)).astype(int) + 1
    z, y, x = np.meshgrid(*[np.arange(lo[k], hi[k]) for k in (2, 1, 0)], indexing="ij")
    pts = np.stack([x.ravel() + 0.5, y.ravel() + 0.5, z.ravel() + 0.5], -1)
    far = M.surface_distance(vg, tri, pts) > 1e-3
    inside = np.abs(M.winding_number(vg, tri, pts)) > 0.5
    got = mask[z.ravel(), y.ravel(), x.ravel()]
    assert far.sum() > 0.99 * len(pts)
    assert np.array_equal(got[far], inside[far])
    assert mask.sum() == got.sum() and inside.sum() > 20  # nothing beyond the mesh's box is marked
    return mask


@pytest.mark.parametrize("q", [(1.0, 0.0, 0.0, 0.0), TILT, TILT2])
def test_cell_rule_agrees_with_the_winding_number(q):
    c = (23.3, 22.71, 24.13)
    check_against_winding_number(*M.icosphere(2, 1.0), 7.0, body_ref.body("box", 1, 0.5, c, q))
    check_against_winding_number(*M.torus(2.0, 0.8, 24, 12), 4.0, body_ref.body("box", 1, 0.5, c, q))
    check_against_winding_number(*M.l_block(), 4.0, body_ref.body("box", 1, 0.5, c, q))


def parity_counts(pos, tri, b_centre, cube=24):
    """Crossings per row of a mesh placed unrotated with its model origin at b_centre (vertices straight from pos)."""
    vg = (np.asarray(pos, dtype=np.float32) + np.float32(b_centre)).astype(np.float32)
    return M.crossings(vg, tri, (0, 0, 0), cube)


def test_tie_rule_even_parity_on_edges_and_vertices():
    # octahedron centred on a row centre: vertices and edges exactly on rows
    for pos, tri in (M.octahedron(3.0), M.box_mesh((-3, -3, -3), (3, 3, 3)), M.box_mesh((-2.5, -2.5, -2.5), (2.5, 2.5, 2.5))):
        for centre in ((12.5, 12.5, 12.5), (12.0, 12.0, 12.0), (12.5, 12.0, 12.25)):
            rows = parity_counts(pos, tri, centre, cube=40)
            for key, firsts in rows.items():
                assert len(firsts) % 2 == 0, (key, firsts)
            assert rows  # the mesh is crossed at all


def test_permuting_triangles_and_corners_changes_nothing():
    rng = np.random.default_rng(3)
    for pos, tri in (M.octahedron(3.0), M.box_mesh((-3, -3, -3), (3, 3, 3)), M.l_block()):
        vg = (pos + np.float32(12.5)).astype(np.float32)
        base = {k: sorted(v) for k, v in M.crossings(vg, tri, (0, 0, 0), 40).items()}
        t2 = tri[rng.permutation(len(tri))]
        shift = rng.integers(0, 3, len(t2))
        t2 = np.stack([np.roll(t, -s) for t, s in zip(t2, shift)])
        other = {k: sorted(v) for k, v in M.crossings(vg, t2, (0, 0, 0), 40).items()}
        assert base == other


# ---- clamp and integration ----------------------------------------------------------------------------------------------------
def test_free_fall_and_the_asymmetric_floor_clamp():
    """Hand-worked: an L-block at rest above the floor falls one step of dt = 1/60 under g = -60: v_y = -1, c_y -= 1/60; placed with its
    lowest box corner below y = 1 it is lifted so that the corner is at exactly 1 + rounding, and its downward velocity is zeroed."""
    p = F.mesh_body_properties(*M.l_block(), 4.0)
    mid, half = M.mid_and_half(p)
    b = dict(body_ref.body("box", tuple(float(h) for h in half), 0.5, (20, 30, 20)), shape="mesh")
    g = (0.0, -60.0, 0.0)
    dt = float(f32(1.0 / 60.0))
    out = M.integrate(b, (0, 0, 0), (0, 0, 0), dt, g, (64, 64, 64), p["mass"], p["moments"], mid)
    assert out["velocity"] == (0.0, float(f32(dt) * f32(-60.0)), 0.0)
    assert out["centre"][1] == float(f32(30) + f32(dt) * f32(out["velocity"][1]))
    low = dict(b, centre=(20.0, float(f32(1.0) + half[1] - mid[1] - f32(0.25)), 20.0))
    out = M.integrate(low, (0, 0, 0), (0, 0, 0), dt, g, (64, 64, 64), p["mass"], p["moments"], mid)
    assert out["velocity"][1] == 0.0
    assert abs((f32(out["centre"][1]) + f32(mid[1])) - f32(half[1]) - 1.0) < 1e-5
    # the box body's clamp would rest the centre at 1 + half: the mesh's rests lower or higher by mid
    assert mid[1] != 0.0 and out["centre"][1] != float(f32(1.0) + half[1])
    # torque about the principal axes: alpha_j = tau_j / I_j with an identity pose
    out = M.integrate(b, (0, 0, 0), (0, 0, 1 << 8), dt, (0, 0, 0), (64, 64, 64), p["mass"], p["moments"], mid)
    assert out["angular_velocity"][2] == float(f32(dt) * (f32(1.0) / f32(p["moments"][2])))


# ---- state file version 16 --------------------------------------------------------------------------------------------------
import json  # noqa: E402
import os  # noqa: E402
import struct  # noqa: E402
import zlib  # noqa: E402

from tests import util  # noqa: E402
from tests.test_bodies_kat import BODY_SLOT  # noqa: E402
from tests.test_state_file import GRID, HEADER_BYTES, header, payloads, section, write  # noqa: E402

MESH_HEAD = struct.Struct("<4I4f6f2f20d")  # body, vertices, triangles, reserved; mass, moments; bounds lo, hi; scale, reserved; the float64s
assert MESH_HEAD.size == 224
L_POS, L_TRI = M.l_block()


def mesh_record(body, pos, tri, scale, rho, vertices=None, **override):
    p = F.mesh_body_properties(pos, tri, scale)
    vb = F.mesh_body_vertices(pos, tri, scale) if vertices is None else vertices
    f = dict(mass=float(f32(rho * p["volume"])), moments=[float(f32(rho * m)) for m in p["principal_moments"]], lo=p["bounds_lo"], hi=p["bounds_hi"],
             nv=len(vb), nt=len(tri))
    f.update(override)
    head = MESH_HEAD.pack(body, f["nv"], f["nt"], 0, f["mass"], *f["moments"], *f["lo"], *f["hi"], scale, 0.0, p["volume"], *p["centroid"],
                          *p["principal_moments"], *p["principal_rotation"], *np.asarray(p["inertia"]).ravel())
    return head + np.asarray(vb, dtype=np.float32).tobytes() + np.asarray(tri, dtype=np.uint32).tobytes(), p


def v16_bytes(records=None, count=None, shape=2, half=None, centre=(16.0, 16.0, 20.0), corrupt_crc=False, pad=b""):
    rec, p = mesh_record(0, L_POS, L_TRI, 3.0, 0.5)
    records = [rec] if records is None else records
    lo, hi = [f32(v) for v in p["bounds_lo"]], [f32(v) for v in p["bounds_hi"]]
    half = [float(f32(0.5) * (hi[k] - lo[k])) for k in range(3)] if half is None else half
    data = bytearray(header(version=16))
    data[HEADER_BYTES - 8:HEADER_BYTES - 4] = struct.pack("<I", 16)
    data[HEADER_BYTES - 4:HEADER_BYTES] = struct.pack("<I", zlib.crc32(bytes(data[:HEADER_BYTES - 4])))
    out = bytes(data)
    for sid, pl in enumerate(payloads(), start=1):
        out += section(sid, pl)
    out += section(14, bytes(1056))
    slot = BODY_SLOT.pack(shape, *half, 0.5, *centre, 1.0, 0.0, 0.0, 0.0, 0, 0, 0, 0, 0, 0)
    out += section(15, struct.pack("<I", 1) + slot + bytes(72 * 15))
    payload = struct.pack("<II", len(records) if count is None else count, 0) + b"".join(records) + pad
    sec = section(16, payload)
    if corrupt_crc:
        sec = sec[:-4] + struct.pack("<I", zlib.crc32(payload) ^ 1)
    return out + sec


def test_version_16_written_from_the_documented_layout_is_accepted(tmp_path):
    info = F.state_info(write(tmp_path, v16_bytes()))
    assert info.format_version == 16 and tuple(info.grid_dimension) == GRID


@pytest.mark.parametrize("case, make, needle", [
    ("no record", lambda: v16_bytes(records=[]), "its header describes"),  # shorter than the smallest section 16
    ("count zero", lambda: v16_bytes(count=0, pad=bytes(224 + 8)), "at least one mesh body"),
    ("bad CRC", lambda: v16_bytes(corrupt_crc=True), "checksum mismatch in section 16"),
    ("bytes beyond the records", lambda: v16_bytes(pad=b"\0\0\0\0"), "beyond the last record"),
    ("count above the records", lambda: v16_bytes(count=2), "truncated record"),
    ("record for a box", lambda: v16_bytes(shape=0, half=[3.0, 3.0, 3.0]), "names no mesh body"),
    ("index out of range", lambda: v16_bytes(records=[mesh_record(0, L_POS, L_TRI, 3.0, 0.5)[0][:-4] + struct.pack("<I", 999)]), "out of range"),
    ("zero mass", lambda: v16_bytes(records=[mesh_record(0, L_POS, L_TRI, 3.0, 0.5, mass=0.0)[0]]), "mass"),
    ("bounds not the vertices'", lambda: v16_bytes(records=[mesh_record(0, L_POS, L_TRI, 3.0, 0.5, lo=(-9.0, -9.0, -9.0))[0]]), "bound"),
    ("half extent not the bounds'", lambda: v16_bytes(half=[5.0, 5.0, 5.0]), "bound"),
    ("outside the tank", lambda: v16_bytes(centre=(2.0, 16.0, 20.0)), "bounding box"),
])
def test_malformed_version_16_files_are_parse_errors(tmp_path, case, make, needle):
    path = write(tmp_path, make())
    L = F.lib()
    rc = L.blub_state_info(os.fsencode(path), F.StateInfo())
    assert rc == 5, case
    assert needle in L.blub_last_error().decode(), (case, L.blub_last_error().decode())


# ---- scene key --------------------------------------------------------------------------------------------------------------
def v3(x, y, z):
    return {"x": x, "y": y, "z": z}


def write_obj(path, pos, tri):
    with open(path, "w") as f:
        f.writelines(f"v {x} {y} {z}\n" for x, y, z in pos)
        f.writelines(f"f {a + 1} {b + 1} {c + 1}\n" for a, b, c in tri)


def mesh_scene(tmp_path, bodies, sub="scenes"):
    d = tmp_path / sub
    d.mkdir(exist_ok=True)
    write_obj(str(d / "l.obj"), L_POS, L_TRI)
    sc = json.load(open(util.scene_path("dam_small")))  # 32^3 cells of 0.01 m
    sc["fluid"]["bodies"] = bodies
    path = str(d / "s.json")
    json.dump(sc, open(path, "w"))
    return path


MESH = {"shape": "mesh", "model": "l.obj", "scale": 0.03, "position": v3(0.12, 0.14, 0.16), "relative_density": 0.5,
        "rotation_angles_deg": v3(0.0, 30.0, 0.0)}


def test_scene_mesh_bodies_resolve_their_model_and_convert(tmp_path):
    path = mesh_scene(tmp_path, [MESH, {"shape": "sphere", "position": v3(0.08, 0.08, 0.08), "half_extent": 0.03, "relative_density": 2.0}])
    got = F.scene_bodies(path)
    assert got[0]["shape"] == "mesh" and got[1]["shape"] == "sphere"
    assert got[0]["centre"] == tuple(float(f32(v) / f32(0.01)) for v in (0.12, 0.14, 0.16))  # the model origin: its placement
    model, scale = F.scene_body_model(path, 0)
    assert model == str(tmp_path / "scenes" / "l.obj") and scale == f32(0.03) / f32(0.01)
    with pytest.raises(F.BlubError):
        F.scene_body_model(path, 1)
    F.scene_info(path)


@pytest.mark.parametrize("what, body", [
    ("missing model", {k: v for k, v in MESH.items() if k != "model"}),
    ("missing file", dict(MESH, model="nope.obj")),
    ("zero scale", dict(MESH, scale=0.0)),
    ("thin", dict(MESH, scale=0.002)),
    ("outside the tank", dict(MESH, position=v3(0.29, 0.14, 0.16))),
    ("zero density", dict(MESH, relative_density=0.0)),
])
def test_bad_scene_mesh_bodies_are_parse_errors(tmp_path, what, body):
    path = mesh_scene(tmp_path, [body])
    assert F.lib().blub_scene_info(os.fsencode(path), F.SceneInfo()) == 5, what


def test_an_open_model_is_a_parse_error(tmp_path):
    path = mesh_scene(tmp_path, [MESH])
    write_obj(os.path.join(os.path.dirname(path), "l.obj"), L_POS, L_TRI[1:])
    assert F.lib().blub_scene_info(os.fsencode(path), F.SceneInfo()) == 5
    assert "not closed" in F.lib().blub_last_error().decode()


def test_a_shape_mesh_dict_without_a_mesh_is_a_blub_error():
    arr = F.Body.from_dict(dict(body_ref.body(), shape="mesh"))
    assert arr.shape == 2
    with pytest.raises(F.BlubError):
        F.Body.from_dict(dict(body_ref.body(), shape="cone"))
